"""The KITTI object devkit's evaluate_object (Car) restated as plain sequential Python in fp64 (DESIGN.md §9): the
checker of csrc/kitti_eval.cu, in the same operation order, so the two agree bit for bit (AOS to the last bits of cos).

Rows are the packed rows of the device ABI (SB_KITTI_ROW = 16 doubles: trunc, occ, alpha, x1, y1, x2, y2, h, w, l,
x, y, z, cos(ry), sin(ry), score) with an int code per row (0 Car, 1 Van, 2 DontCare, 3 other).  An image is a tuple
(gt_rows, gt_codes, det_rows, det_codes).  Test infrastructure only."""
import math

import numpy as np

TRUNC, OCC, ALPHA, X1, Y1, X2, Y2, H, W, L, X, Y, Z, COS, SIN, SCORE = range(16)
DONTCARE = 2
N_T = 41
MAX_POLY = 16
NO_MATCH = -10000000.0
MIN_HEIGHT = (40.0, 25.0, 25.0)
MAX_OCCLUSION = (0.0, 1.0, 2.0)
MAX_TRUNCATION = (0.15, 0.30, 0.50)


# ------------------------------------------------------------------------------------------------ overlaps ----
def bev_corners(r):
    """the rectangle of a row in the x-z plane, counter-clockwise"""
    hl, hw, c, s = r[L] * 0.5, r[W] * 0.5, r[COS], r[SIN]
    x, z = [], []
    for dx, dz in ((hl, hw), (hl, -hw), (-hl, -hw), (-hl, hw)):
        x.append(r[X] + (c * dx + s * dz))
        z.append(r[Z] + (c * dz - s * dx))
    a = 0.0
    for k in range(4):
        k1 = (k + 1) & 3
        a = a + (x[k] * z[k1] - x[k1] * z[k])
    order = (0, 3, 2, 1) if a < 0.0 else (0, 1, 2, 3)
    return [x[k] for k in order], [z[k] for k in order]


def _side(ax, az, ex, ez, x, z):
    return ex * (z - az) - ez * (x - ax)


def bev_intersection(d, g):
    """area of det's rectangle clipped by gt's (Sutherland-Hodgman), by the shoelace formula"""
    cx, cz = d[X] - g[X], d[Z] - g[Z]
    rd = math.sqrt(d[L] * d[L] + d[W] * d[W]) * 0.5
    rg = math.sqrt(g[L] * g[L] + g[W] * g[W]) * 0.5
    rr = rd + rg
    if cx * cx + cz * cz > rr * rr:                    # circumscribed circles apart
        return 0.0
    qx, qz = bev_corners(g)
    px, pz = bev_corners(d)
    for e in range(4):
        if not px:
            break
        ax, az = qx[e], qz[e]
        ex, ez = qx[(e + 1) & 3] - ax, qz[(e + 1) & 3] - az
        n = len(px)
        ox, oz = [], []
        for k in range(n):
            kp = n - 1 if k == 0 else k - 1
            cc = _side(ax, az, ex, ez, px[k], pz[k])
            cp = _side(ax, az, ex, ez, px[kp], pz[kp])
            if (cc >= 0.0) != (cp >= 0.0) and len(ox) < MAX_POLY:
                t = cp / (cp - cc)
                ox.append(px[kp] + t * (px[k] - px[kp]))
                oz.append(pz[kp] + t * (pz[k] - pz[kp]))
            if cc >= 0.0 and len(ox) < MAX_POLY:
                ox.append(px[k])
                oz.append(pz[k])
        px, pz = ox, oz
    n = len(px)
    if n < 3:
        return 0.0
    a = 0.0
    for k in range(n):
        k1 = 0 if k + 1 == n else k + 1
        a = a + (px[k] * pz[k1] - px[k1] * pz[k])
    return abs(a) * 0.5


def _ratio(inter, area_d, area_g, crit0):
    den = area_d if crit0 else (area_d + area_g) - inter
    return 0.0 if den == 0.0 else inter / den


def overlap_2d(d, g, crit0=False):
    iw = min(d[X2], g[X2]) - max(d[X1], g[X1])
    ih = min(d[Y2], g[Y2]) - max(d[Y1], g[Y1])
    if not (iw > 0.0 and ih > 0.0):
        return 0.0
    return _ratio(iw * ih, (d[X2] - d[X1]) * (d[Y2] - d[Y1]), (g[X2] - g[X1]) * (g[Y2] - g[Y1]), crit0)


def overlap_bev(d, g, crit0=False, inter=None):
    inter = bev_intersection(d, g) if inter is None else inter
    return _ratio(inter, d[L] * d[W], g[L] * g[W], crit0)


def overlap_3d(d, g, crit0=False, inter=None):
    inter = bev_intersection(d, g) if inter is None else inter
    ih = max(0.0, min(d[Y], g[Y]) - max(d[Y] - d[H], g[Y] - g[H]))
    return _ratio(inter * ih, (d[H] * d[W]) * d[L], (g[H] * g[W]) * g[L], crit0)


def overlaps(gt, gt_codes, det):
    """-> three [n_det, n_gt] fp64 matrices (2D, BEV, 3D); DontCare columns hold intersection / area(det)"""
    gt, det = [list(map(float, r)) for r in np.asarray(gt)], [list(map(float, r)) for r in np.asarray(det)]
    out = np.zeros((3, len(det), len(gt)))
    for j, d in enumerate(det):
        for i, g in enumerate(gt):
            crit0 = int(gt_codes[i]) == DONTCARE
            inter = bev_intersection(d, g)
            out[0, j, i] = overlap_2d(d, g, crit0)
            out[1, j, i] = overlap_bev(d, g, crit0, inter)
            out[2, j, i] = overlap_3d(d, g, crit0, inter)
    return out


# ------------------------------------------------------------------------------------------------ matching ----
def gt_flags(gt, codes, d):
    out = []
    for r, c in zip(gt, codes):
        if c == 1:
            out.append(1)
        elif c != 0:
            out.append(-1)
        else:
            hard = r[OCC] > MAX_OCCLUSION[d] or r[TRUNC] > MAX_TRUNCATION[d] or (r[Y2] - r[Y1]) <= MIN_HEIGHT[d]
            out.append(1 if hard else 0)
    return out


def det_flags(det, codes, d):
    return [1 if (r[Y2] - r[Y1]) < MIN_HEIGHT[d] else (0 if c == 0 else -1) for r, c in zip(det, codes)]


def above(ov, n_gt, bar):
    """per gt column, the detections (row order) whose overlap is above the bar: every branch of stats() requires
    o > bar, so the others are skipped without changing anything"""
    return [[(j, ov[j][i]) for j in range(len(ov)) if ov[j][i] > bar] for i in range(n_gt)]


def stats(cand, ig, idf, gt_codes, score, alpha_gt, alpha_det, compute_fp, thresh=0.0):
    """computeStatistics for one image: cand = above(ov, n_gt, bar) of the metric -> (tp, fp, fn, sim, tp_scores)"""
    nd = len(idf)
    assigned = [False] * nd
    ignored_thr = [compute_fp and score[j] < thresh for j in range(nd)]
    tp = fp = fn = 0
    sim = 0.0
    tp_scores = []
    for i in range(len(ig)):
        if ig[i] == -1:
            continue
        best, valid, max_iou, took_ignored = -1, NO_MATCH, 0.0, False
        for j, o in cand[i]:
            if idf[j] == -1 or assigned[j] or ignored_thr[j]:
                continue
            if not compute_fp and score[j] > valid:
                best, valid = j, score[j]
            elif compute_fp and (o > max_iou or took_ignored) and idf[j] == 0:
                max_iou, best, valid, took_ignored = o, j, 1.0, False
            elif compute_fp and valid == NO_MATCH and idf[j] == 1:
                best, valid, took_ignored = j, 1.0, True
        if valid == NO_MATCH and ig[i] == 0:
            fn += 1
        elif valid != NO_MATCH and (ig[i] == 1 or idf[best] == 1):
            assigned[best] = True
        elif valid != NO_MATCH:
            tp += 1
            tp_scores.append(score[best])
            sim = sim + (1.0 + math.cos(alpha_gt[i] - alpha_det[best])) * 0.5
            assigned[best] = True
    if compute_fp:
        fp = sum(1 for j in range(nd) if not assigned[j] and idf[j] == 0 and not ignored_thr[j])
        for c in range(len(ig)):
            if gt_codes[c] != DONTCARE:
                continue
            for j, _o in cand[c]:
                if assigned[j] or idf[j] != 0 or ignored_thr[j]:
                    continue
                assigned[j] = True
                fp -= 1
    return tp, fp, fn, sim, tp_scores


def thresholds(scores, n_gt):
    """getThresholds: sorted descending, the scores nearest the 41 recall points"""
    v = sorted(scores, reverse=True)
    out, cur = [], 0.0
    for i in range(len(v)):
        if len(out) == N_T:
            break
        l = float(i + 1) / float(n_gt)
        r = float(i + 2) / float(n_gt) if i < len(v) - 1 else l
        if (r - cur) < (cur - l) and i < len(v) - 1:
            continue
        out.append(v[i])
        cur = cur + 1.0 / 40.0
    return out


def evaluate(images, bars=(0.7, 0.5)):
    """images: list of (gt_rows [n,16], gt_codes, det_rows [m,16], det_codes) -> dict of the sb_kitti_eval outputs,
    configuration c = (metric * len(bars) + bar) * 3 + difficulty"""
    prep = []
    for g, gc, dt, dc in images:
        g = [list(map(float, r)) for r in np.asarray(g, np.float64).reshape(-1, 16)]
        dt = [list(map(float, r)) for r in np.asarray(dt, np.float64).reshape(-1, 16)]
        gc, dc = [int(c) for c in gc], [int(c) for c in dc]
        ov = overlaps(g, gc, dt)
        prep.append((g, gc, dt, dc, [m.tolist() for m in ov]))
    C = 9 * len(bars)
    res = dict(thresholds=np.zeros((C, N_T)), n_thresholds=np.zeros(C, np.int32), tp=np.zeros((C, N_T), np.int64),
               fp=np.zeros((C, N_T), np.int64), fn=np.zeros((C, N_T), np.int64), sim=np.zeros((C, N_T)),
               precision=np.zeros((C, N_T)), recall=np.zeros((C, N_T)), aos=np.zeros((C, N_T)),
               ap=np.zeros((C, 4)), n_gt=np.zeros(C, np.int64))
    for cfg in range(C):
        d, bar, metric = cfg % 3, bars[(cfg // 3) % len(bars)], cfg // (3 * len(bars))
        per = []
        for g, gc, dt, dc, ov in prep:
            per.append((above(ov[metric], len(g), bar), gt_flags(g, gc, d), det_flags(dt, dc, d), gc, [r[SCORE] for r in dt],
                        [r[ALPHA] for r in g], [r[ALPHA] for r in dt]))
        scores, n_gt = [], 0
        for ov, ig, idf, gc, sc, ag, ad in per:
            scores += stats(ov, ig, idf, gc, sc, ag, ad, False)[4]
            n_gt += sum(1 for f in ig if f == 0)
        thr = thresholds(scores, n_gt)
        res["n_gt"][cfg], res["n_thresholds"][cfg] = n_gt, len(thr)
        prec, aos = [0.0] * N_T, [0.0] * N_T
        for t, th in enumerate(thr):
            tp = fp = fn = 0
            sim = 0.0
            for ov, ig, idf, gc, sc, ag, ad in per:
                a, b, c, s, _ = stats(ov, ig, idf, gc, sc, ag, ad, True, th)
                tp, fp, fn, sim = tp + a, fp + b, fn + c, sim + s
            res["thresholds"][cfg, t] = th
            res["tp"][cfg, t], res["fp"][cfg, t], res["fn"][cfg, t], res["sim"][cfg, t] = tp, fp, fn, sim
            prec[t] = 0.0 if tp + fp == 0 else float(tp) / float(tp + fp)
            res["recall"][cfg, t] = 0.0 if tp + fn == 0 else float(tp) / float(tp + fn)
            aos[t] = 0.0 if tp + fp == 0 else sim / float(tp + fp)
        for k in range(N_T - 2, -1, -1):
            prec[k] = max(prec[k], prec[k + 1])
            aos[k] = max(aos[k], aos[k + 1])
        res["precision"][cfg], res["aos"][cfg] = prec, aos
        p11 = a11 = p40 = a40 = 0.0
        for k in range(0, N_T, 4):
            p11, a11 = p11 + prec[k], a11 + aos[k]
        for k in range(1, N_T):
            p40, a40 = p40 + prec[k], a40 + aos[k]
        res["ap"][cfg] = [p11 / 11.0 * 100.0, p40 / 40.0 * 100.0, a11 / 11.0 * 100.0, a40 / 40.0 * 100.0]
    return res
