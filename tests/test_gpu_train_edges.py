"""GPU: the train-time target layers and losses (csrc/train_targets.cu, csrc/train_loss.cu) at their edges, against the
CPU oracle (oracle/train_targets.py) on the same inputs and the same random words.

The inputs are built on the CPU so that every branch of the kernels is taken (tests/test_train_args.py counts them
without a GPU):

  IoU thresholds  anchors / RoIs bisected on the fp32 lattice (np.nextafter steps) until the oracle's stepwise-fp32 IoU
                  straddles 0.7 / 0.3 (RPN) or 0.5 (FG_THRESH, BG_THRESH_HI): each pair is the last coordinate with
                  IoU >= t and its neighbour one ulp away.  Many land exactly on float32(t), and at least ten pairs per
                  threshold would flip under an FMA-contracted union fmaf(ax, ay, garea) - inter.  BG_THRESH_LO 0.0:
                  RoIs touching a box (IoU exactly 0) and point boxes (-1).
  argmax ties     duplicate gt rows, zero-padded gt rows between real rows, anchors equidistant from two boxes, and
                  anchors overlapping nothing (every IoU 0): the first index wins, as torch.max on the CPU.
  K               1, 31, 32, 33, 63, 64 (both instances of the overlap kernel, the last box always real and unique).
  image edges     anchors at x1 / y1 = 0 and x2 / y2 = W / H and one ulp inside and outside, gt boxes on the border.
  sampler keys    all equal, 2- and 4-value alphabets (a threshold tie across several 1024-anchor blocks), keys that
                  differ only in the low byte or only in bytes 1-2, increasing / decreasing keys, {0, 0xFFFFFFFF}.
  batches         RPN_BATCHSIZE 1, 7, 256, 512 and more than the anchors, num_fg = 0, B = 1, 2, 4 with a last image
                  without ground truth or with many more foreground anchors (the outside weight is the last image's).
  proposals       R + K = 4096, BATCH_SIZE 1 / 100 / 512 / 1024, FG_FRACTION 0 / 0.25 / 1, more than 1024 foreground
                  candidates, zero-padded proposal rows, gt classes 1..3, KPTS_GRID 14, no candidate at all.
  losses          B*A = 1 ... 2 x 298 476 around the 131 072 threads of the partial-sum grid, logits of +-60, smooth-L1
                  arguments at float32(1/9) and one ulp either side; R = 1 ... 2048 rows with C = 2..4 classes, a batch
                  without class 1 and fractional keypoint weights (sum < 1); clip_gradient over 47 ... 97 tensors of
                  1..31 elements and a norm exactly at the clip value.

Bars (DESIGN.md 4.4): labels, keep_inds, weights, integer keypoint targets and status bit-exact; box regression targets
bit-exact in dx / dy; in dw / dh within one ulp of the oracle with a correctly rounded log (anchor targets) or two
after the division by BBOX_NORMALIZE_STDS 0.2 (proposal targets); losses within 2e-6 (RPN) / 3e-6 (R-CNN) relative and gradients within 1e-6 / 2e-6 of their maximum of
torch autograd of oracle.rpn_losses / rcnn_losses in float64 on the CPU; clip_gradient's scaled tensors bit-exact.
Every loss test prints its worst measured error."""
import collections
import contextlib
import math

import numpy as np
import pytest
import torch

from oracle import ops as O
from oracle import train_targets as T
from stereo_rcnn_b200 import synth
from stereo_rcnn_b200 import train as G

pytestmark = pytest.mark.gpu

F32 = np.float32
HUGE_BATCH = 1 << 20                 # no subsampling: every label of the threshold cases stays visible
KEY_PATTERNS = ("uniform", "equal", "alpha2", "alpha4", "low", "mid", "inc", "dec", "ext")

Case = collections.namedtuple("Case", "id kind p")


def _c(kind, name, **p):
    return Case("%s-%s" % (kind, name), kind, p)


# ---------------------------------------------------------------------------------------------- CPU builders
def feat_shapes(H, W):
    return [[int(np.ceil(H / s)), int(np.ceil(W / s))] for s in (4, 8, 16, 32, 64)]


def pyramid(H, W):
    return O.anchors_all_pyramids(feat_shapes(H, W)).astype(F32)


def make_keys(pattern, shape, seed):
    rs = np.random.RandomState(seed)
    u = rs.randint(0, 2 ** 32, shape, dtype=np.uint64).astype(np.uint32)
    n = shape[-1]
    if pattern == "uniform":
        return u
    if pattern == "equal":
        return np.full(shape, 0x5A5A5A5A, np.uint32)
    if pattern in ("alpha2", "alpha4"):
        alpha = rs.randint(0, 2 ** 32, int(pattern[-1]), dtype=np.uint64).astype(np.uint32)
        return alpha[rs.randint(0, alpha.size, shape)]
    if pattern == "low":                                  # the three high bytes shared: the first radix passes see one bucket
        return (np.uint32(0xABCDEF00) | (u & np.uint32(0xFF))).astype(np.uint32)
    if pattern == "mid":                                  # only bytes 1-2 differ
        return (np.uint32(0xAB0000CD) | (u & np.uint32(0xFFFF00))).astype(np.uint32)
    if pattern in ("inc", "dec"):
        k = (np.arange(n, dtype=np.uint64) * (2 ** 32 // max(n, 1))).astype(np.uint32)
        k = k if pattern == "inc" else k[::-1].copy()
        return np.broadcast_to(k, shape).copy()
    if pattern == "ext":
        return np.where(u & np.uint32(1), np.uint32(0xFFFFFFFF), np.uint32(0)).astype(np.uint32)
    raise ValueError(pattern)


def iou32(a, g, fma=False):
    """one entry of bbox_overlaps_batch per row of a [n,4] against g [n,4], stepwise fp32 in the oracle's order; fma:
    the union as fmaf(ax, ay, garea) - inter (a contracted multiply-add, emulated exactly in float64)"""
    a, g = np.asarray(a, F32), np.asarray(g, F32)
    one = F32(1)
    gx, gy = g[:, 2] - g[:, 0] + one, g[:, 3] - g[:, 1] + one
    ax, ay = a[:, 2] - a[:, 0] + one, a[:, 3] - a[:, 1] + one
    iw = np.maximum(np.minimum(a[:, 2], g[:, 2]) - np.maximum(a[:, 0], g[:, 0]) + one, F32(0))
    ih = np.maximum(np.minimum(a[:, 3], g[:, 3]) - np.maximum(a[:, 1], g[:, 1]) + one, F32(0))
    inter = iw * ih
    if fma:
        s = (ax.astype(np.float64) * ay.astype(np.float64) + (gx * gy).astype(np.float64)).astype(F32)
    else:
        s = ax * ay + gx * gy
    return inter / (s - inter)


def boundary_pairs(g, t, rng):
    """anchors contained in the boxes g [n,4] whose x2 is bisected on the fp32 lattice: -> (hi, lo), hi the last x2 with
    IoU >= t, lo one ulp below it with IoU < t"""
    g = np.asarray(g, F32)
    n = g.shape[0]
    w, h = g[:, 2] - g[:, 0], g[:, 3] - g[:, 1]
    a = g.copy()
    a[:, 0] = g[:, 0] + F32(rng.uniform(0, 0.06, n)) * w
    a[:, 1] = g[:, 1] + F32(rng.uniform(0, 0.06, n)) * h
    a[:, 3] = g[:, 3] - F32(rng.uniform(0, 0.06, n)) * h
    lo, hi = a[:, 0].copy().view(np.int32).astype(np.int64), g[:, 2].copy().view(np.int32).astype(np.int64)

    def at(xi):
        b = a.copy()
        b[:, 2] = xi.astype(np.int32).view(F32)
        return b
    assert (iou32(at(lo), g) < t).all() and (iou32(at(hi), g) >= t).all()
    while True:
        m = hi - lo > 1
        if not m.any():
            break
        mid = lo + (hi - lo) // 2
        ge = iou32(at(mid), g) >= t
        hi, lo = np.where(m & ge, mid, hi), np.where(m & ~ge, mid, lo)
    return at(hi), at(lo)


def fma_flips(hi, lo, g, t):
    """pairs whose compare against t an FMA-contracted union would flip"""
    return (iou32(hi, g, fma=True) < t) | (iou32(lo, g, fma=True) >= t)


def grid_boxes(K, H, W, rng, integer=False, fill=0.6):
    """K disjoint boxes, one per cell of a grid over the image (gaps of at least 12 % of a cell between them);
    integer: whole-pixel corners and one common size (ties by symmetry are exact)"""
    cols = int(math.ceil(math.sqrt(K * W / float(H))))
    rows = int(math.ceil(K / float(cols)))
    cw, ch = W / float(cols), H / float(rows)
    out = np.zeros((K, 4), F32)
    for k in range(K):
        r, c = divmod(k, cols)
        if integer:
            w, h = math.floor(cw * fill), math.floor(ch * fill)
            x1, y1 = math.floor(c * cw + (cw - w) / 2), math.floor(r * ch + (ch - h) / 2)
        else:
            w, h = cw * fill * rng.uniform(0.8, 1.0), ch * fill * rng.uniform(0.8, 1.0)
            x1, y1 = c * cw + (cw - w) * rng.uniform(0.3, 0.7), r * ch + (ch - h) * rng.uniform(0.3, 0.7)
        out[k] = [x1, y1, x1 + w, y1 + h]
    return out, cols


def gt_tables(box, rng, disparity=6.0, cls=None):
    """[B,K,4] left boxes (all-zero rows = padding) -> gt_left, gt_right [B,K,5], gt_dim_orien [B,K,5], gt_kpts [B,K,6]"""
    B, K = box.shape[:2]
    real = np.abs(box).sum(2) > 0
    gl = np.zeros((B, K, 5), F32)
    gl[:, :, :4] = box
    gl[:, :, 4] = np.where(real, 1 if cls is None else cls, 0)
    gr = gl.copy()
    gr[:, :, 0] -= F32(disparity)
    gr[:, :, 2] -= F32(disparity)
    gr[~real] = 0
    dim = rng.uniform(-1, 4, (B, K, 5)).astype(F32)
    kp = np.full((B, K, 6), -1, F32)
    for b in range(B):
        for k in range(K):
            x1, x2 = float(gl[b, k, 0]), float(gl[b, k, 2])
            kp[b, k, rng.randint(4)] = rng.uniform(x1, x2)
            kp[b, k, 4] = rng.uniform(x1, x1 + 0.3 * (x2 - x1))
            kp[b, k, 5] = rng.uniform(x2 - 0.3 * (x2 - x1), x2)
    return gl, gr, dim, kp


def merge(gl, gr):
    gm = gl.copy()
    gm[:, :, 0] = np.minimum(gl[:, :, 0], gr[:, :, 0])
    gm[:, :, 2] = np.maximum(gl[:, :, 2], gr[:, :, 2])
    return gm


# ------------------------------------------------------------------------------------------ anchor targets
def at_inputs(c):
    """-> dict(anchors [A,4], gl, gr, gm [B,K,5], H, W, keys [B,A] uint32, cfg, thr: thresholds whose both sides the
    case must reach)"""
    p = c.p
    rng = np.random.RandomState(p["seed"])
    H, W, fam = p["H"], p["W"], p["fam"]
    cfg = dict(T.CFG, RPN_BATCHSIZE=p.get("batch", 512), RPN_FG_FRACTION=p.get("frac", 0.5))
    thr, pairs = (), []
    if fam == "bound":                                  # threshold pairs around 0.7 and 0.3, B = 1
        K = p["K"]
        box, _ = grid_boxes(K, H, W, rng)
        parts = [box]                                   # identity anchors: every box's maximum IoU is 1
        for t, n in zip((0.7, 0.3), p["pairs"]):        # FMA flips are rarer at 0.3: more pairs there
            g = box[rng.randint(K, size=n)]
            hi, lo = boundary_pairs(g, F32(t), rng)
            parts += [hi, lo]
            pairs.append((t, hi, lo, g))
        anchors = np.concatenate(parts)
        gm = np.zeros((1, K, 5), F32)
        gm[0, :, :4] = box
        gm[0, :, 4] = 1
        off = np.zeros((1, K, 4), F32)
        off[..., 0] = rng.uniform(0, 2, K)              # left boxes a little inside the merged ones
        gl, gr, _, _ = gt_tables(box[None] + off, rng)
        cfg["RPN_BATCHSIZE"] = HUGE_BATCH
        thr = (0.7, 0.3)
    elif fam == "tie":                                  # duplicate rows, zero rows between real ones, equidistant anchors
        K = p["K"]
        box, cols = grid_boxes(K, H, W, rng, integer=True)
        gm_box = box.copy()
        if K >= 4:
            gm_box[[1, K // 3]] = 0                     # zero-padded rows between real rows
            gm_box[K // 2] = gm_box[2]                  # a duplicate of an earlier row (last row stays unique)
        real = np.abs(gm_box).sum(1) > 0
        parts = [pyramid(H, W), gm_box[real]]
        w = box[0, 2] - box[0, 0]
        for k in range(K - 1):                          # equidistant from two horizontal neighbours
            if (k + 1) % cols and real[k] and real[k + 1]:
                o = F32(math.floor(w / 3))
                y = box[k, [1, 3]]
                parts.append(np.array([[box[k, 2] - o, y[0], box[k + 1, 0] + o, y[1]]], F32))
        anchors = np.concatenate(parts)
        jit = F32(rng.uniform(-1.5, 1.5, (1, K, 4))) * real[None, :, None]
        gl, gr, _, _ = gt_tables(gm_box[None] + jit, rng)   # distinct left / right rows behind the duplicate
        gm = np.zeros((1, K, 5), F32)
        gm[0, :, :4] = gm_box
        gm[0, :, 4] = real
    elif fam == "edge":                                 # anchors on and one ulp around the image border
        d = np.nextafter(F32(0), F32(1))
        bx = np.array([[0, 0, 60.5, 40.25], [W - 1 - 50.5, H - 1 - 40.75, W - 1, H - 1], [0, H - 1 - 30.5, 45.25, H - 1],
                       [W - 1 - 70.25, 0, W - 1, 35.5], [100.5, 50.25, 140.75, 90.5]], F32)
        parts = [pyramid(H, W), bx]
        for j, (xe, ye) in enumerate(((0, 0), (W, H), (0, H), (W, 0))):
            for v in ((-d, F32(0), d) if xe == 0 else (np.nextafter(F32(W), F32(0)), F32(W), np.nextafter(F32(W), F32(W + 1)))):
                a = bx[j].copy()
                a[0 if xe == 0 else 2] = v
                parts.append(a[None])
            for v in ((-d, F32(0), d) if ye == 0 else (np.nextafter(F32(H), F32(0)), F32(H), np.nextafter(F32(H), F32(H + 1)))):
                a = bx[j].copy()
                a[1 if ye == 0 else 3] = v
                parts.append(a[None])
        anchors = np.concatenate(parts)
        gl, gr, _, _ = gt_tables(bx[None], rng)
        gr[0, :, 0] = np.maximum(gr[0, :, 0], 0)
        gm = merge(gl, gr)
    else:                                               # "pyr": the anchor pyramid and synthetic ground truth
        B, K = p["B"], p.get("K", 30)
        gl, gr, gm, _, _, _ = synth.synth_train_gt(B, K, H, W, p["seed"], n_boxes=p.get("n_boxes"))
        anchors = pyramid(H, W)
    keys = make_keys(p.get("keys", "uniform"), (gl.shape[0], anchors.shape[0]), p["seed"] + 1)
    return dict(anchors=np.ascontiguousarray(anchors, F32), gl=gl, gr=gr, gm=gm, H=H, W=W, keys=keys, cfg=cfg, thr=thr,
                pairs=pairs)


@contextlib.contextmanager
def rounded_log():
    """the oracle's float32 log correctly rounded (float64 log, one rounding): numpy's own float32 log can be 2-3 ulp
    off, the device's logf at most one"""
    log = np.log

    def log32(x, *a, **k):
        x = np.asarray(x)
        return log(x.astype(np.float64), *a, **k).astype(F32) if x.dtype == F32 else log(x, *a, **k)
    np.log = log32
    try:
        yield
    finally:
        np.log = log


def at_oracle(inp):
    with rounded_log():
        return _at_oracle(inp)


def _at_oracle(inp):
    return T.anchor_target_layer(inp["anchors"], inp["gl"], inp["gr"], inp["gm"],
                                 np.array([[inp["H"], inp["W"], 1.0]] * inp["gl"].shape[0], F32),
                                 T.KeySampler(inp["keys"]), inp["cfg"])


def at_max_overlap(inp):
    """[B,A] max IoU per anchor (NaN outside the image) and the inside mask"""
    a = inp["anchors"]
    keep = (a[:, 0] >= 0) & (a[:, 1] >= 0) & (a[:, 2] < inp["W"]) & (a[:, 3] < inp["H"])
    mx = np.full((inp["gl"].shape[0], a.shape[0]), np.nan, F32)
    mx[:, keep] = T.bbox_overlaps_batch(a[keep], inp["gm"]).max(2)
    return mx, keep


def select_cells(cand, keys, keep):
    """what at_sample does with one (image, side): candidates `cand` (anchor indices, ascending), keep -> cell names"""
    n = cand.size
    if n <= keep:
        return ["no sampling"]
    want = n - keep
    if want >= n:
        return ["everything goes"]
    k = keys[cand]
    order = np.lexsort((cand, k))
    T_ = k[order[want - 1]]
    d = want - int((k < T_).sum())
    tied = cand[k == T_]
    if d == tied.size:
        return ["unique threshold"]
    out = ["threshold tie"]
    if tied[d - 1] >= 1024:
        out.append("tie past the first 1024-block")
    return out


def at_cells(c, inp=None):
    """branch cells an anchor-target case reaches (evaluated with the oracle on the CPU)"""
    inp = inp or at_inputs(c)
    cfg = inp["cfg"]
    cnt = collections.Counter()
    K = inp["gl"].shape[1]
    cnt["K <= 32" if K <= 32 else "K > 32"] += 1
    pre = T.anchor_target_layer(inp["anchors"], inp["gl"], inp["gr"], inp["gm"],
                                np.array([[inp["H"], inp["W"], 1.0]] * inp["gl"].shape[0], F32),
                                T.KeySampler(inp["keys"]), dict(cfg, RPN_BATCHSIZE=HUGE_BATCH))[0]
    num_fg = int(cfg["RPN_FG_FRACTION"] * cfg["RPN_BATCHSIZE"])
    for b in range(pre.shape[0]):
        fg, bg = np.nonzero(pre[b] == 1)[0], np.nonzero(pre[b] == 0)[0]
        for side, cand, keep in (("fg", fg, num_fg), ("bg", bg, cfg["RPN_BATCHSIZE"] - fg.size)):
            for cell in select_cells(cand, inp["keys"][b], keep):
                cnt[cell] += 1
    mx, _ = at_max_overlap(inp)
    for t in inp["thr"]:
        cnt.update(threshold_cells(mx, t, "RPN"))
    for t, hi, lo, g in inp["pairs"]:
        cnt["FMA flips at %g" % t] += int(fma_flips(hi, lo, g, F32(t)).sum())
    return cnt


def threshold_cells(v, t, tag):
    t = F32(t)
    v = v[np.isfinite(v)]
    up, dn = np.nextafter(t, F32(2)), np.nextafter(t, F32(-2))
    return collections.Counter({"%s IoU = %g" % (tag, t): int((v == t).sum()),
                                "%s IoU just above %g" % (tag, t): int(((v > t) & (v <= t + 8 * (up - t))).sum()),
                                "%s IoU just below %g" % (tag, t): int(((v < t) & (v >= t - 8 * (t - dn))).sum())})


# ---------------------------------------------------------------------------------------- proposal targets
def pt_inputs(c):
    """-> dict(rl, rr [B,R,5], gl, gr, dim [B,K,5], kp [B,K,6], keys [B,R+K], words [B,S], cfg, bound)"""
    p = c.p
    rng = np.random.RandomState(p["seed"])
    cfg = dict(T.CFG, BATCH_SIZE=p.get("batch", 512), FG_FRACTION=p.get("frac", 0.25), KPTS_GRID=p.get("grid", 28))
    fam = p["fam"]
    bound = False
    if fam == "bound":                                  # 0.5 pairs on either side, IoU exactly 0, point boxes, zero rows
        H, W, K, n = p["H"], p["W"], p["K"], p["pairs"]
        box, _ = grid_boxes(K, H, W, rng)
        gl, gr, dim, kp = gt_tables(box[None], rng)
        rows_l, rows_r = [], []
        for side in (0, 1):                             # bisected on one side, identical to the box on the other
            idx = rng.randint(K, size=n // 2)
            own, other = (gl, gr) if side == 0 else (gr, gl)
            hi, lo = boundary_pairs(own[0, idx, :4], F32(0.5), rng)
            for j in range(idx.size):
                for a in (hi[j], lo[j]):
                    (rows_l if side == 0 else rows_r).append(a)
                    (rows_r if side == 0 else rows_l).append(other[0, idx[j], :4])
        for k in range(K):
            g = box[k]
            x2 = g[0] - F32(1)                          # iw = 0 exactly: IoU 0, in [BG_THRESH_LO, BG_THRESH_HI)
            rows_l.append(np.array([x2 - 5, g[1], x2, g[3]], F32))
            rows_r.append(gr[0, k, :4])
            rows_l.append(np.array([g[0] + 3, g[1] + 3, g[0] + 3, g[1] + 3], F32))   # a point box: IoU -1
            rows_r.append(gr[0, k, :4])
        rows_l += [np.zeros(4, F32)] * 40               # zero-padded rows
        rows_r += [np.zeros(4, F32)] * 40
        perm = rng.permutation(len(rows_l))
        rl = np.zeros((1, len(rows_l), 5), F32)
        rr = np.zeros_like(rl)
        rl[0, :, 1:] = np.array(rows_l, F32)[perm]
        rr[0, :, 1:] = np.array(rows_r, F32)[perm]
        bound = True
    elif fam == "none":                                 # no candidate at all: status 1
        B, R, K = 1, p["R"], p.get("K", 30)
        z = np.zeros((B, K, 5), F32)
        gl, gr, dim, kp = z, z.copy(), z.copy(), np.zeros((B, K, 6), F32)
        rl = np.zeros((B, R, 5), F32)
        rr = rl.copy()
    else:                                               # "synth"
        H, W, B, K = p.get("H", 160), p.get("W", 256), p.get("B", 2), p.get("K", 30)
        gl, gr, _gm, dim, kp, _nb = synth.synth_train_gt(B, K, H, W, p["seed"], n_boxes=p.get("n_boxes"))
        real = gl[:, :, 4] > 0
        if p.get("classes"):
            cls = rng.randint(1, 4, (B, K)).astype(F32) * real
            gl[:, :, 4] = cls
            gr[:, :, 4] = cls
        if p.get("dup"):                                # row 1 duplicates row 0's boxes with another class
            gl[:, 1, :4], gr[:, 1, :4] = gl[:, 0, :4], gr[:, 0, :4]
            gl[:, 1, 4] = gr[:, 1, 4] = np.where(gl[:, 0, 4] == 1, 2, 1) * real[:, 1]
        rl, rr = synth.synth_train_rois(gl, p["R"], H, W, p["seed"] + 100, near_gt=p.get("near", 0.34),
                                        jitter=p.get("jitter", 6.0))
        if p.get("zero_rows"):
            z = rng.uniform(size=rl.shape[:2]) < p["zero_rows"]
            rl[z, 1:] = 0
            rr[z, 1:] = 0
    B, R = rl.shape[:2]
    K = gl.shape[1]
    keys = make_keys(p.get("keys", "uniform"), (B, R + K), p["seed"] + 1)
    words = make_keys("uniform", (B, int(cfg["BATCH_SIZE"])), p["seed"] + 2)
    return dict(rl=rl, rr=rr, gl=gl, gr=gr, dim=dim, kp=kp, keys=keys, words=words, cfg=cfg, bound=bound)


def pt_oracle(inp):
    with rounded_log():
        return T.proposal_target_layer(inp["rl"], inp["rr"], inp["gl"], inp["gr"], inp["dim"], inp["kp"],
                                   T.KeySampler(inp["keys"], inp["words"]), inp["cfg"])


def pt_sets(inp):
    """per image: (foreground candidates, background candidates, max IoU left, max IoU right), as the oracle"""
    out = []
    for b in range(inp["rl"].shape[0]):
        m = []
        for r, g in ((inp["rl"], inp["gl"]), (inp["rr"], inp["gr"])):
            a = np.concatenate((r[b, :, 1:5], g[b, :, :4]))
            ov = T.bbox_overlaps_batch(a, g[b:b + 1])[0]
            m.append((ov.max(1), ov.argmax(1)))
        (ml, al), (mr, ar) = m
        cfg = inp["cfg"]
        fgt, hi, lo = F32(cfg["FG_THRESH"]), F32(cfg["BG_THRESH_HI"]), F32(cfg["BG_THRESH_LO"])
        fg = np.nonzero((ml >= fgt) & (mr >= fgt) & (al == ar))[0]
        bg = np.nonzero(((ml < hi) & (ml >= lo)) | ((mr < hi) & (mr >= lo)))[0]
        out.append((fg, bg, ml, mr))
    return out


def pt_cells(c, inp=None):
    inp = inp or pt_inputs(c)
    cnt = collections.Counter()
    S = int(inp["cfg"]["BATCH_SIZE"])
    n_fg_cap = int(np.round(inp["cfg"]["FG_FRACTION"] * S))
    for b, (fg, bg, ml, mr) in enumerate(pt_sets(inp)):
        cnt["proposals " + ("fg+bg" if fg.size and bg.size else "fg only" if fg.size else
                            "bg only" if bg.size else "none")] += 1
        if fg.size and bg.size:
            k = inp["keys"][b][fg]
            cnt["fg rank with equal keys"] += int(np.unique(k).size < k.size)
            cnt["fg list > 1024"] += int(fg.size > 1024)
            cnt["fg subsampled"] += int(fg.size > n_fg_cap)
        if inp["bound"]:
            v = np.concatenate((ml, mr))
            cnt.update(threshold_cells(v, 0.5, "proposal"))
            cnt["proposal IoU = 0"] += int((ml == 0).sum())
            cnt["proposal IoU = -1"] += int((ml == -1).sum())
    if inp["bound"]:
        t = F32(0.5)
        for r, gt in ((inp["rl"], inp["gl"]), (inp["rr"], inp["gr"])):
            a = r[0, :, 1:]
            g = gt[0, np.argmax(T.bbox_overlaps_batch(a, gt)[0], 1), :4]
            v, vf = iou32(a, g), iou32(a, g, fma=True)
            cnt["FMA flips at 0.5"] += int(((v >= t) != (vf >= t))[np.abs(v - t) < 1e-5].sum())
    return cnt


# -------------------------------------------------------------------------------------------------- losses
def rpn_inputs(c):
    """-> score [B,A,2], pred [B,A,6], labels [B,A], tl, tr [B,A,4], iw, ow [B,A] (float32 numpy), uncert or None"""
    p = c.p
    B, A = p["B"], p["A"]
    rs = np.random.RandomState(p["seed"])
    n = B * A
    lab = rs.choice(np.array([-1, 0, 1], F32), n, p=[0.5, 0.35, 0.15])
    lab[0] = 1                                           # at least one kept anchor with a box target
    score = (rs.randn(n, 2) * 2).astype(F32)
    pred = (rs.randn(n, 6) * 0.3).astype(F32)
    tl = (rs.randn(n, 4) * 0.3).astype(F32)
    tr = (rs.randn(n, 4) * 0.3).astype(F32)
    if p.get("extreme"):
        m = rs.uniform(size=n) < 0.05
        score[m] = rs.choice(np.array([-60, 60], F32), (int(m.sum()), 2))
        # smooth-L1 arguments at the branch point 1/sigma^2 = float32(1/9) and one ulp either side, both signs
        ninth = F32(1) / F32(9)
        vals = np.array([ninth, np.nextafter(ninth, F32(0)), np.nextafter(ninth, F32(1))], F32)
        rows = np.nonzero(lab == 1)[0][:max(1, min(64, n // 4))]
        for j, r in enumerate(rows):
            v = vals[j % 3] * (1 if (j // 3) % 2 == 0 else -1)
            tl[r] = 0
            tr[r] = 0
            pred[r] = v
    iw = (lab == 1).astype(F32)
    last = lab.reshape(B, A)[B - 1]
    w = F32(1.0 / max(int((last >= 0).sum()), 1))
    ow = np.where(lab >= 0, w, F32(0)).astype(F32)
    u = np.array([0.3, -0.2, 0.1, 0.0, 0.5, -0.4], F32) if p.get("uncert") else None
    return (score.reshape(B, A, 2), pred.reshape(B, A, 6), lab.reshape(B, A), tl.reshape(B, A, 4),
            tr.reshape(B, A, 4), iw.reshape(B, A), ow.reshape(B, A), u)


def rcnn_inputs(c):
    """-> preds (6 float32 arrays), tgt (dict of float32 / int64 arrays as proposal_target_layer's), uncert, G"""
    p = c.p
    R, C, Gd = p["R"], p["C"], p.get("G", 28)
    rs = np.random.RandomState(p["seed"])
    classes = np.arange(C) if not p.get("no_class1") else np.array([k for k in range(C) if k != 1])
    lab = classes[rs.randint(0, classes.size, R)]
    lab[:min(R, classes.size)] = classes[::-1][:min(R, classes.size)]    # every class present, a foreground one first
    pos = (lab > 0).astype(F32)
    tgt = dict(labels=lab.astype(F32), bbox_targets_left=(rs.randn(R, 4) * pos[:, None]).astype(F32),
               bbox_targets_right=(rs.randn(R, 4) * pos[:, None]).astype(F32),
               dim_orien_targets=(rs.randn(R, 5) * pos[:, None]).astype(F32),
               inside_w=np.repeat(pos[:, None], 4, 1).astype(F32), outside_w=np.repeat(pos[:, None], 4, 1).astype(F32))
    kt = np.stack((rs.randint(0, 4 * Gd, R), rs.randint(0, Gd, R), rs.randint(0, Gd, R)), 1).astype(np.int64)
    kw = ((lab == 1)[:, None] & (rs.uniform(size=(R, 3)) < 0.8)).astype(F32)
    if p.get("frac_w"):                                  # fractional weights, sum 0.5 per head: the sum(w) < 1 branch
        kw[:] = 0
        ones = np.nonzero(lab == 1)[0][:2]
        kw[ones] = 0.25
    tgt["kpts_targets"] = np.where(kw > 0, kt, 0)
    tgt["kpts_weight"] = kw
    preds = [(rs.randn(R, n) * s).astype(F32) for n, s in
             ((C, 2.0), (6 * C, 0.5), (5 * C, 0.5), (4 * Gd, 1.5), (Gd, 1.5), (Gd, 1.5))]
    u = np.array([0.3, -0.2, 0.1, 0.25, 0.5, -0.4], F32) if p.get("uncert") else None
    return preds, tgt, u, Gd


def clip_inputs(c):
    """-> list of float32 arrays, clip norm (float), exact norm (float64)"""
    p = c.p
    rs = np.random.RandomState(p["seed"])
    sizes = [int(s) for s in rs.randint(1, 32, p["n"])] if p.get("tiny") else \
        [int(s) for s in rs.choice([1, 7, 31, 300, 4099, 70000], p["n"])]
    if p.get("at_clip"):                                 # entries in {0, +-0.5}, n^2 nonzero: the norm is n / 2 exactly
        grads = [np.zeros(s, F32) for s in sizes]
        slots = [(t, i) for t, s in enumerate(sizes) for i in range(s)]
        m = int(math.isqrt(len(slots)))
        for j in rs.permutation(len(slots))[:m * m]:
            t, i = slots[j]
            grads[t][i] = rs.choice([-0.5, 0.5])
        norm = m / 2.0
        return grads, norm, norm
    grads = [(rs.randn(s) * p.get("scale", 1.0)).astype(F32) for s in sizes]
    norm = math.sqrt(sum(float((g.astype(np.float64) ** 2).sum()) for g in grads))
    return grads, p.get("clip", 10.0), norm


def rpn_trips(c):
    return int(math.ceil(c.p["B"] * c.p["A"] / float(512 * 256)))


# ------------------------------------------------------------------------------------------------- the cases
CASES = (
    # anchor targets: IoU threshold pairs (K <= 32 and K > 32 instances)
    [_c("at", "bound-K30", fam="bound", H=384, W=640, K=30, pairs=(600, 2000), seed=1),
     _c("at", "bound-K48", fam="bound", H=512, W=768, K=48, pairs=(600, 2000), seed=2)] +
    # argmax ties through both instances, K around the template switch
    [_c("at", "tie-K%d" % K, fam="tie", H=256, W=512, K=K, seed=10 + K) for K in (1, 31, 32, 33, 63, 64)] +
    [_c("at", "edge", fam="edge", H=160, W=256, seed=3, batch=HUGE_BATCH)] +
    # structured sampler keys through at_sample
    [_c("at", "keys-%s" % k, fam="pyr", H=160, W=256, B=2, batch=64, keys=k, seed=20 + i)
     for i, k in enumerate(KEY_PATTERNS)] +
    [_c("at", "keys-alpha2-b256", fam="pyr", H=224, W=400, B=1, batch=256, keys="alpha2", seed=40),
     _c("at", "keys-alpha4-b512", fam="pyr", H=224, W=400, B=1, batch=512, keys="alpha4", seed=41)] +
    # RPN_BATCHSIZE and num_fg
    [_c("at", "batch-%d" % b, fam="pyr", H=160, W=256, B=2, batch=b, seed=50 + b) for b in (1, 7, 256, 512)] +
    [_c("at", "batch-all", fam="pyr", H=160, W=256, B=2, batch=20000, seed=60),
     _c("at", "num-fg-0", fam="pyr", H=160, W=256, B=2, batch=256, frac=0.0, seed=61)] +
    # batch composition: the last image's counts set the outside weight
    [_c("at", "B1", fam="pyr", H=160, W=256, B=1, batch=256, seed=70),
     _c("at", "B2-last-empty", fam="pyr", H=160, W=256, B=2, n_boxes=[6, 0], batch=256, seed=71),
     _c("at", "B4-last-many", fam="pyr", H=160, W=256, B=4, n_boxes=[2, 3, 1, 30], batch=512, seed=72),
     _c("at", "B4-last-empty", fam="pyr", H=160, W=256, B=4, n_boxes=[5, 9, 3, 0], batch=64, keys="alpha2", seed=73)] +
    # proposal targets
    [_c("pt", "bound", fam="bound", H=384, W=640, K=30, pairs=300, batch=1024, frac=1.0, seed=80),
     _c("pt", "bound-K40", fam="bound", H=512, W=768, K=40, pairs=300, batch=1024, frac=1.0, seed=81),
     _c("pt", "none", fam="none", R=8, seed=82),
     _c("pt", "R4066", fam="synth", R=4096 - 30, near=0.3, seed=83),
     _c("pt", "fg-over-1024", fam="synth", B=1, R=3000, near=1.0, jitter=1.0, batch=1024, frac=1.0, seed=84),
     _c("pt", "fg-over-1024-sub", fam="synth", B=1, R=3000, near=1.0, jitter=1.0, batch=1024, frac=0.5,
        keys="alpha2", seed=85),
     _c("pt", "fg-only", fam="synth", B=1, R=200, near=1.0, jitter=0.5, batch=100, seed=86),
     _c("pt", "bg-only-last", fam="synth", B=2, R=300, n_boxes=[5, 0], seed=87),
     _c("pt", "zero-rows", fam="synth", R=2000, near=0.4, zero_rows=0.3, seed=88),
     _c("pt", "classes-dup-grid14", fam="synth", R=600, near=0.5, classes=True, dup=True, grid=14, seed=89)] +
    [_c("pt", "batch-%d-frac-%g" % (b, f), fam="synth", R=700, near=0.5, batch=b, frac=f, seed=90 + i)
     for i, (b, f) in enumerate(((1, 1.0), (100, 0.25), (512, 0.0), (512, 1.0), (1024, 0.25), (1024, 0.0)))] +
    [_c("pt", "keys-%s" % k, fam="synth", R=900, near=0.6, jitter=3.0, keys=k, seed=100 + i)
     for i, k in enumerate(KEY_PATTERNS)] +
    # RPN loss around the partial-sum grid (512 CTAs x 256 threads)
    [_c("rpn", "n%d-%s" % (B * A, "x" if ex else "p") + ("-u" if u else ""), B=B, A=A, extreme=ex, uncert=u, seed=110 + i)
     for i, (B, A, ex, u) in enumerate(((1, 1, False, True), (3, 85, True, False), (1, 131071, True, True),
                                        (2, 65536, False, False), (3, 43691, True, True), (2, 298476, True, False),
                                        (2, 298476, False, True)))] +
    # R-CNN loss: R around the 1024-thread CTA, C = 2..4
    [_c("rcnn", "R%d-C%d" % (R, C) + ("-u" if u else ""), R=R, C=C, uncert=u, seed=130 + i)
     for i, (R, C, u) in enumerate(((1, 2, True), (31, 3, False), (1023, 4, True), (1024, 2, False), (1025, 3, True),
                                    (2048, 4, False), (2048, 2, True)))] +
    [_c("rcnn", "no-class1-C3", R=700, C=3, no_class1=True, uncert=True, seed=140),
     _c("rcnn", "no-class1-C2", R=64, C=2, no_class1=True, seed=141),
     _c("rcnn", "frac-weights", R=300, C=3, frac_w=True, uncert=True, seed=142),
     _c("rcnn", "G14", R=513, C=2, G=14, seed=143)] +
    # clip_gradient chunks of 48 tensors
    [_c("clip", "n%d" % n + ("-tiny" if tiny else ""), n=n, tiny=tiny, scale=5.0, seed=150 + i)
     for i, (n, tiny) in enumerate(((47, False), (48, True), (49, False), (96, True), (97, False), (1, False)))] +
    [_c("clip", "n97-small", n=97, scale=1e-4, seed=160),
     _c("clip", "n49-at-clip", n=49, tiny=True, at_clip=True, seed=161),
     _c("clip", "n97-at-clip", n=97, at_clip=True, seed=162)]
)

assert len({c.id for c in CASES}) == len(CASES)


def of(kind):
    return [pytest.param(c, id=c.id) for c in CASES if c.kind == kind]


# --------------------------------------------------------------------------------------------- device calls
def cu(a, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.cuda()


def words(w):
    return cu(np.ascontiguousarray(w, np.uint32).view(np.int32))


def at_device(inp):
    got = G.anchor_targets(cu(inp["anchors"]), cu(inp["gl"]), cu(inp["gr"]), cu(inp["gm"]), (inp["H"], inp["W"]),
                           words(inp["keys"]), inp["cfg"])
    return [t.cpu().numpy() for t in got]


def pt_device(inp):
    got = G.proposal_targets(cu(inp["rl"]), cu(inp["rr"]), cu(inp["gl"]), cu(inp["gr"]), cu(inp["dim"]), cu(inp["kp"]),
                             words(inp["keys"]), words(inp["words"]), inp["cfg"])
    return {k: v.cpu().numpy() for k, v in got.items()}


def assert_ulps(got, ref, n, what):
    d = np.abs(got.astype(np.float64) - ref.astype(np.float64))
    lim = n * np.spacing(np.abs(ref)).astype(np.float64)
    bad = ~(d <= lim)
    assert not bad.any(), "%s: %d elements beyond %d ulp, e.g. got %r ref %r" % (
        what, int(bad.sum()), n, got[bad][:4], ref[bad][:4])


def assert_box_targets(got, ref, log_ulps, what):
    """dx, dy bit-exact (single _rn operations); dw, dh within log_ulps of the oracle's correctly rounded log (logf is
    within one ulp of the exact log; the proposal targets then divide by 0.2)"""
    np.testing.assert_array_equal(got[..., :2], ref[..., :2], err_msg=what)
    assert_ulps(got[..., 2:], ref[..., 2:], log_ulps, what)


# ------------------------------------------------------------------------------------------------- the tests
@pytest.mark.parametrize("c", of("at"))
def test_anchor_targets_edges(c):
    inp = at_inputs(c)
    ref = at_oracle(inp)
    lab, tl, tr, iw, ow = at_device(inp)
    np.testing.assert_array_equal(lab, ref[0], err_msg="labels")
    np.testing.assert_array_equal(iw, ref[3], err_msg="inside_w")
    np.testing.assert_array_equal(ow, ref[4], err_msg="outside_w")
    assert_box_targets(tl, ref[1], 1, "targets_left")
    assert_box_targets(tr, ref[2], 1, "targets_right")
    mx, inside = at_max_overlap(inp)
    for t in inp["thr"]:                                  # both sides of every threshold occur, and exactly t
        cells = threshold_cells(mx, t, "RPN")
        assert all(v > 0 for v in cells.values()), cells
    if c.p["fam"] == "edge":
        assert inside.sum() < inside.size and (lab[:, ~inside] == -1).all() and (lab[:, inside] == 1).any()
    n_keep = (lab >= 0).sum(1)
    assert (n_keep <= c.p.get("batch", 512)).all() or c.p["fam"] in ("bound",)
    print("%s: A=%d K=%d fg=%s bg=%s" % (c.id, lab.shape[1], inp["gl"].shape[1], (lab == 1).sum(1).tolist(),
                                         (lab == 0).sum(1).tolist()))


@pytest.mark.parametrize("c", of("pt"))
def test_proposal_targets_edges(c):
    inp = pt_inputs(c)
    got = pt_device(inp)
    B, S = got["labels"].shape
    if c.p["fam"] == "none":
        assert got["status"].tolist() == [1] * B
        assert (got["keep_inds"] == -1).all()
        for n in ("labels", "bbox_targets_left", "bbox_targets_right", "dim_orien_targets", "kpts_targets",
                  "kpts_weight", "inside_w", "outside_w"):
            assert not got[n].any(), n
        assert not got["rois_left"][..., 1:].any() and not got["rois_right"][..., 1:].any()
        with pytest.raises(ValueError):
            pt_oracle(inp)
        return
    ref = pt_oracle(inp)
    assert got["status"].tolist() == [0] * B
    np.testing.assert_array_equal(got["keep_inds"], ref["keep_inds"], err_msg="keep_inds")
    for n in ("rois_left", "rois_right", "labels", "dim_orien_targets", "kpts_weight", "inside_w", "outside_w"):
        np.testing.assert_array_equal(got[n], ref[n], err_msg=n)
    np.testing.assert_array_equal(got["kpts_targets"].astype(np.int64), ref["kpts_targets"], err_msg="kpts_targets")
    assert_box_targets(got["bbox_targets_left"], ref["bbox_targets_left"], 2, "bbox_targets_left")
    assert_box_targets(got["bbox_targets_right"], ref["bbox_targets_right"], 2, "bbox_targets_right")
    # keypoint targets only for class 1
    assert not got["kpts_weight"][got["labels"] != 1].any() and not got["kpts_targets"][got["labels"] != 1].any()
    if inp["bound"]:
        ml = np.concatenate([s[2] for s in pt_sets(inp)] + [s[3] for s in pt_sets(inp)])
        cells = threshold_cells(ml, 0.5, "proposal")
        assert all(v > 0 for v in cells.values()), cells
        assert (ml == 0).any() and (ml == -1).any()
    print("%s: fg kept %s of %s" % (c.id, (got["labels"] > 0).sum(1).tolist(), [s[0].size for s in pt_sets(inp)]))


def _rpn_ref(score, pred, lab, tl, tr, iw, ow, u):
    s = torch.from_numpy(score).double().requires_grad_()
    p = torch.from_numpy(pred).double().requires_grad_()
    t = [torch.from_numpy(x).double() for x in (lab, tl, tr, iw, ow)]
    lc, lb = T.rpn_losses(s, p, *t)
    e = torch.exp(-torch.from_numpy(u).double()) if u is not None else torch.ones(2, dtype=torch.float64)
    (lc * e[0] + lb * e[1]).backward()
    return np.array([float(lc.detach()), float(lb.detach())]), s.grad.numpy(), p.grad.numpy()


def _rpn_dev(score, pred, lab, tl, tr, iw, ow, u):
    losses, d_cls, d_box = G.rpn_loss(cu(score), cu(pred), cu(lab), cu(tl), cu(tr), cu(iw), cu(ow),
                                      uncert=cu(u) if u is not None else None)
    return losses.cpu().numpy(), d_cls.cpu().numpy(), d_box.cpu().numpy()


def rel_err(got, ref):
    return float(np.abs(got.astype(np.float64) - ref).max() / max(np.abs(ref).max(), 1e-300))


@pytest.mark.parametrize("c", of("rpn"))
def test_rpn_loss_edges(c):
    args = rpn_inputs(c)
    rl, rs_, rp = _rpn_ref(*args)
    gl, gs, gp = _rpn_dev(*args)
    el = np.abs(gl - rl) / np.abs(rl)
    es, ep = rel_err(gs, rs_), rel_err(gp, rp)
    print("%s: %d grid-stride trip(s); loss rel err %.2e %.2e (bar 2e-6), d_cls %.2e, d_box %.2e of max (bar 1e-6)"
          % (c.id, rpn_trips(c), el[0], el[1], es, ep))
    assert (el <= 2e-6).all(), (gl, rl)
    assert es <= 1e-6 and ep <= 1e-6
    assert np.abs(rp).max() > 0 and np.abs(rs_).max() > 0


def _rcnn_ref(preds, tgt, u):
    ps = [torch.from_numpy(p).double().requires_grad_() for p in preds]
    tt = {k: torch.from_numpy(v).double() if v.dtype == F32 else torch.from_numpy(v) for k, v in tgt.items()}
    ls = T.rcnn_losses(*ps, tt)
    e = torch.exp(-torch.from_numpy(u).double()) if u is not None else torch.ones(6, dtype=torch.float64)
    sum(l * e[2 + i] for i, l in enumerate(ls)).backward()
    return np.array([float(l.detach()) for l in ls]), [p.grad.numpy() for p in ps]


def _rcnn_dev(preds, tgt, u, Gd):
    tg = {k: cu(v, torch.int32) if v.dtype == np.int64 else cu(v) for k, v in tgt.items()}
    losses, grads = G.rcnn_loss(*[cu(p) for p in preds], tg, uncert=cu(u) if u is not None else None, kpts_grid=Gd)
    return losses.cpu().numpy(), [g.cpu().numpy() for g in grads]


@pytest.mark.parametrize("c", of("rcnn"))
def test_rcnn_loss_edges(c):
    preds, tgt, u, Gd = rcnn_inputs(c)
    rl, rg = _rcnn_ref(preds, tgt, u)
    gl, gg = _rcnn_dev(preds, tgt, u, Gd)
    el = np.abs(gl - rl) / np.maximum(np.abs(rl), 1e-300)
    errs = {n: rel_err(g, r) for n, g, r in zip(("cls", "bbox", "dim", "kpts", "left", "right"), gg, rg)}
    print("%s: loss rel err %s (bar 3e-6); gradients of max %s (bar 2e-6)"
          % (c.id, " ".join("%.1e" % e for e in el), " ".join("%s %.1e" % kv for kv in errs.items())))
    assert ((el <= 3e-6) | ((rl == 0) & (gl == 0))).all(), (gl, rl)
    for (n, e), r in zip(errs.items(), rg):
        if np.abs(r).max() == 0:
            continue
        assert e <= 2e-6, n
    if c.p.get("no_class1"):                              # sum(w) = 0: no keypoint loss, zero keypoint gradients
        assert gl[3] == 0 and not gg[3].any() and not gg[4].any() and not gg[5].any()
    assert np.abs(rg[0]).max() > 0 and np.abs(rg[2]).max() > 0 and (np.abs(rg[1]).max() > 0) == (tgt["labels"] > 0).any()
    # the class-selected gather: only the labelled class of each row has a box / dimension gradient
    lab = tgt["labels"].astype(np.int64)
    C = c.p["C"]
    other = np.ones((lab.size, C), bool)
    other[np.arange(lab.size), lab] = False
    assert not gg[1].reshape(-1, C, 6)[other].any() and not gg[2].reshape(-1, C, 5)[other].any()


@pytest.mark.parametrize("c", of("clip"))
def test_clip_gradient_edges(c):
    grads, clip, norm = clip_inputs(c)
    dev = [cu(g) for g in grads]
    out = G.clip_gradient(dev, clip).cpu().numpy()
    f = clip / max(norm, clip)
    print("%s: %d tensors, %d launch chunk(s), norm %.6g rel err %.1e, factor %.9g"
          % (c.id, len(grads), -(-len(grads) // 48), norm, abs(out[0] - norm) / norm, out[1]))
    assert abs(out[0] - norm) <= 2e-6 * norm and abs(out[1] - f) <= 2e-6
    if c.p.get("at_clip"):                                # the norm is exactly the clip value: nothing is scaled
        assert out[0] == F32(clip) and out[1] == 1.0
    for a, b in zip(dev, grads):
        np.testing.assert_array_equal(a.cpu().numpy(), b * F32(out[1]))


def test_clip_gradient_just_above_the_norm():
    """a clip value one ulp below an exact norm scales every tensor by clip / norm"""
    c = next(x for x in CASES if x.id == "clip-n49-at-clip")
    grads, norm, _ = clip_inputs(c)
    clip = float(np.nextafter(F32(norm), F32(0)))
    dev = [cu(g) for g in grads]
    out = G.clip_gradient(dev, clip).cpu().numpy()
    assert out[0] == F32(norm) and out[1] == F32(F32(clip) / F32(norm)) and out[1] < 1
    for a, b in zip(dev, grads):
        np.testing.assert_array_equal(a.cpu().numpy(), b * F32(out[1]))


def test_determinism_of_the_four_entry_points():
    """two calls on the same inputs give identical bits (fixed-order reductions, no atomics in any result)"""
    inp = at_inputs(next(c for c in CASES if c.id == "at-keys-alpha2"))
    a, b = at_device(inp), at_device(inp)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    inp = pt_inputs(next(c for c in CASES if c.id == "pt-keys-equal"))
    a, b = pt_device(inp), pt_device(inp)
    assert all(np.array_equal(a[k], b[k]) for k in a)
    args = rpn_inputs(next(c for c in CASES if c.id.startswith("rpn-n596952-x")))
    a, b = _rpn_dev(*args), _rpn_dev(*args)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    preds, tgt, u, Gd = rcnn_inputs(next(c for c in CASES if c.id == "rcnn-R2048-C4"))
    (la, ga), (lb, gb) = _rcnn_dev(preds, tgt, u, Gd), _rcnn_dev(preds, tgt, u, Gd)
    assert np.array_equal(la, lb) and all(np.array_equal(x, y) for x, y in zip(ga, gb))


@pytest.mark.parametrize("H,W", [(375, 1242), (161, 257), (333, 999)])
def test_device_anchor_table_at_odd_sizes(H, W):
    """generate_anchors.py:112-173 on the device, bit-equal to the fp64 numpy table cast to fp32, at sizes whose
    feature maps are rounded up"""
    assert H % 64 and W % 64
    fs = feat_shapes(H, W)
    got = G.generate_anchors(fs, "cuda").cpu().numpy()
    np.testing.assert_array_equal(got, O.anchors_all_pyramids(fs).astype(F32))
