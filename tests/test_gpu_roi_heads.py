"""GPU: the pyramid RoIAlign (roi_align.cu, roi_align_pyramid_nhwc) and the head tails (misc.cu, sb_kpts_tail and
sb_box_tail) element by element against float64.

Pyramid RoIAlign.  A test-side mirror restates the kernel's arithmetic: fp32 x*scale, rw = (float)((double)(ew-sw)
+ 1.), bin = (float)(rw/(L-1)); the lattice coordinate fma(p, bin, start) is rebuilt exactly (p*bin is exact in
float64, start is added with TwoSum and the error term breaks an fp32 midpoint tie); hr = h - hstart is exact, the
four bilinear weights are exact products in float64, and each lattice value L64 = sum f*w is taken in float64 from the
fp32 features.  The kernel forms the same sum with its own float64 roundings (with or without fma), at most 4 of
2^-53 * S each, S = sum |f*w|; the mirror's differs by as much again.  So:

  mode 0   bit-exact with ((L00+L01)+(L10+L11))*0.25 in fp32 of L32 = fl32(L64), except where an L64 lies within
           2^-50 * S of an fp32 midpoint (a "tie": either rounding is right).  Every element, tie or not, obeys
           |out - avg64| <= 2^-22 A, A = 1/4 sum over the 4 lattice points of S: each L32 is off by 2^-24 S, the
           three fp32 adds by 2^-24 of their partial sums, in all 3 * 2^-24 A < 2^-22 A.
  mode 1   torch.equal(mode1, round_tf32_(mode0))       (cvt.rna.tf32: ties away, like ops.round_tf32_)
  mode 2   torch.equal(mode2, mode0.half())             (__floats2half2_rn: ties to even, like .half())

Level routing is round(logf(sqrt(h*w)/224) + 4) clamped to P2..P5, with h, w, h*w, sqrt and /224 in fp32 (all
correctly rounded) and logf within 1 ulp of the correctly rounded log (CUDA's definition of its ulp error).  The
mirror takes the float64 log rounded to fp32 and its two fp32 neighbours; when they round to two levels the RoI is
ambiguous and must match the mirror at one of them (reported).

Every output sits in a buffer filled with a NaN sentinel: guard rows before and after the R RoIs, a channel slice
of wider rows (out_ld = C+8, out_coff = 4) or the 512-wide concat of two calls.  Every logical element must be
written and every other byte left alone.  A repeated call is bit-identical and permuting the RoIs permutes the output.

Head tails, per element against float64 (u = 2^-24):
  kpts logits  |d| <= 2^-18 A, A = sum_c |w_jc| sum_h |x_hc| + G |b_j|: a column sum runs through at most G = 30
               fp32 adds, the dot product through C/256 fmas (8 per lane on the fp16 path), 5 shuffle levels, 8
               per-warp partials and the bias, < 64 roundings of at most u A each.
  box linears  |d| <= (ceil(K/256) + 16) u A, A = sum_k |f_k w_k| + |b|: a chain of K/256 fmas, 5 shuffles, 8
               partials, the bias.
  softmax      against a float64 softmax of the kernel's own logits z (max m):
               |dp_e| <= p_e u (|z_e - m| + sum_k p_k |z_k - m| + 20) + 2^-126: z - m in fp32 costs u |z - m|
               through exp; expf 2 ulp, the sum <= 9 adds, the division 1 ulp; 2^-126 covers underflow.  The box
               tail's class logits are not an output, so there its reference is the float64 logits and each p_e
               also carries 2 p_e (d_e + sum_k p_k d_k) for the logits' own bounds d.
"""
import collections
import ctypes
import math
import zlib

import numpy as np
import pytest
import torch

from oracle import ops as O
from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import ops as G

F32, F64 = np.float32, np.float64
SENT32 = 0x7FA5A5A5            # NaN bit patterns the kernels never produce
SENT16 = 0x7E5A
TIE = 2.0 ** -50
ERR = 2.0 ** -22
PYRAMIDS = {"bench": ((150, 497), (75, 249), (38, 125), (19, 63)), "small": ((40, 64), (20, 32), (10, 16), (5, 8))}
IMAGE = {"bench": (600.0, 1987.0), "small": (160.0, 256.0)}
BOUNDARIES = (49.98, 135.86, 369.31)      # sqrt(h*w) at log(sqrt(h*w)/224) + 4 = 2.5, 3.5, 4.5
B = 2                                     # images per side: left = feats[:B], right = feats[B:]


# ------------------------------------------------------------------------------------------ host mirror (numpy)
def level_sets(rois):
    """-> (lo, hi, raw): the levels (0..3 = P2..P5) logf may route each RoI to, and the unclamped round of the
    correctly rounded log + 4"""
    r = np.asarray(rois, F32)
    h = (r[:, 4] - r[:, 2]) + F32(1)
    w = (r[:, 3] - r[:, 1]) + F32(1)
    q = np.sqrt(h * w) / F32(224)
    with np.errstate(divide="ignore"):
        l64 = np.log(q.astype(F64))
    c = l64.astype(F32)                       # correctly rounded; CUDA states logf's error in ulps from this value
    cand = np.stack([np.nextafter(c, F32(-np.inf)), c, np.nextafter(c, F32(np.inf))], 1)
    lv = np.clip(np.rint(cand + F32(4)), 2, 5) - 2
    return lv.min(1).astype(np.int64), lv.max(1).astype(np.int64), np.rint(c + F32(4))


def roi_geometry(rois, scale, L):
    r = np.asarray(rois, F32)
    s = F32(scale)
    sw, sh, ew, eh = r[:, 1] * s, r[:, 2] * s, r[:, 3] * s, r[:, 4] * s
    rw = np.maximum(((ew - sw).astype(F64) + 1.0).astype(F32), F32(0))
    rh = np.maximum(((eh - sh).astype(F64) + 1.0).astype(F32), F32(0))
    return sw, sh, (rw.astype(F64) / (L - 1.0)).astype(F32), (rh.astype(F64) / (L - 1.0)).astype(F32)


def axis_taps(start, bin_, L, size):
    """lattice coordinates fma(p, bin, start) along one axis -> (x [R,L] fp32, x0, xr float64, zero)"""
    a = np.arange(L, dtype=F64)[None, :] * bin_.astype(F64)[:, None]          # exact: 24 bits times p < 2^5
    b = np.broadcast_to(start.astype(F64)[:, None], a.shape)
    s = a + b
    bb = s - a
    err = (a - (s - bb)) + (b - bb)                                          # TwoSum: a + b == s + err
    c = s.astype(F32)
    dn, up = np.nextafter(c, F32(-np.inf)), np.nextafter(c, F32(np.inf))
    c64 = c.astype(F64)
    x = np.where((s == (c64 + up.astype(F64)) / 2) & (err > 0), up,
                 np.where((s == (c64 + dn.astype(F64)) / 2) & (err < 0), dn, c))
    x0 = np.minimum(np.floor(x), F32(size - 2))
    zero = (x < 0) | (x >= size)
    return x, x0.astype(np.int64), (x - x0).astype(F64), zero


def level_scale(H, im_h):
    return F32(H / float(im_h))


def mirror_check(got, feat, rois, scale, P, chunk_elems=1 << 22):
    """got [R,P,P,C] fp32 output of mode 0 for `rois` pooled from `feat` [N,H,W,C] at `scale`.
    -> (ok [R] bool: bit-exact off ties and within the bound, ratio [R]: worst |got - avg64| / (2^-22 A),
        ties: lattice ties, tie_outs: outputs that depend on one, exact_outs)"""
    N, H, W, C = feat.shape
    L = P + 1
    R = rois.shape[0]
    dev = feat.device
    sw, sh, bw, bh = roi_geometry(rois, scale, L)
    _, h0, hr, hz = axis_taps(sh, bh, L, H)
    _, w0, wr, wz = axis_taps(sw, bw, L, W)
    bidx = rois[:, 0].astype(np.int64)
    zero = hz[:, :, None] | wz[:, None, :]
    off = np.where(zero, 0, (bidx[:, None, None] * H + h0[:, :, None]) * W + w0[:, None, :])
    hr3, wr3 = hr[:, :, None], wr[:, None, :]
    wts = ((1. - hr3) * (1. - wr3), (1. - hr3) * wr3, hr3 * (1. - wr3), hr3 * wr3)
    flat = feat.reshape(-1, C)
    ok = np.zeros(R, bool)
    ratio = np.zeros(R)
    ties = tie_outs = exact_outs = 0
    step = max(1, chunk_elems // (L * L * C))
    for r0 in range(0, R, step):
        sl = slice(r0, min(R, r0 + step))
        o = torch.from_numpy(off[sl]).to(dev)
        z = torch.from_numpy(zero[sl]).to(dev)[..., None]
        L64 = torch.zeros(o.shape + (C,), dtype=torch.float64, device=dev)
        S = torch.zeros_like(L64)
        for dofs, wt in zip((0, 1, W, W + 1), wts):
            f = flat[o + dofs].double()
            wt = torch.from_numpy(np.ascontiguousarray(wt[sl])).to(dev)[..., None]
            L64 = L64 + f * wt
            S = S + f.abs() * wt.abs()
        L64 = torch.where(z, torch.zeros_like(L64), L64)
        S = torch.where(z, torch.zeros_like(S), S)
        L32 = L64.float()
        c64 = L32.double()
        mup = (c64 + torch.nextafter(L32, torch.full_like(L32, math.inf)).double()) / 2
        mdn = (c64 + torch.nextafter(L32, torch.full_like(L32, -math.inf)).double()) / 2
        tie = torch.minimum((L64 - mup).abs(), (L64 - mdn).abs()) <= TIE * S

        def avg(t):
            return ((t[:, :-1, :-1] + t[:, :-1, 1:]) + (t[:, 1:, :-1] + t[:, 1:, 1:])) * 0.25

        out32, avg64, A = avg(L32), avg(L64), avg(S)
        tie_o = tie[:, :-1, :-1] | tie[:, :-1, 1:] | tie[:, 1:, :-1] | tie[:, 1:, 1:]
        g = got[sl]
        same = g == out32
        d = (g.double() - avg64).abs()
        rt = torch.where(d == 0, torch.zeros_like(d), d / (ERR * A))
        rmax = rt.flatten(1).max(1).values
        ok[sl] = ((same | tie_o).flatten(1).all(1) & (rmax <= 1)).cpu().numpy()
        ratio[sl] = rmax.cpu().numpy()
        ties += int(tie.sum())
        tie_outs += int(tie_o.sum())
        exact_outs += int(same.sum())
    return ok, ratio, ties, tie_outs, exact_outs


def pooled_vs_mirror(got, feats, rois, im_h, P):
    """the kernel output of one call against the mirror at the level(s) each RoI may take.
    -> dict(ratio, ties, tie_outs, ambiguous [(roi, lo, hi, took)])"""
    lo, hi, _ = level_sets(rois)
    R = rois.shape[0]
    ok_at, ratio_at = np.zeros((4, R), bool), np.full((4, R), np.inf)
    st = dict(ties=0, tie_outs=0)
    for l in range(4):
        sel = np.nonzero((lo == l) | (hi == l))[0]
        if sel.size == 0:
            continue
        ok, ratio, t, to, ex = mirror_check(got[torch.from_numpy(sel).to(got.device)], feats[l], rois[sel],
                                            level_scale(feats[l].shape[1], im_h), P)
        ok_at[l, sel], ratio_at[l, sel] = ok, ratio
        st["ties"] += t
        st["tie_outs"] += to
    amb, worst = [], 0.0
    for i in range(R):
        took = [l for l in {lo[i], hi[i]} if ok_at[l, i]]
        assert took, ("RoI %d %s matches the mirror at no level (candidates P%d..P%d; worst err/bound %s)"
                      % (i, rois[i].tolist(), lo[i] + 2, hi[i] + 2, ratio_at[:, i].tolist()))
        worst = max(worst, min(ratio_at[l, i] for l in took))
        if lo[i] != hi[i]:
            amb.append((i, lo[i] + 2, hi[i] + 2, "/".join("P%d" % (l + 2) for l in sorted(took))))
    st.update(ratio=worst, ambiguous=amb)
    return st


# ------------------------------------------------------------------------------------------------- RoI families
def boundary_sweep(k, n_ulps=3000):
    """x2 over +-n_ulps fp32 ulps around the x2 at which sqrt(h*w) crosses BOUNDARIES[k]"""
    h = (40.0, 100.0, 300.0)[k]
    y1, x1 = F32(10.25), F32(5.5)
    w = BOUNDARIES[k] ** 2 / h
    mid = F32(x1 + w - 1.0)
    x2 = (mid.view(np.int32) + np.arange(-n_ulps, n_ulps + 1, dtype=np.int32)).view(F32)
    r = np.zeros((x2.size, 5), F32)
    r[:, 0] = np.arange(x2.size) % 2
    r[:, 1], r[:, 2], r[:, 3], r[:, 4] = x1, y1, x2, F32(y1 + h - 1.0)
    return r


def mixed_rois(R, pyr, seed):
    """every family in one batch of R RoIs (shuffled), batch indices 0 and 1"""
    im_h, im_w = IMAGE[pyr]
    rs = np.random.RandomState(seed)
    m = max(1, R // 10)

    def boxes(x1, y1, x2, y2):
        return np.stack([x1, y1, x2, y2], 1)

    def loguni(n, lo=4.0, hi=None):
        side = np.exp(rs.uniform(np.log(lo), np.log(hi or 1.3 * max(im_h, im_w)), n))
        asp = np.exp(rs.uniform(-1, 1, n))
        return side * np.sqrt(asp), side / np.sqrt(asp)

    fam = []
    n = max(1, R - 8 * m)
    w, h = loguni(n)                                                          # every level
    x1, y1 = rs.uniform(-0.05 * im_w, im_w - w / 2), rs.uniform(-0.05 * im_h, im_h - h / 2)
    fam.append(boxes(x1, y1, x1 + w, y1 + h))
    w, h = rs.uniform(0, 5, m), rs.uniform(0, 5, m)                           # tiny: below P2, clamped
    x1, y1 = rs.uniform(0, im_w - 6, m), rs.uniform(0, im_h - 6, m)
    fam.append(boxes(x1, y1, x1 + w, y1 + h))
    big = np.array([[0, 0, im_w - 1, im_h - 1], [-50, -30, im_w + 80, im_h + 40]])   # full box, above P5, clamped
    fam.append(big[rs.randint(0, 2, m)])
    fam.append(np.zeros((m, 4)))                                              # zero-padded rows
    w, h = loguni(m)                                                          # ending at im - 1: [H-1, H) taps
    fam.append(boxes(im_w - 1 - w, im_h - 1 - h, np.full(m, im_w - 1), np.full(m, im_h - 1)))
    w, h = loguni(m)                                                          # past the right / bottom edges
    x1, y1 = rs.uniform(0.6 * im_w, im_w, m), rs.uniform(0.6 * im_h, im_h, m)
    fam.append(boxes(x1, y1, x1 + w, y1 + h))
    w, h = loguni(m)                                                          # negative starts
    x1 = np.where(rs.rand(m) < 0.5, -rs.uniform(0, 4, m), -rs.uniform(0, 60, m))
    y1 = np.where(rs.rand(m) < 0.5, -rs.uniform(0, 4, m), -rs.uniform(0, 60, m))
    fam.append(boxes(x1, y1, x1 + w, y1 + h))
    x1, y1 = rs.uniform(0, im_w - 2, m), rs.uniform(0, im_h - 2, m)            # one pixel thin
    hh = np.exp(rs.uniform(0, np.log(im_h), m))
    fam.append(boxes(x1, y1, x1, y1 + hh))
    ln = rs.uniform(0.5, 1.0, m) * im_w                                       # very elongated
    x1, y1 = rs.uniform(-10, im_w - ln, m), rs.uniform(0, im_h - 3, m)
    fam.append(boxes(x1, y1, x1 + ln, y1 + rs.uniform(0, 2, m)))
    b = np.concatenate(fam)[:R]
    r = np.concatenate([rs.randint(0, 2, (b.shape[0], 1)), b], 1).astype(F32)
    r[:, 3] = np.maximum(r[:, 3], r[:, 1])                                    # x2 >= x1, y2 >= y1 (proposals)
    r[:, 4] = np.maximum(r[:, 4], r[:, 2])
    return r[rs.permutation(r.shape[0])]


# ------------------------------------------------------------------------------------------------------- cases
PCase = collections.namedtuple("PCase", "id pyr C P R layout")
PYR_CASES = [PCase("%s-c%d-p%d-r%d-%s" % c, *c) for c in (
    ("bench", 64, 7, 600, "dense"),
    ("bench", 64, 14, 300, "slice"),
    ("bench", 4, 1, 600, "slice"),
    ("bench", 12, 2, 600, "dense"),
    ("small", 12, 9, 200, "slice"),
    ("small", 4, 15, 300, "dense"),
    ("small", 64, 8, 300, "slice"),
    ("small", 12, 14, 600, "dense"),
    ("bench", 512, 14, 40, "dense"),       # 66 KB of shared memory: the attribute path
    ("small", 512, 15, 16, "slice"),
    ("small", 256, 7, 100, "slice"),
    ("bench", 256, 9, 64, "slice"),
    ("bench", 4, 2, 18003, "sweep"),       # the three level-boundary sweeps
    ("bench", 256, 7, 600, "concat"),      # the engine's box-head calls: left at out_coff 0, right at 256
    ("bench", 256, 14, 600, "kpts"),       # the engine's keypoint call: dense, left features
)]


def case_calls(c):
    """-> [(side, rois, out_coff)] of the calls that fill one output; side 0 = left features, 1 = right"""
    seed = zlib.crc32(c.id.encode())
    if c.layout == "sweep":
        rois = np.concatenate([boundary_sweep(k) for k in range(3)])
        return [(1, rois, 4)]
    if c.layout == "concat":
        return [(0, mixed_rois(c.R, c.pyr, seed), 0), (1, mixed_rois(c.R, c.pyr, seed + 1), c.C)]
    side = 0 if c.layout == "kpts" else 1
    return [(side, mixed_rois(c.R, c.pyr, seed), 4 if c.layout == "slice" else 0)]


def out_ld(c):
    return {"concat": 2 * c.C, "slice": c.C + 8, "sweep": c.C + 8}.get(c.layout, c.C)


def layout_name(c):
    return {"sweep": "slice", "kpts": "dense"}.get(c.layout, c.layout)


def row_blocks(P):
    if P <= 8:
        return "single"
    rb = (P + 1) // 2
    return "%d+%d" % (rb, P - rb)


# ------------------------------------------------------------------------------------------------ CPU census
def census():
    cnt = collections.Counter()
    for c in PYR_CASES:
        shapes = PYRAMIDS[c.pyr]
        im_h = IMAGE[c.pyr][0]
        cnt["rows " + row_blocks(c.P)] += 1
        for mode in (0, 1, 2):
            cnt["mode %d x %s" % (mode, layout_name(c))] += 1
        for _, rois, _ in case_calls(c):
            lo, hi, raw = level_sets(rois)
            cnt["batch index 1"] += int((rois[:, 0] == 1).sum())
            one = lo == hi
            for l in range(4):
                cnt["P%d routed" % (l + 2)] += int((one & (lo == l) & (raw == l + 2)).sum())
                cnt["P%d clamped" % (l + 2)] += int((one & (lo == l) & (raw != l + 2)).sum())
            for l in range(3):
                cnt["ambiguous P%d|P%d" % (l + 2, l + 3)] += int(((lo == l) & (hi == l + 1)).sum())
            for l in range(4):
                sel = (lo == l) | (hi == l)
                if not sel.any():
                    continue
                H, W = shapes[l]
                sw, sh, bw, bh = roi_geometry(rois[sel], level_scale(H, im_h), c.P + 1)
                hx = axis_taps(sh, bh, c.P + 1, H)[0]
                wx = axis_taps(sw, bw, c.P + 1, W)[0]
                hin, win = ((hx >= 0) & (hx < H)).any(1), ((wx >= 0) & (wx < W)).any(1)
                cnt["zero taps top"] += int((hx < 0).any(1).sum())
                cnt["zero taps bottom"] += int((hx >= H).any(1).sum())
                cnt["zero taps left"] += int((wx < 0).any(1).sum())
                cnt["zero taps right"] += int((wx >= W).any(1).sum())
                cnt["band [H-1,H) taps"] += int((((hx >= H - 1) & (hx < H)).any(1) & win).sum())
                cnt["band [W-1,W) taps"] += int((((wx >= W - 1) & (wx < W)).any(1) & hin).sum())
    return cnt


REQUIRED = (["P%d routed" % l for l in range(2, 6)] + ["P2 clamped", "P5 clamped"] +
            ["ambiguous P%d|P%d" % (l, l + 1) for l in range(2, 5)] +
            ["zero taps " + s for s in ("top", "bottom", "left", "right")] +
            ["band [H-1,H) taps", "band [W-1,W) taps", "batch index 1"] +
            ["rows " + s for s in ("single", "5+4", "7+7", "8+7")] +
            ["mode %d x %s" % (m, lay) for m in (0, 1, 2) for lay in ("dense", "slice", "concat")])


def test_pyramid_case_matrix_census():
    """CPU: the case matrix reaches every branch of the kernel (P3 and P4 cannot be reached by clamping)"""
    cnt = census()
    print("\npyramid RoIAlign census:")
    for k in sorted(cnt):
        print("  %-24s %d" % (k, cnt[k]))
    missing = [k for k in REQUIRED if not cnt[k]]
    assert not missing, missing
    assert {c.C // 4 for c in PYR_CASES} >= {1, 3, 16, 64, 128}
    assert {c.P for c in PYR_CASES} >= {1, 2, 7, 8, 9, 14, 15}
    assert all(r.shape[0] == c.R for c in PYR_CASES for _, r, _ in case_calls(c))
    assert max(c.R for c in PYR_CASES if c.layout != "sweep") == 600


def oracle_cases(seed, pyr, C, R):
    rs = np.random.RandomState(seed)
    feats = [rs.randn(2, C, h, w).astype(F32) for h, w in PYRAMIDS[pyr]]
    return feats, mixed_rois(R, pyr, seed)


@pytest.mark.parametrize("P", [1, 7, 9])
def test_mirror_vs_oracle(P):
    """CPU: the mirror and the oracle's PyramidRoI_Feat agree within the bound (they group the bilinear products
    differently, so they may differ by an ulp on rare elements) at the oracle's level"""
    feats, rois = oracle_cases(P, "small", 12, 300)
    ora = torch.from_numpy(O.pyramid_roi_feat(feats, rois, IMAGE["small"][0], P).transpose(0, 2, 3, 1).copy())
    lv = O.roi_levels(rois) - 2
    fd = [torch.from_numpy(f.transpose(0, 2, 3, 1).copy()) for f in feats]
    exact = 0
    for l in range(4):
        sel = np.nonzero(lv == l)[0]
        if sel.size:
            ok, ratio, _, _, ex = mirror_check(ora[torch.from_numpy(sel)], fd[l], rois[sel],
                                               level_scale(fd[l].shape[1], IMAGE["small"][0]), P)
            assert (ratio <= 1).all(), ratio.max()
            exact += ex
    print("\nmirror vs oracle, P=%d: %d of %d elements bit-identical" % (P, exact, ora.numel()))
    assert exact >= 0.99 * ora.numel()


# ------------------------------------------------------------------------------------------------- GPU: pyramid

def sentinel_buffer(n, half, dev):
    buf = torch.empty(n, dtype=torch.int16 if half else torch.int32, device=dev)
    buf.fill_(SENT16 if half else SENT32)
    return buf


def run_pyramid(c, feats, calls, mode, perm=None):
    """fill a sentinel buffer with the case's calls; -> (buffer, written mask, [got per call])"""
    P, C, ld = c.P, c.C, out_ld(c)
    R = calls[0][1].shape[0]
    lead = trail = P * P * ld + 3 * ld
    n = lead + R * P * P * ld + trail
    buf = sentinel_buffer(n, mode == 2, "cuda")
    view = buf.view(torch.float16 if mode == 2 else torch.float32)[lead:lead + R * P * P * ld].view(R, P, P, ld)
    written = torch.zeros(n, dtype=torch.bool, device="cuda")
    wview = written[lead:lead + R * P * P * ld].view(R, P, P, ld)
    im_h = IMAGE[c.pyr][0]
    for side, rois, coff in calls:
        r = rois if perm is None else rois[perm]
        G.roi_align_pyramid_nhwc(feats[side], im_h, torch.from_numpy(r).cuda(), P, out=view, out_coff=coff,
                                 round_tf32=mode == 1, half=mode == 2)
        wview[..., coff:coff + C] = True
    torch.cuda.synchronize()
    return buf, written, [view[..., coff:coff + C] for _, _, coff in calls]


def check_sentinel(buf, written, got, what):
    sent = SENT16 if buf.dtype == torch.int16 else SENT32
    assert bool((buf[~written] == sent).all()), "%s: bytes outside the output were written" % what
    for g in got:
        assert bool(torch.isfinite(g).all()), "%s: elements not written" % what


def make_feats(c):
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(c.id.encode()) & 0x7FFFFFFF)
    full = [torch.randn(2 * B, h, w, c.C, generator=g, device="cuda") for h, w in PYRAMIDS[c.pyr]]
    return [f[:B] for f in full], [f[B:] for f in full]


@pytest.mark.gpu
@pytest.mark.parametrize("c", PYR_CASES, ids=[c.id for c in PYR_CASES])
def test_roi_align_pyramid_vs_mirror(c, capsys):
    left, right = make_feats(c)
    feats = (left, right)
    calls = case_calls(c)
    b0, w0, got0 = run_pyramid(c, feats, calls, 0)
    check_sentinel(b0, w0, got0, "mode 0")
    line = "%-32s rows %-6s" % (c.id, row_blocks(c.P))
    worst, ties, tie_outs, amb = 0.0, 0, 0, []
    for (side, rois, coff), g in zip(calls, got0):
        st = pooled_vs_mirror(g, feats[side], rois, IMAGE[c.pyr][0], c.P)
        worst = max(worst, st["ratio"])
        ties += st["ties"]
        tie_outs += st["tie_outs"]
        amb += st["ambiguous"]
    # modes 1 and 2: mode 0 rounded, in the same layout
    b1, w1, got1 = run_pyramid(c, feats, calls, 1)
    check_sentinel(b1, w1, got1, "mode 1")
    b2, w2, got2 = run_pyramid(c, feats, calls, 2)
    check_sentinel(b2, w2, got2, "mode 2")
    for g0, g1, g2 in zip(got0, got1, got2):
        assert torch.equal(g1, G.round_tf32_(g0.clone())), "mode 1 is not mode 0 rounded to TF32"
        assert torch.equal(g2, g0.half()), "mode 2 is not mode 0 converted to fp16"
    # invariants: a repeated call, and a permutation of the RoIs
    assert torch.equal(run_pyramid(c, feats, calls, 0)[0], b0), "a repeated call differs"
    perm = np.random.RandomState(c.R).permutation(calls[0][1].shape[0])
    _, _, gotp = run_pyramid(c, feats, calls, 0, perm=perm)
    pt = torch.from_numpy(perm).cuda()
    for g0, gp in zip(got0, gotp):
        assert torch.equal(gp, g0[pt]), "permuting the RoIs does not permute the output"
    line += " err/bound %.3f  ties %d (outputs %d)  ambiguous %d" % (worst, ties, tie_outs, len(amb))
    with capsys.disabled():
        print(line)
        for i, l0, l1, took in amb:
            print("    ambiguous RoI %5d  P%d|P%d  took %s" % (i, l0, l1, took))


@pytest.mark.gpu
def test_roi_align_pyramid_no_rois_no_launch():
    left, _ = make_feats(PCase("r0", "small", 12, 7, 0, "dense"))
    buf = sentinel_buffer(64, False, "cuda")
    n0 = G.launch_count()
    out = buf.view(torch.float32)[:0].view(0, 7, 7, 12)
    G.roi_align_pyramid_nhwc(left, 160.0, torch.zeros(0, 5, device="cuda"), 7, out=out)
    torch.cuda.synchronize()
    assert G.launch_count() == n0
    assert bool((buf == SENT32).all())


@pytest.mark.gpu
@pytest.mark.parametrize("pooled", [7, 14])
def test_roi_align_pyramid_nhwc_vs_oracle(pooled):
    rs = np.random.RandomState(11)
    shapes = [(150, 497), (75, 249), (38, 125), (19, 63)]
    C = 64
    feats = [rs.randn(1, C, h, w).astype(np.float32) for h, w in shapes]
    R = 120
    x1 = rs.rand(R) * 1500
    y1 = rs.rand(R) * 400
    side = np.exp(rs.uniform(np.log(8), np.log(900), R))
    rois = np.stack([np.zeros(R), x1, y1, np.minimum(x1 + side * rs.uniform(0.5, 2, R), 1986),
                     np.minimum(y1 + side, 599)], 1).astype(np.float32)
    rois[0] = 0
    ref = O.pyramid_roi_feat(feats, rois, 600.0, pooled)             # R,C,p,p
    assert len(set(O.roi_levels(rois).tolist())) == 4
    fd = [torch.from_numpy(f.transpose(0, 2, 3, 1).copy()).cuda() for f in feats]
    out = G.roi_align_pyramid_nhwc(fd, 600.0, torch.from_numpy(rois).cuda(), pooled).cpu().numpy().transpose(0, 3, 1, 2)
    np.testing.assert_allclose(out, ref, rtol=1e-5, atol=1e-5)
    # the mirror and the oracle within the bound, at the oracle's level
    ora = torch.from_numpy(ref.transpose(0, 2, 3, 1).copy()).cuda()
    lv = O.roi_levels(rois) - 2
    for l in range(4):
        sel = np.nonzero(lv == l)[0]
        ok, ratio, _, _, _ = mirror_check(ora[torch.from_numpy(sel).cuda()], fd[l], rois[sel],
                                          level_scale(shapes[l][0], 600.0), pooled)
        assert (ratio <= 1).all(), ratio.max()


# --------------------------------------------------------------------------------------------- GPU: head tails
U = 2.0 ** -24
GUARD = 67


def guarded(shape, dev="cuda"):
    n = int(np.prod(shape))
    buf = sentinel_buffer(n + 2 * GUARD, False, dev)
    return buf, buf.view(torch.float32)[GUARD:GUARD + n].view(shape)


def check_guarded(buf, view, what):
    assert bool((buf[:GUARD] == SENT32).all()) and bool((buf[GUARD + view.numel():] == SENT32).all()), \
        "%s: bytes outside the output were written" % what
    assert bool(torch.isfinite(view).all()), "%s: elements not written" % what


def vp(t):
    return ctypes.c_void_p(t.data_ptr())


def softmax_check(p, z, what, extra=None):
    """p: kernel probabilities [R, n]; z: float64 logits [R, n] the softmax is taken of"""
    m = z.max(1, keepdim=True).values
    e = (z - m).exp()
    ref = e / e.sum(1, keepdim=True)
    dz = (z - m).abs()
    bound = ref * U * (dz + (ref * dz).sum(1, keepdim=True) + 20) + 2.0 ** -126
    if extra is not None:
        bound = bound + 2 * ref * (extra + (ref * extra).sum(1, keepdim=True))
    r = ((p.double() - ref).abs() / bound).max().item()
    assert r <= 1, (what, r)
    return r


KPTS_PATHS = (("f16", 256), ("f16", 128), ("f32", 256), ("f32", 260))    # kpts_colsum16, <__half>, <float>
FAMILIES = ("relu", "signed", "logits200", "equal")
KCase = collections.namedtuple("KCase", "id dtype C G R family")
KPTS_CASES = []
for _pi, (_dt, _c) in enumerate(KPTS_PATHS):
    for _gi, _g in enumerate((1, 7, 9, 28, 30)):
        for _ri, _r in enumerate((1, 300)):
            _f = FAMILIES[(_pi + _gi + 2 * _ri) % 4]
            KPTS_CASES.append(KCase("%s-c%d-g%d-r%d-%s" % (_dt, _c, _g, _r, _f), _dt, _c, _g, _r, _f))


def test_head_tail_case_lists_cover_every_family():
    """CPU: each kpts path sees every input family, and so does the box tail"""
    for dt, cc in KPTS_PATHS:
        assert {k.family for k in KPTS_CASES if (k.dtype, k.C) == (dt, cc)} == set(FAMILIES)
    assert {b.family for b in BOX_CASES} == set(FAMILIES)


@pytest.mark.gpu
@pytest.mark.parametrize("k", KPTS_CASES, ids=[k.id for k in KPTS_CASES])
def test_kpts_tail_vs_float64(k, capsys):
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(zlib.crc32(k.id.encode()) & 0x7FFFFFFF)
    R, Gd, C = k.R, k.G, k.C
    x = torch.randn(R, Gd, Gd, C, generator=g, device=dev)
    if k.family == "relu":
        x = x.clamp_min(0)
    x = x.half() if k.dtype == "f16" else x
    x64 = x.double()
    w = torch.randn(6, C, generator=g, device=dev) / math.sqrt(C * Gd)
    b = torch.randn(6, generator=g, device=dev)
    colsum, acol = x64.sum(1), x64.abs().sum(1)                   # [R, col, C]
    if k.family == "logits200":
        raw = torch.einsum("rgc,jc->rjg", colsum, w.double())
        w = (w * (200.0 / raw.abs().max().item())).float()
    elif k.family == "equal":
        w = torch.zeros_like(w)
        b = torch.full_like(b, 0.37)
    w64, b64 = w.double(), b.double()
    ref = torch.einsum("rgc,jc->rjg", colsum, w64) + Gd * b64[None, :, None]
    A = torch.einsum("rgc,jc->rjg", acol, w64.abs()) + Gd * b64.abs()[None, :, None]
    (bkp, kp), (blp, lp), (brp, rp), (bka, ka) = (guarded((R, 4 * Gd)), guarded((R, Gd)), guarded((R, Gd)),
                                                  guarded((R, 6, Gd)))
    n0 = G.launch_count()
    rc = L.load().sb_kpts_tail(vp(x), 1 if k.dtype == "f16" else 0, R, Gd, C, vp(w), vp(b), vp(kp), vp(lp), vp(rp),
                               vp(ka), L.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0 and G.launch_count() == n0 + 2
    for buf, v, what in ((bkp, kp, "kpts_prob"), (blp, lp, "left_prob"), (brp, rp, "right_prob"),
                         (bka, ka, "pred_all")):
        check_guarded(buf, v, what)
    r_lin = ((ka.double() - ref).abs() / (2.0 ** -18 * A).clamp_min(1e-300)).max().item()
    assert r_lin <= 1, ("logits", r_lin)
    z = ka.double()
    r_sm = max(softmax_check(kp, z[:, :4].reshape(R, 4 * Gd), "kpts_prob"),
               softmax_check(lp, z[:, 4], "left_prob"), softmax_check(rp, z[:, 5], "right_prob"))
    with capsys.disabled():
        print("%-34s logits err/bound %.3f  softmax err/bound %.3f" % (k.id, r_lin, r_sm))


BCase = collections.namedtuple("BCase", "id nc K R family")
BOX_CASES = []
for _ni, _nc in enumerate((1, 2, 3, 4)):
    for _ki, _k in enumerate((1, 255, 256, 257, 2048, 4099)):
        for _ri, _r in enumerate((1, 300)):
            _f = FAMILIES[(_ni + _ki + 2 * _ri) % 4]
            BOX_CASES.append(BCase("nc%d-k%d-r%d-%s" % (_nc, _k, _r, _f), _nc, _k, _r, _f))


@pytest.mark.gpu
@pytest.mark.parametrize("bc", BOX_CASES, ids=[b.id for b in BOX_CASES])
def test_box_tail_vs_float64(bc, capsys):
    dev = "cuda"
    g = torch.Generator(device=dev).manual_seed(zlib.crc32(bc.id.encode()) & 0x7FFFFFFF)
    R, K, nc = bc.R, bc.K, bc.nc
    f = torch.randn(R, K, generator=g, device=dev)
    if bc.family in ("relu", "equal"):
        f = f.clamp_min(0)
    ws = [torch.randn(n * nc, K, generator=g, device=dev) / math.sqrt(K) for n in (1, 6, 5)]
    bs = [torch.randn(n * nc, generator=g, device=dev) for n in (1, 6, 5)]
    if bc.family == "logits200":
        ws[0] = (ws[0] * (200.0 / (f.double() @ ws[0].double().t()).abs().max().item())).float()
    elif bc.family == "equal":
        ws[0] = torch.zeros_like(ws[0])
        bs[0] = torch.full_like(bs[0], -1.25)
    f64 = f.double()
    refs = [f64 @ w.double().t() + b.double() for w, b in zip(ws, bs)]
    As = [f64.abs() @ w.double().abs().t() + b.double().abs() for w, b in zip(ws, bs)]
    n_chain = -(-K // 256) + 16
    (bcp, cp), (bbx, bx), (bdm, dm) = guarded((R, nc)), guarded((R, 6 * nc)), guarded((R, 5 * nc))
    rc = L.load().sb_box_tail(vp(f), R, K, nc, vp(ws[0]), vp(bs[0]), vp(ws[1]), vp(bs[1]), vp(ws[2]), vp(bs[2]),
                              vp(cp), vp(bx), vp(dm), L.stream_ptr())
    torch.cuda.synchronize()
    assert rc == 0
    for buf, v, what in ((bcp, cp, "cls_prob"), (bbx, bx, "bbox_pred"), (bdm, dm, "dim_orien")):
        check_guarded(buf, v, what)
    r_lin = 0.0
    for got, ref, A, what in ((bx, refs[1], As[1], "bbox_pred"), (dm, refs[2], As[2], "dim_orien")):
        r = ((got.double() - ref).abs() / (n_chain * U * A).clamp_min(1e-300)).max().item()
        assert r <= 1, (what, r)
        r_lin = max(r_lin, r)
    r_sm = softmax_check(cp, refs[0], "cls_prob", extra=n_chain * U * As[0])
    with capsys.disabled():
        print("%-28s linear err/bound %.3f  softmax err/bound %.3f" % (bc.id, r_lin, r_sm))
