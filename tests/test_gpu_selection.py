"""GPU: the selection kernels -- the proposal layer (csrc/proposal.cu: radix select, ordered compaction, rank sort,
decode, two-sided NMS), the NMS (csrc/nms.cu: bitmask + device greedy scan) and the per-class NMS (class_nms_kernel of
csrc/misc.cu) -- bit for bit against the CPU oracle on identical inputs: keep lists, counts, every mask word, RoI rows
including the zero padding and the batch column.

Their decisions are discrete: a wrong one changes which RoIs exist rather than drifting a value.  The inputs are built
on the CPU so that each decision is taken at its edge, and each case prints what it exercised:

  IoU             box pairs bisected on the fp32 lattice so that the stepwise-fp32 devIoU straddles `> t` (t = 0.3,
                  0.5, 0.7): many exactly on float32(t), their one-ulp neighbours, and at least ten per threshold inside
                  the +-1e-4 band where sb_iou_gt falls back to the division; touching, identical, point and inverted
                  boxes, coordinates near 1e38, and thresholds 0, 1, -0.5, 1.5 and NaN.
  greedy scan     chains (box i overlaps only i +- 1) across lanes 31/32, 63/64 and chunk ends, one box of chunk 0
                  suppressing the last chunk, suppressed suppressors, identical / disjoint boxes, dense clusters, up to
                  n = 16384.
  selection cut   the K-th and (K+1)-th score keys first differing in the top 11 bits, in bits 10-20, in bits 0-9, or
                  equal (a tie decided by anchor index over many 2048-anchor blocks); constant, two-valued, monotone
                  scores; 0, 1, subnormals, +-inf, +-NaN and -0.0, ranked as torch.sort(descending=True) ranks them.
  sizes           pre_nms_top_n 0, 1, A-1, A, A+1; K from 1 to 16384; A just above 2 097 152 (the multi-pass block
                  scan) and A = 2048 * 4096; 1 and 8 levels, 1 and 4 ratios with other scales and strides.
  two sides       left / right deltas whose keep lists differ, post_nms_top_n reached mid-chunk, exactly at a chunk
                  end, never (zero rows), and 1; batches of 2 and 3 images with their own im_info; one workspace
                  reused across decreasing and increasing A.
  per-class NMS   R = 0 ... 512 (all eight mask words), 2-4 classes and every class, scores at score_thresh and one
                  ulp above, equal, NaN, inf and +-0 scores, chains and long-range suppression over the eight words."""
import numpy as np
import pytest
import torch

from oracle import ops as O
from stereo_rcnn_b200 import ops as G

pytestmark = pytest.mark.gpu

F32 = np.float32
THRESHOLDS = (0.3, 0.5, 0.7)
SMALL = [[40, 64], [20, 32], [10, 16], [5, 8], [3, 4]]                  # A = 3 * 3412 = 10 236


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def bits(a):
    return np.ascontiguousarray(a, F32).view(np.uint32)


def assert_bits(got, ref, what):
    got, ref = np.asarray(got), np.asarray(ref)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    bad = np.nonzero(bits(got).reshape(-1) != bits(ref).reshape(-1))[0]
    assert bad.size == 0, "%s: %d elements differ, first at flat %d: %r vs %r" % (
        what, bad.size, bad[0], got.reshape(-1)[bad[0]], ref.reshape(-1)[bad[0]])


# ---------------------------------------------------------------------------------------------------------- IoU
def iou32(a, b):
    """devIoU of nms_cuda_kernel.cu:31-39 row by row (broadcasting), stepwise fp32 in its order"""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    one = F32(1)
    with np.errstate(all="ignore"):
        w = np.maximum(np.minimum(a[..., 2], b[..., 2]) - np.maximum(a[..., 0], b[..., 0]) + one, F32(0))
        h = np.maximum(np.minimum(a[..., 3], b[..., 3]) - np.maximum(a[..., 1], b[..., 1]) + one, F32(0))
        inter = w * h
        sa = (a[..., 2] - a[..., 0] + one) * (a[..., 3] - a[..., 1] + one)
        sb = (b[..., 2] - b[..., 0] + one) * (b[..., 3] - b[..., 1] + one)
        return inter, sa + sb - inter, inter / (sa + sb - inter)


def in_band(a, b, t):
    """pairs inside sb_iou_gt's +-1e-4 band: decided by the division, not by the multiplications"""
    inter, uni, _ = iou32(a, b)
    with np.errstate(all="ignore"):
        tu = F32(t) * uni
        return (uni > 0) & np.isfinite(tu) & ~(inter > tu * F32(1.0001)) & ~(inter < tu * F32(0.9999))


def boundary_pairs(t, n, rng, scale):
    """boxes a inside boxes g whose x2 is bisected on the fp32 lattice: -> g, hi, lo with hi the first x2 whose IoU with
    g is > t and lo one ulp below it (IoU <= t, often exactly float32(t))"""
    g = np.zeros((n, 4), F32)
    g[:, :2] = rng.uniform(0, 4, (n, 2)) * scale
    g[:, 2:] = g[:, :2] + (rng.uniform(0.5, 1.5, (n, 2)) * scale).astype(F32)
    a = g.copy()
    a[:, 1] = g[:, 1] + F32(rng.uniform(0, 0.05, n)) * (g[:, 3] - g[:, 1])
    lo, hi = a[:, 0].copy().view(np.int32).astype(np.int64), g[:, 2].copy().view(np.int32).astype(np.int64)

    def at(xi):
        b = a.copy()
        b[:, 2] = xi.astype(np.int32).view(F32)
        return b
    ok = (iou32(at(lo), g)[2] <= F32(t)) & (iou32(at(hi), g)[2] > F32(t))
    g, a, lo, hi = g[ok], a[ok], lo[ok], hi[ok]
    while True:
        m = hi - lo > 1
        if not m.any():
            break
        mid = lo + (hi - lo) // 2
        gt = iou32(at(mid), g)[2] > F32(t)
        hi, lo = np.where(m & gt, mid, hi), np.where(m & ~gt, mid, lo)
    return g, at(hi), at(lo)


def boundary_boxes(t, rng, per_scale=120):
    """[n,4] boxes in triplets (g, hi, lo) and the CPU census of the pairs around t"""
    parts = [boundary_pairs(t, per_scale, rng, s) for s in (3.0, 11.0, 40.0, 150.0, 700.0)]
    g, hi, lo = (np.concatenate(p) for p in zip(*parts))
    tt = F32(t)
    on = int((iou32(lo, g)[2] == tt).sum())
    band = int(in_band(lo, g, t).sum() + in_band(hi, g, t).sum())
    assert (iou32(hi, g)[2] > tt).all() and (iou32(lo, g)[2] <= tt).all()
    boxes = np.stack([g, hi, lo], 1).reshape(-1, 4)
    return boxes, dict(pairs=g.shape[0], on_t=on, in_band=band)


def special_boxes():
    """touching, identical, point, inverted and huge boxes, each next to a partner"""
    b = [[10, 10, 50, 50], [51, 10, 90, 50],                         # touching: right - left + 1 == 0
         [10, 51, 50, 90], [10, 10, 50, 50], [10, 10, 50, 50],         # touching below; identical
         [5, 5, 5, 5], [5, 5, 5, 5], [5, 5, 6, 6],                     # point boxes (area 1) and their neighbour
         [30, 30, 20, 20], [20, 20, 30, 30], [30, 30, 28, 40],         # inverted: negative widths / areas
         [40, 40, 38.5, 38.5], [38.5, 38.5, 40, 40],                   # area (-0.5)^2 > 0 from two negative sides
         [0, 0, -1, 10], [0, 0, -1, -1], [-1, -1, 0, 0],               # zero-area boxes (width exactly 0)
         [-1e38, -1e38, 1e38, 1e38], [-1e38, 0, 1e38, 10], [0, -1e38, 10, 1e38],   # areas / unions overflow
         [-3e38, -3e38, 3e38, 3e38], [1e38, 1e38, 3e38, 3e38], [-1e38, -1e38, -2e37, -2e37],
         [0, 0, 1e38, 1e38], [0, 0, 1e38, 1e38], [1e37, 1e37, 2e37, 2e37]]
    return np.asarray(b, F32)


def with_scores(boxes):
    n = boxes.shape[0]
    return np.concatenate([boxes, np.linspace(1, 0, n, dtype=F32)[:, None]], 1).astype(F32)


def check_mask(dets, t, what):
    m = G.nms_mask(cu(dets), t).cpu().numpy().view(np.uint64)
    ref = O.nms_mask(dets, t)
    n, cb = ref.shape
    upper = np.arange(cb)[None, :] >= (np.arange(n) // 64)[:, None]
    np.testing.assert_array_equal(np.where(upper, m, 0), np.where(upper, ref, 0), err_msg=what)
    assert not m[~upper].any(), what
    return int(np.unpackbits(np.ascontiguousarray(m[upper]).view(np.uint8)).sum())


def check_nms(dets, t, what, pin=False):
    keep = G.nms(cu(dets), t).cpu().numpy().reshape(-1)
    ref = O.nms(dets, t)
    np.testing.assert_array_equal(keep, ref, err_msg=what)
    if pin:
        np.testing.assert_array_equal(ref, greedy(dets, t), err_msg=what + " (oracle against the plain greedy)")
    return ref


def greedy(dets, t):
    """the host scan of nms_cuda_kernel.cu, as plainly as it can be written"""
    dead, keep = np.zeros(dets.shape[0], bool), []
    for i in range(dets.shape[0]):
        if not dead[i]:
            keep.append(i)
            dead[i + 1:] |= iou32(dets[i, :4], dets[i + 1:, :4])[2] > F32(t)
    return np.asarray(keep, np.int32)


@pytest.mark.parametrize("t", THRESHOLDS)
def test_iou_boundary_pairs(t):
    """every pairwise decision of the bisected pairs through sb_nms_mask, the keep lists through sb_nms, and the
    per-class NMS (512-row slices, thresh t)"""
    rng = np.random.RandomState(int(t * 10))
    boxes, census = boundary_boxes(t, rng)
    assert census["in_band"] >= 10 and census["on_t"] >= 10, census
    dets = with_scores(boxes)
    ones = check_mask(dets, t, "mask t=%g" % t)
    keep = check_nms(dets, t, "nms t=%g" % t)
    # pair by pair: (g, lo) never suppresses, (g, hi) always does -- through the NMS alone and the per-class NMS
    for name, pb in (("hi", np.concatenate([boxes[0::3], boxes[1::3]], 1).reshape(-1, 4)),
                     ("lo", np.concatenate([boxes[0::3], boxes[2::3]], 1).reshape(-1, 4))):
        for s in range(0, pb.shape[0], 512):
            sl = pb[s:s + 512]
            R = sl.shape[0]
            scores = np.stack([np.zeros(R, F32), np.linspace(0.9, 0.1, R, dtype=F32)], 1)
            bx = np.concatenate([np.zeros((R, 4), F32), sl], 1)
            got = class_nms(scores, bx, 1, 0.05, t)
            ref = O.per_class_nms(scores, bx, 1, 0.05, t)
            np.testing.assert_array_equal(got, ref, err_msg="class_nms %s t=%g" % (name, t))
        check_mask(with_scores(pb), t, "pairs %s t=%g" % (name, t))
        check_nms(with_scores(pb), t, "pairs %s t=%g" % (name, t))
    print("IoU t=%g: %d pairs, %d exactly on float32(t), %d compares inside the 1e-4 band, %d mask bits, %d kept"
          % (t, census["pairs"], census["on_t"], census["in_band"], ones, keep.size))


@pytest.mark.parametrize("t", [0.0, 1.0, -0.5, 1.5, float("nan"), 0.3, 0.5, 0.7, -0.0])
def test_iou_special_boxes_and_thresholds(t):
    rng = np.random.RandomState(3)
    sp = special_boxes()
    boxes, _ = boundary_boxes(0.5, rng, per_scale=20)
    mix = np.concatenate([sp, boxes[:150], sp[::-1], rng.permutation(sp)])
    dets = with_scores(mix)
    ones = check_mask(dets, t, "special t=%r" % t)
    keep = check_nms(dets, t, "special t=%r" % t, pin=True)
    R = min(mix.shape[0], 512)
    scores = np.stack([np.zeros(R, F32), np.linspace(0.9, 0.1, R, dtype=F32)], 1)
    bx = np.concatenate([np.zeros((R, 4), F32), mix[:R]], 1)
    np.testing.assert_array_equal(class_nms(scores, bx, 1, 0.05, t), O.per_class_nms(scores, bx, 1, 0.05, t))
    with np.errstate(all="ignore"):
        _, uni, iou = iou32(mix[:, None], mix[None, :])
    print("special boxes t=%r: n=%d, %d unions <= 0, %d non-finite IoUs, %d mask bits, %d kept"
          % (t, mix.shape[0], int((uni <= 0).sum()), int((~np.isfinite(iou)).sum()), ones, keep.size))


# ---------------------------------------------------------------------------------------------- greedy scan
def row_boxes(n, x0, step, w=99.0, h=99.0):
    """n boxes along x: with step 50 and width 99, box i overlaps only i - 1 and i + 1 (IoU 1/3 and 0)"""
    x = x0 + step * np.arange(n, dtype=np.float64)
    return np.stack([x, np.zeros(n), x + w, np.full(n, h)], 1).astype(F32)


def layout(n, chains=(), groups=()):
    """n isolated boxes (IoU 0 with each other), then chains: index lists whose consecutive members overlap (IoU 1/3),
    groups: index lists of identical boxes"""
    b = np.zeros((n, 4), F32)
    b[:, 0] = (np.arange(n) % 128) * 1000.0
    b[:, 1] = (np.arange(n) // 128) * 1000.0 + 100000.0
    b[:, 2], b[:, 3] = b[:, 0] + 99, b[:, 1] + 99
    for c, idx in enumerate(chains):
        idx = np.asarray(idx)
        b[idx] = row_boxes(idx.size, 0.0, 50.0) + np.array([0, 200.0 * c, 0, 200.0 * c], F32) - 1e5
    for c, idx in enumerate(groups):
        b[np.asarray(idx)] = np.array([c * 500.0, -3e5, c * 500.0 + 99, -3e5 + 99], F32)
    return with_scores(b)


def scan_cases():
    out = []
    for n in (1, 63, 64, 65, 127, 128, 129, 300, 4097):
        out.append(("chain", n, layout(n, [np.arange(n)])))
    for n in (64, 129, 4097, 16383, 16384):
        # links across lanes 31/32, 63/64, chunk ends and the last chunk, all in one scan
        ch = [np.arange(28, 37), np.arange(60, 70), np.arange(n - 70, n)] + \
             [np.arange(s - 3, s + 3) for s in range(192, n - 80, 640)]
        ch = [c[(c >= 0) & (c < n)] for c in ch]
        ch = [c for c in ch if c.size > 1]
        ch = [c for i, c in enumerate(ch) if not any(np.intersect1d(c, d).size for d in ch[:i])]
        out.append(("chains at lane and chunk edges", n, layout(n, ch)))
    for n in (129, 4097, 16384):
        # long range: box 0 (chunk 0) and a box of every 7th chunk suppress boxes of the last chunks (the gather of
        # chunks < c); suppressed suppressors: 1 is removed by 0 and must not remove its partner in the last chunk
        # and pairs from chunk j to chunk j + 1 (the carry) and to chunk j + 2 (the gather of chunk c - 1)
        last = n - 1
        g = [[0, last, last - 1, last - 64 if n > 128 else last - 2]] + \
            [[c * 64 + 5, last - 10 - k] for k, c in enumerate(range(7, (n - 1) // 64 - 1, 7)) if k < 40] + \
            [[64 * j + 40, 64 * (j + 1) + 3] for j in range(0, (n - 1) // 64 - 1, 3)] + \
            [[64 * j + 20, 64 * (j + 2) + 30] for j in range(0, (n - 1) // 64 - 2, 5)]
        used, groups = {0, 1, last - 5}, []
        for grp in g:
            if not used.intersection(grp[1:] if grp[0] == 0 else grp):
                used.update(grp)
                groups.append(grp)
        d = layout(n, groups=groups)
        # 1 overlaps 0 (removed), 1 overlaps last-5 but 0 does not: last-5 is kept
        d[1, :4] = d[0, :4] + np.array([50, 0, 50, 0], F32)
        d[last - 5, :4] = d[1, :4] + np.array([50, 0, 50, 0], F32)
        out.append(("long range + suppressed suppressor", n, d))
    for n in (65, 4097, 16384):
        d = layout(n)
        d[:, :4] = np.array([3, 4, 103, 104], F32)
        out.append(("all identical", n, d))
        out.append(("all disjoint", n, layout(n)))
    rng = np.random.RandomState(0)
    for n in (300, 4097, 16384):
        c = rng.randint(0, max(n // 40, 1), n)
        ctr = rng.uniform(0, 3000, (n // 40 + 1, 2))[c] + rng.normal(0, 6, (n, 2))
        wh = rng.uniform(30, 60, (n, 2))
        b = np.concatenate([ctr - wh / 2, ctr + wh / 2], 1).astype(F32)
        out.append(("dense clusters", n, with_scores(b)))
    return out


SCAN = scan_cases()


@pytest.mark.parametrize("i", range(len(SCAN)), ids=["%s-%d" % (c[0].replace(" ", "_"), c[1]) for c in SCAN])
def test_greedy_scan_structured(i):
    name, n, dets = SCAN[i]
    for t in (0.3, 0.7):
        keep = check_nms(dets, t, "%s n=%d t=%g" % (name, n, t), pin=n <= 300)
        if name == "chain" and t == 0.3:
            np.testing.assert_array_equal(keep, np.arange(0, n, 2))
        if name == "all identical":
            np.testing.assert_array_equal(keep, [0])
        if name == "all disjoint":
            assert keep.size == n
        if name.startswith("long range") and t == 0.3:
            assert n - 5 - 1 in keep and n - 1 not in keep and n - 2 not in keep and 1 not in keep
        print("%s n=%d t=%g: %d chunks, %d kept" % (name, n, t, (n + 63) // 64, keep.size))


# ------------------------------------------------------------------------------------------- proposal layer
def score_key(x):
    """sb_score_key of common.cuh on the CPU"""
    x = np.asarray(x, F32)
    b = x.view(np.uint32).copy()
    b[b == 0x80000000] = 0
    k = np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)
    k[np.isnan(x)] = 0xFF800001
    return k


def key_float(k):
    k = np.asarray(k, np.uint32)
    return np.where(k & np.uint32(0x80000000), k & np.uint32(0x7FFFFFFF), ~k).astype(np.uint32).view(F32)


def n_anchors(shapes, ratios=3):
    return ratios * sum(h * w for h, w in shapes)


def run_proposals(prob, bbox, info, shapes, pre, post, thr, scales=None, ratios=None, strides=None, what=""):
    cfg = dict(G.CFG, TEST=dict(RPN_PRE_NMS_TOP_N=pre, RPN_POST_NMS_TOP_N=post, RPN_NMS_THRESH=thr))
    pc = G.make_proposal_cfg("TEST", shapes, ratios=ratios, scales=scales, strides=strides, cfg=cfg)
    rl, rr = G.proposal_layer(cu(prob), cu(bbox), cu(info), "TEST", shapes, pc=pc)
    ol, orr, dbg = O.proposal_layer(prob, bbox, info, "TEST", shapes, return_debug=True, pre_nms_top_n=pre,
                                    post_nms_top_n=post, nms_thresh=thr, scales=scales, ratios=ratios, strides=strides)
    assert_bits(rl.cpu().numpy(), ol, what + " rois_left")
    assert_bits(rr.cpu().numpy(), orr, what + " rois_right")
    for b, d in enumerate(dbg):
        K = d["order"].size
        print("%s image %d: A=%d K=%d, kept left %d right %d both %d, rows %d of %d"
              % (what, b, prob.shape[1], K, d["keep_l"].size, d["keep_r"].size, np.intersect1d(d["keep_l"], d["keep_r"]).size,
                 d["keep"].size, post))
    return dbg


def run_to_the_cut(prob, bbox, info, shapes, pre, what, **pyramid):
    """the proposal layer with post_nms_top_n = K, so that every survivor is written and compared.  At nms_thresh 1.0
    nothing is suppressed (IoU <= 1): the rows are all K selected candidates in rank order, the box ranked K-th last,
    so a wrong cut or a wrong member of an equal-key group changes a row.  At 0.7 the usual NMS follows."""
    A = prob.shape[1]
    K = pre if 0 < pre < A else A
    for d in run_proposals(prob, bbox, info, shapes, pre, K, 1.0, what=what + " thresh 1", **pyramid):
        np.testing.assert_array_equal(d["keep"], np.arange(K), err_msg="every candidate must be a row")
        print("%s thresh 1: rows are ranks 0..%d, %d distinct boxes" % (
            what, K - 1, np.unique(d["prop_l"], axis=0).shape[0]))
    for d in run_proposals(prob, bbox, info, shapes, pre, K, 0.7, what=what + " thresh 0.7", **pyramid):
        print("%s thresh 0.7: last row has rank %d of K=%d" % (what, d["keep"][-1], K))


def inputs(A, B=1, seed=0, scores=None, spread=0.3, right=None):
    rs = np.random.RandomState(seed)
    prob = rs.rand(B, A, 2).astype(F32)
    if scores is not None:
        prob[:, :, 1] = scores
    bbox = (rs.randn(B, A, 6) * spread).astype(F32)
    if right is not None:
        bbox[:, :, 4:6] = (rs.randn(B, A, 2) * right).astype(F32)
    return prob, bbox


def info_for(shapes, B=1):
    h, w = shapes[0][0] * 4, shapes[0][1] * 4
    return np.array([[h - 3 * b, w - 7 * b, 1.0 + b] for b in range(B)], F32)


def cut_scores(A, K, level, rng):
    """scores whose K-th and (K+1)-th keys (oracle order) first differ in the given bit range: 'pass0' the top 11 bits,
    'pass1' bits 10-20, 'pass2' bits 0-9, 'tie' not at all (equal keys over many 2048-anchor blocks)"""
    X = np.uint32(0xBF000000 | rng.randint(1, 2048) << 10 | rng.randint(1, 1024))     # a float in [0.5, 1)
    Y = {"pass0": X - np.uint32(1 << 21), "pass1": X - np.uint32(1 << 10), "pass2": X - np.uint32(1), "tie": X}[level]
    shared = {"pass0": 0, "pass1": 11, "pass2": 22, "tie": 32}[level]
    keep_bits = np.uint32((0xFFFFFFFF << (32 - shared)) & 0xFFFFFFFF) if shared else np.uint32(0)
    n_eq = 5000 if level == "tie" else 1
    n_gt = K - 1 if level != "tie" else K - 2500
    # above: half share the cut's prefix (they crowd its histogram bucket), half anywhere above it
    lo_above = np.uint64(X) + 1
    near = (np.uint64(X) & np.uint64(keep_bits)) + np.uint64((~keep_bits) & np.uint32(0xFFFFFFFF))
    hi_above = np.uint64(0xFF7FFFFF)
    a1 = rng.randint(int(lo_above), int(max(min(near, hi_above), lo_above)) + 1, n_gt // 2, dtype=np.uint64)
    a2 = rng.randint(int(lo_above), int(hi_above) + 1, n_gt - n_gt // 2, dtype=np.uint64)
    n_lt = A - n_gt - n_eq - (0 if level == "tie" else 1)
    floor_near = np.uint64(Y) & np.uint64(keep_bits) if shared else np.uint64(0x00800000)
    b1 = rng.randint(int(floor_near), int(Y) + 1, n_lt // 2, dtype=np.uint64)
    b2 = rng.randint(0x00800000, int(Y) + 1, n_lt - n_lt // 2, dtype=np.uint64)
    keys = np.concatenate([a1, a2, np.full(n_eq, X, np.uint64), b1, b2] +
                          ([np.array([Y], np.uint64)] if level != "tie" else [])).astype(np.uint32)
    keys = keys[rng.permutation(A)]
    s = key_float(keys)
    k = score_key(s)
    order = O.stable_order_desc(s)
    kk, k1 = int(k[order[K - 1]]), int(k[order[K]])
    first = 32 - (kk ^ k1).bit_length()                 # leading bits the two keys share
    want = {"pass0": range(0, 11), "pass1": range(11, 22), "pass2": range(22, 32), "tie": [32]}[level]
    assert first in want, (level, hex(kk), hex(k1))
    span = np.nonzero(k == kk)[0]
    return s, "cut after %d shared bits, %d keys equal to the K-th over anchor blocks %d..%d" % (
        first, span.size, span.min() // 2048, span.max() // 2048)


CUT_SHAPES = [[80, 128], [40, 64], [20, 32], [10, 16], [5, 8]]     # A = 3 * 13 640 = 40 920, 20 blocks


@pytest.mark.parametrize("level", ["pass0", "pass1", "pass2", "tie"])
@pytest.mark.parametrize("K", [6000, 12000])
def test_proposal_selection_cut(level, K):
    A = n_anchors(CUT_SHAPES)
    rng = np.random.RandomState(K + len(level))
    s, census = cut_scores(A, K, level, rng)
    prob, bbox = inputs(A, scores=s, seed=1)
    print("selection %s K=%d: %s" % (level, K, census))
    run_to_the_cut(prob, bbox, info_for(CUT_SHAPES), CUT_SHAPES, K, "cut %s" % level)


def alphabet_scores(kind, A, rng):
    if kind == "equal":
        return np.full(A, 0.75, F32)
    if kind == "two values":
        return np.where(rng.rand(A) < 0.3, F32(0.9), F32(0.1))
    if kind == "increasing":
        return np.linspace(0, 1, A, dtype=F32)
    if kind == "decreasing":
        return np.linspace(1, 0, A, dtype=F32)
    if kind == "specials":
        tiny = np.finfo(F32).tiny
        alpha = np.array([0.0, -0.0, 1.0, tiny / 4, -tiny / 4, tiny, np.inf, -np.inf, np.nan, -np.nan, 0.5],
                         F32)
        s = rng.rand(A).astype(F32)
        sel = rng.rand(A) < 0.5
        s[sel] = alpha[rng.randint(0, alpha.size, int(sel.sum()))]
        return s
    if kind == "sign-bit NaN":
        s = rng.rand(A).astype(F32)
        s[rng.rand(A) < 0.05] = np.uint32(0xFFC00000).view(F32)     # the NaN an overflowing fp16 softmax returns
        s[rng.rand(A) < 0.05] = np.uint32(0x7FC00000).view(F32)
        s[rng.rand(A) < 0.05] = -0.0
        s[rng.rand(A) < 0.05] = 0.0
        return s
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["equal", "two values", "increasing", "decreasing", "specials", "sign-bit NaN"])
@pytest.mark.parametrize("pre", [6000, 0])
def test_proposal_score_alphabets(kind, pre):
    shapes = SMALL
    A = n_anchors(shapes)
    s = alphabet_scores(kind, A, np.random.RandomState(5))
    prob, bbox = inputs(A, scores=s, seed=2)
    order = O.stable_order_desc(s)
    K = pre if 0 < pre < A else A
    k = score_key(s)
    print("alphabet %s pre=%d: %d NaN, %d -0.0, keys at the cut %08x / %s" % (
        kind, pre, int(np.isnan(s).sum()), int((bits(s) == 0x80000000).sum()), k[order[K - 1]],
        "%08x" % k[order[K]] if K < A else "-"))
    run_to_the_cut(prob, bbox, info_for(shapes), shapes, pre, "alphabet %s" % kind)


@pytest.mark.parametrize("pre", ["0", "1", "A-1", "A", "A+1"])
def test_proposal_pre_nms_sizes(pre):
    shapes = SMALL
    A = n_anchors(shapes)
    p = {"0": 0, "1": 1, "A-1": A - 1, "A": A, "A+1": A + 1}[pre]
    prob, bbox = inputs(A, seed=3)
    run_proposals(prob, bbox, info_for(shapes), shapes, p, 2000, 0.7, what="pre=%s" % pre)


K_SHAPES = [[160, 256], [80, 128], [40, 64], [20, 32], [10, 16]]     # A = 3 * 54 560


@pytest.mark.parametrize("K", [1, 63, 64, 65, 2047, 2048, 2049, 16384])
def test_proposal_k_sizes(K):
    A = n_anchors(K_SHAPES)
    prob, bbox = inputs(A, seed=K)
    run_proposals(prob, bbox, info_for(K_SHAPES), K_SHAPES, K, min(2000, K + 7), 0.7, what="K=%d" % K)


@pytest.mark.parametrize("shapes, ratios, K", [([[700, 1000]], [0.5, 1, 2], 6000),          # A = 2 100 000
                                               ([[2048, 1024]], [0.25, 0.5, 1, 2], 16384)])  # A = 2048 * 4096
def test_proposal_large_a(shapes, ratios, K):
    """more than 1024 compaction blocks: the block scan carries its prefix over several passes"""
    A = n_anchors(shapes, len(ratios))
    rs = np.random.RandomState(11)
    prob = np.zeros((1, A, 2), F32)
    prob[0, :, 1] = np.round(rs.rand(A).astype(F32) * 4096) / 4096                # ties straddle the cut
    bbox = (rs.randn(1, A, 6) * 0.3).astype(F32)
    order = O.stable_order_desc(prob[0, :, 1])[:K]
    print("large A=%d: %d compaction blocks, survivors in blocks %d..%d, %d survivors past block 1024" % (
        A, (A + 2047) // 2048, order.min() // 2048, order.max() // 2048, int((order >= 1024 * 2048).sum())))
    run_to_the_cut(prob, bbox, np.array([[shapes[0][0] * 4, shapes[0][1] * 4, 1.0]], F32), shapes, K, "large A",
                   scales=[64], ratios=ratios, strides=[4])


@pytest.mark.parametrize("shapes, scales, strides, ratios", [
    ([[50, 70]], [24], [6], [1.7]),
    ([[96, 160], [48, 80], [24, 40], [12, 20], [6, 10], [3, 5], [2, 3], [1, 2]],
     [16, 32, 48, 64, 128, 192, 256, 384], [2, 4, 8, 16, 32, 64, 96, 160], [0.25, 0.5, 1.0, 3.0]),
    ([[33, 47], [17, 24]], [40, 90], [5, 11], [0.3, 2.5]),
])
def test_proposal_pyramids(shapes, scales, strides, ratios):
    A = n_anchors(shapes, len(ratios))
    prob, bbox = inputs(A, B=2, seed=len(shapes))
    info = np.array([[shapes[0][0] * strides[0], shapes[0][1] * strides[0], 1.0],
                     [shapes[0][0] * strides[0] - 37, shapes[0][1] * strides[0] - 51, 2.0]], F32)
    run_proposals(prob, bbox, info, shapes, 3000, 300, 0.7, scales=scales, ratios=ratios, strides=strides,
                  what="%d levels x %d ratios" % (len(shapes), len(ratios)))


def two_sided_counts(prob, bbox, info, shapes, K, thr):
    _, _, dbg = O.proposal_layer(prob, bbox, info, "TEST", shapes, return_debug=True, pre_nms_top_n=K,
                                 post_nms_top_n=K, nms_thresh=thr)
    both = np.intersect1d(dbg[0]["keep_l"], dbg[0]["keep_r"])
    return dbg[0], both


def test_proposal_two_sided_post_nms():
    shapes = SMALL
    A = n_anchors(shapes)
    prob, bbox = inputs(A, seed=7, spread=0.4, right=1.2)
    info = info_for(shapes)
    K = 6000
    d, both = two_sided_counts(prob, bbox, info, shapes, K, 0.7)
    only = np.setxor1d(d["keep_l"], d["keep_r"]).size
    assert only > 200, "the two sides' keep lists should differ substantially"
    last = both[(both % 64 == 63) & (both > 64 * 8)]            # survivors that close their chunk
    mids = both[(both % 64 > 8) & (both % 64 < 56) & (both > 64 * 8)]
    assert last.size and mids.size
    at_end = int((both <= last[last.size // 2]).sum())          # the post_nms_top_n-th survivor is a chunk's box 63
    mid = int((both <= mids[mids.size // 2]).sum())
    print("two sides: left %d, right %d, in one list only %d, both %d; post %d ends chunk %d, post %d mid-chunk %d" % (
        d["keep_l"].size, d["keep_r"].size, only, both.size, at_end, last[last.size // 2] // 64, mid,
        mids[mids.size // 2] // 64))
    for post in (at_end, mid, both.size - 1, both.size, both.size + 1, K, 1):
        run_proposals(prob, bbox, info, shapes, K, post, 0.7, what="post=%d" % post)


def test_proposal_iou_at_the_threshold():
    """nms_thresh equal to the IoU of many decoded stride-4 box pairs, and one ulp below it"""
    shapes = SMALL
    A = n_anchors(shapes)
    prob, bbox = inputs(A, seed=8, spread=0.0)
    bbox[:] = 0
    info = info_for(shapes)
    _, _, dbg = O.proposal_layer(prob, bbox, info, "TEST", shapes, return_debug=True, pre_nms_top_n=6000,
                                 post_nms_top_n=6000, nms_thresh=0.7)
    pl = dbg[0]["prop_l"]
    iou = iou32(pl[:600, None], pl[None, :600])[2]
    vals, cnt = np.unique(iou[np.triu(np.ones_like(iou, bool), 1) & (iou > 0.05) & (iou < 0.95)], return_counts=True)
    for v in vals[np.argsort(-cnt)[:3]]:
        for t in (float(v), float(np.nextafter(F32(v), F32(0)))):
            print("proposal IoU threshold %.9g: %d of the first 600 boxes' pairs exactly on it" % (t, int((iou == v).sum())))
            run_proposals(prob, bbox, info, shapes, 6000, 2000, t, what="thresh=%.9g" % t)


@pytest.mark.parametrize("B", [2, 3])
def test_proposal_batches(B):
    shapes = SMALL
    A = n_anchors(shapes)
    rs = np.random.RandomState(B)
    prob, bbox = inputs(A, B=B, seed=B)
    prob[1, :, 1] = np.round(prob[1, :, 1] * 16) / 16                         # heavy ties in the second image only
    if B == 3:
        prob[2, :, 1] = rs.rand(A).astype(F32) ** 8
    info = np.array([[160, 256, 1.0], [97, 131, 1.5], [160, 61, 0.5]][:B], F32)
    run_proposals(prob, bbox, info, shapes, 6000, 300, 0.7, what="B=%d" % B)
    run_proposals(prob, bbox, info, shapes, 2000, 2000, 0.5, what="B=%d TRAIN-like" % B)


def test_proposal_workspace_reuse():
    """one workspace (the default owner's) across decreasing and increasing A: every call reproduces the oracle, and
    the first call's output is reproduced at the end"""
    seq = [K_SHAPES, SMALL, [[8, 8]], SMALL, K_SHAPES]
    first = None
    for i, shapes in enumerate(seq):
        A = n_anchors(shapes)
        prob, bbox = inputs(A, seed=100 + len(shapes))
        run_proposals(prob, bbox, info_for(shapes), shapes, 6000, 300, 0.7, what="reuse %d" % i)
        rl, _ = G.proposal_layer(cu(prob), cu(bbox), cu(info_for(shapes)), "TEST", shapes)
        if i == 0:
            first = rl.cpu().numpy()
        elif i == len(seq) - 1:
            assert_bits(rl.cpu().numpy(), first, "reuse: the first call again")


# -------------------------------------------------------------------------------------------- per-class NMS
def class_nms(scores, boxes, cls, score_thresh, nms_thresh):
    R = scores.shape[0]
    keep = torch.full((max(R, 1),), -7, dtype=torch.int32, device="cuda")
    num = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    s = cu(scores) if R else torch.zeros(0, scores.shape[1], device="cuda")
    b = cu(boxes) if R else torch.zeros(0, boxes.shape[1], device="cuda")
    G.class_nms(s, b, cls, score_thresh, nms_thresh, keep=keep, num=num)
    n = int(num[0])
    assert 0 <= n <= R
    k = keep.cpu().numpy()
    assert (k[n:] == -7).all()                                               # nothing written past the count
    return k[:n]


def class_case(R, nc, seed, pattern):
    rs = np.random.RandomState(seed)
    scores = rs.rand(R, nc).astype(F32)
    boxes = np.zeros((R, 4 * nc), F32)
    for j in range(nc):
        xy = rs.rand(R, 2) * 300
        wh = rs.rand(R, 2) * 150 + 10
        boxes[:, 4 * j:4 * j + 2], boxes[:, 4 * j + 2:4 * j + 4] = xy, xy + wh
    thr = F32(0.05)
    if pattern == "at threshold":
        scores[::3] = thr
        scores[1::3] = np.nextafter(thr, F32(1))
    elif pattern == "equal":
        scores[:] = 0.5
    elif pattern == "nan inf":
        scores[::4] = np.nan
        scores[1::4] = np.inf
        scores[2::9] = np.uint32(0xFFC00000).view(F32)
    elif pattern == "signed zeros":                                     # passes a negative threshold: -0.0 == +0.0
        scores[::2] = -0.0
        scores[1::2] = 0.0
        scores[::7] = -np.inf
    elif pattern in ("chain", "long range"):
        scores[:] = np.linspace(0.9, 0.1, R, dtype=F32)[:, None]
        d = layout(R, [np.arange(R)] if pattern == "chain" else [],
                   [] if pattern == "chain" else [[0] + list(range(R - 1, R - 6, -1)), [65, 200, R - 10]])
        for j in range(nc):
            boxes[:, 4 * j:4 * j + 4] = d[:, :4]
    return scores, boxes


CLASS_CASES = [(R, nc, p) for R in (0, 1, 63, 64, 65, 300, 511, 512) for nc, p in ((2, "random"), (3, "at threshold"))] + \
    [(512, 4, p) for p in ("equal", "nan inf", "signed zeros", "chain", "long range")] + \
    [(R, 2, p) for R in (65, 300) for p in ("nan inf", "signed zeros", "chain")]


@pytest.mark.parametrize("R, nc, pattern", CLASS_CASES)
def test_class_nms_edges(R, nc, pattern):
    scores, boxes = class_case(R, nc, R + nc, pattern)
    st = -1.0 if pattern == "signed zeros" else 0.05
    for cls in range(nc):
        for t in (0.3, 0.7):
            got = class_nms(scores, boxes, cls, st, t)
            ref = O.per_class_nms(scores, boxes, cls, st, t)
            np.testing.assert_array_equal(got, ref, err_msg="R=%d nc=%d %s cls=%d t=%g" % (R, nc, pattern, cls, t))
            if pattern == "chain" and t == 0.3:
                np.testing.assert_array_equal(got, np.arange(0, R, 2))
    passing = int((scores[:, -1] > F32(st)).sum()) if R else 0
    print("class NMS R=%d nc=%d %s: %d rows pass the score threshold in the last class, %d words, %d kept" % (
        R, nc, pattern, passing, (passing + 63) // 64, ref.size))
