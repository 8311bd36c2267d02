"""CPU: the case builders of test_gpu_heads_backward_edges.py (the R-CNN heads' backward kernels of heads_bwd.cu at
their edges) and the proofs behind its two kinds of comparison.

* Exact-arithmetic cases: small integers scaled by powers of two, so that every product and every partial sum the
  kernels form is exact in fp32 whatever the summation order or FMA contraction.  Every fp32 output must then equal
  the float64 result bit for bit, every fp16 output its single round-to-nearest.  test_*_exact_* below prove, for
  every case the GPU file runs, that each class of intermediate stays below 2^24 times its quantum.
* Random cases: float64 references with a per-element a-priori bound (depth + SLACK) 2^-24 sum|terms|, the depth
  read off the kernel's order.  test_*_bound_* run a numpy float32 restatement of that order twice, with products
  rounded and with FMAs emulated (exact product, round-to-odd sum in float64, one rounding to float32): both lie
  inside the bound.  Dropping a term, duplicating one or moving one to the neighbouring row each leaves it.
* Each builder's boundary (block tails, grid-stride passes, thresholds, column splits, phases) is shown reached.
"""
import math

import numpy as np
import pytest
import torch

U = 2.0 ** -24                   # fp32 unit roundoff
SLACK = 2                        # the c of (depth + c) u sum|terms|: the product rounding plus the 1 / (1 - n u) factor
GRID_CAP = 256 * 4 * 132 * 8     # grid_for (heads_bwd.cu) stops growing the grid at this many elements
ONE_BELOW_ONE = 1.0 - 2.0 ** -32


def grid_for(n):
    return (n + 255) // 256 if n < GRID_CAP else 4 * 132 * 8


def passes(n):
    """grid-stride passes of dropout_kernel / permute3_kernel over n elements"""
    return -(-n // (grid_for(n) * 256))


def ordered_depth(R):
    """ordered_sum (heads_bwd.cu): eight interleaved lanes of ceil(R/8) adds, then a 3-level tree"""
    return -(-R // 8) + 3


# ================================================================================================ dropout ====
DROP_NS = [1, 255, 256, 257, GRID_CAP - 1, GRID_CAP, GRID_CAP + 1, 2 * 512 * 2048, 2 * 512 * 2048 + 3]
DROP_PS = [0.0, 0.2, 0.5, ONE_BELOW_ONE]


def threshold(p):
    return int(math.ceil(p * 2.0 ** 32))


def drop_scale(p):
    return np.float32(1.0 / (1.0 - p))


def _special_pairs(p, half):
    """(word, x) pairs: words at thr - 1, thr, thr + 1, 0 and 2^32 - 1; non-finite inputs on dropped and kept words;
    the largest finite input on a kept word"""
    thr = threshold(p)
    big = 65504.0 if half else 3.0e38
    keep = 2 ** 32 - 1                      # never < thr, as p < 1
    pairs = [(w, 1.5 + i) for i, w in enumerate((thr - 1, thr, thr + 1, 0, 2 ** 32 - 1)) if 0 <= w < 2 ** 32]
    if thr > 0:
        pairs += [(0, np.nan), (0, np.inf), (thr - 1, -np.inf)]
    pairs += [(keep, np.inf), (keep, -np.inf), (keep, big), (keep, -big), (thr, np.nan)]
    return pairs


def dropout_case(n, p, half, seed=0):
    """-> x (float16 / float32), words (uint32): random, with the special pairs at the start, at the end and across
    the first grid-stride pass boundary"""
    rs = np.random.RandomState(seed + n % 1000 + int(p * 1000) + 7 * half)
    words = rs.randint(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32)
    x = rs.standard_normal(n).astype(np.float32)
    pairs = _special_pairs(p, half)
    stride = grid_for(n) * 256
    starts = [0, max(n - len(pairs), 0)] + ([stride - len(pairs) // 2] if n > stride else [])
    for s in starts:
        for i, (w, v) in enumerate(pairs):
            if s + i < n:
                words[s + i] = w
                x[s + i] = v
    return x.astype(np.float16 if half else np.float32), words


def dropout_ref(x, words, p, le=False):
    """x[i] = 0 where words[i] < thr (<= with le), else the float32 product x * scale rounded once to x's type"""
    w = words.astype(np.uint64)
    drop = w <= threshold(p) if le else w < threshold(p)
    with np.errstate(over="ignore", invalid="ignore"):
        y = (x.astype(np.float32) * drop_scale(p)).astype(x.dtype)
    y[drop] = 0
    return y


def same_bits(a, b):
    """bit-identical, except that any NaN matches any NaN (the device returns the canonical NaN)"""
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype != b.dtype:
        return False
    it = np.uint16 if a.dtype == np.float16 else np.uint32
    return bool(((a.view(it) == b.view(it)) | (np.isnan(a) & np.isnan(b))).all())


@pytest.mark.parametrize("half", [True, False])
@pytest.mark.parametrize("p", DROP_PS)
@pytest.mark.parametrize("n", DROP_NS)
def test_dropout_case_reaches_its_boundaries(n, p, half):
    x, words = dropout_case(n, p, half)
    thr = threshold(p)
    assert threshold(0.5) == 2 ** 31 and threshold(ONE_BELOW_ONE) == 2 ** 32 - 1 and threshold(0.0) == 0
    present = set(words[:20].tolist())
    assert {w for w in (thr - 1, thr, thr + 1, 0, 2 ** 32 - 1) if 0 <= w < 2 ** 32} & present or n < 5
    ref = dropout_ref(x, words, p)
    # at thr the word is kept, at thr - 1 dropped: '<=' would change the result wherever thr is present
    if n >= 5:
        assert not same_bits(ref, dropout_ref(x, words, p, le=True))
    # more than one grid-stride pass above the cap, and the second pass changes the data (unless p = 0: x * 1)
    assert passes(n) == (2 if n > GRID_CAP else 1)
    if n > GRID_CAP and p > 0:
        stride = grid_for(n) * 256
        assert not same_bits(ref[stride:], x[stride:])
    # dropped NaN / inf become +0, kept inf stays inf, a kept fp16 65504 overflows at scale > 1 exactly as the
    # float32 product rounded to fp16 does
    if n >= 20 and p > 0:
        w = words.astype(np.uint64)
        assert (ref[(w < thr) & ~np.isfinite(x)] == 0).all() and (~np.signbit(ref[w < thr])).all()
        k_inf = (w >= thr) & np.isinf(x)
        assert np.array_equal(ref[k_inf], x[k_inf])
        if half:
            assert np.isinf(ref[(w >= thr) & (x == 65504)]).all()


# ================================================================================================ kpts_logits ====
LOGIT_GS = [1, 2, 27, 28, 64, 65]
LOGIT_RS = [1, 7, 43]


def logits_case(R, G):
    """[R,6,G] float32, every element a distinct value"""
    rs = np.random.RandomState(R * 100 + G)
    v = (np.arange(R * 6 * G, dtype=np.float32) + 1.0) * np.float32(0.25)
    return (v * np.where(rs.rand(v.size) < 0.5, -1, 1).astype(np.float32)).reshape(R, 6, G)


def logits_ref(a):
    R, _, G = a.shape
    return a[:, :4].reshape(R, 4 * G), a[:, 4].copy(), a[:, 5].copy()


def test_logits_cases_cross_the_block_tail():
    ns = [R * 6 * G for R in LOGIT_RS for G in LOGIT_GS]
    assert min(ns) < 256 and any(n > 256 and n % 256 for n in ns) and any(n // 256 >= 2 for n in ns)
    for R in LOGIT_RS:
        for G in LOGIT_GS:
            a = logits_case(R, G)
            assert np.unique(a).size == a.size          # a left / right swap or a channel shift changes the output


# ================================================================================================ box tail ====
BOX_SMALL_RS = [1, 7, 8, 9, 15, 16, 17]
BOX_LARGE_RS = [511, 512, 513, 1024, 1031]
BOX_KS = [1, 31, 255, 256, 257, 2048, 2049]
NCS = [1, 2, 3, 4]
SCALES = [(1.0, 1.0), (1.25, 2.0 ** 12), (1.25, 1.0), (1.0, 2.0 ** 12)]     # (mask_scale, grad_scale)


def box_cases():
    """(R, K, nc, mask_scale, grad_scale).  The full product R x K x nc for R <= 17, the four scale pairs in turn;
    for R >= 511 a pairwise-covering subset: every (R, K), every (R, nc) and every (R, scale pair)"""
    out = []
    for R in BOX_SMALL_RS:
        for K in BOX_KS:
            for nc in NCS:
                out.append((R, K, nc) + SCALES[len(out) % 4])
    for i, R in enumerate(BOX_LARGE_RS):
        for j, K in enumerate(BOX_KS):
            out.append((R, K, NCS[(i + j) % 4]) + SCALES[(i + j) % 4])
        for nc in NCS:
            out.append((R, BOX_KS[(i + 3 * nc) % 7], nc) + SCALES[(i + nc + 1) % 4])
    return out


BOX_CASES = box_cases()
BOX_BOUND_CASES = [(9, 257, 3, 1.25, 1.0), (17, 2049, 4, 1.0, 2.0 ** 12), (513, 255, 2, 1.25, 2.0 ** 12),
                   (1031, 31, 1, 1.0, 1.0)]


def box_exact(R, K, nc, seed=0):
    """d = k 2^-10 (|k| <= 8), W = k 2^-8 (|k| <= 8), fc7 an integer in 0..15, ~30 % exact zeros plus a few -0.0 and
    negative entries (the mask's edge).  The cls and dim blocks hold odd k, the box block even k, so every element
    differs from its neighbour across a block boundary.  -> d_cls, d_box, d_dim, fc7, w_cls, w_box, w_dim (float32)"""
    rs = np.random.RandomState(1 + seed + R * 7919 + K * 31 + nc)
    k = lambda shape, odd: rs.randint(-4, 4, shape) * 2 + odd          # -8..6 even or -7..7 odd
    d = [(k((R, n * nc), n != 6) * 2.0 ** -10).astype(np.float32) for n in (1, 6, 5)]
    W = [(k((n * nc, K), n != 6) * 2.0 ** -8).astype(np.float32) for n in (1, 6, 5)]
    fc7 = rs.randint(1, 16, (R, K)).astype(np.float32)
    q = rs.rand(R, K)
    fc7[q < 0.30] = 0.0
    fc7[(q >= 0.30) & (q < 0.33)] = -0.0
    fc7[(q >= 0.33) & (q < 0.36)] = -rs.randint(1, 5, ((q >= 0.33) & (q < 0.36)).sum())
    return d[0], d[1], d[2], fc7, W[0], W[1], W[2]


def box_random(R, K, nc, seed=0):
    """random fp32 operands of the same layout: fc7 ReLU'd normal with -0.0 and negatives, d ~ 1e-2, W ~ 2e-2"""
    rs = np.random.RandomState(2 + seed + R * 7919 + K * 31 + nc)
    d = [(rs.standard_normal((R, n * nc)) * 1e-2).astype(np.float32) for n in (1, 6, 5)]
    W = [(rs.standard_normal((n * nc, K)) * 2e-2).astype(np.float32) for n in (1, 6, 5)]
    fc7 = np.maximum(rs.standard_normal((R, K)), 0).astype(np.float32)
    q = rs.rand(R, K)
    fc7[q < 0.03] = -0.0
    fc7[(q >= 0.03) & (q < 0.06)] *= -1
    return d[0], d[1], d[2], fc7, W[0], W[1], W[2]


def box_ref(d_cls, d_box, d_dim, fc7, w_cls, w_box, w_dim, ms, gs):
    """float64 references and per-element bounds (torch, on the operands' device):
    dz = gs ms [fc7 > 0] d W: 12 nc FMAs in o order, one rounding for ms (gs a power of two);
    dW = d^T fc7 and db = sum_r d: ordered_sum's depth, plus the product rounding for dW"""
    t = lambda a: torch.as_tensor(a).double()
    d = torch.cat([t(d_cls), t(d_box), t(d_dim)], 1)
    W = torch.cat([t(w_cls), t(w_box), t(w_dim)], 0)
    f = t(fc7)
    R, n_out = d.shape
    m = (f > 0).double() * ms * gs
    ref = {"dz": torch.where(f > 0, (d @ W) * m, torch.zeros_like(f)), "dw": d.t() @ f, "db": d.sum(0)}   # +0 masked
    bound = {"dz": (n_out + 1 + SLACK) * U * (d.abs() @ W.abs()) * m,
             "dw": (ordered_depth(R) + 1 + SLACK) * U * (d.abs().t() @ f.abs()),
             "db": (ordered_depth(R) + SLACK) * U * d.abs().sum(0)}
    return ref, bound


def fp16_bound(ref, b32):
    """|fp16(a) - ref| for a float32 result a with |a - ref| <= b32: b32 plus half an fp16 ulp of a"""
    return b32 * (1 + 2.0 ** -11) + 2.0 ** -11 * ref.abs() + 2.0 ** -25


def _multiple_below(x, q):
    """every value an integer multiple of q and below 2^24 q in magnitude (exact in fp32)"""
    x = np.asarray(x, np.float64)
    return bool((np.floor(x / q) == x / q).all()) and float(np.abs(x).max(initial=0)) < 2.0 ** 24 * q


def box_exact_proof(R, K, nc, ms, gs):
    d_cls, d_box, d_dim, fc7, w_cls, w_box, w_dim = box_exact(R, K, nc)
    d = np.concatenate([d_cls, d_box, d_dim], 1).astype(np.float64)
    W = np.concatenate([w_cls, w_box, w_dim], 0).astype(np.float64)
    f = fc7.astype(np.float64)
    assert _multiple_below(d, 2.0 ** -10) and _multiple_below(W, 2.0 ** -8) and _multiple_below(f, 1.0)
    # dz: products and FMA partials (quantum 2^-18) bounded by sum_o |d W|, then x ms (quantum 2^-20), x gs exact
    s = np.abs(d) @ np.abs(W)
    assert s.max() < 2.0 ** 24 * 2.0 ** -18 and s.max() * ms < 2.0 ** 24 * 2.0 ** -20
    assert s.max() * ms * gs < 65504                                                      # dz16 stays finite
    # dW: products, lane partials and tree sums (quantum 2^-10) bounded by sum_r |d fc7|; db by sum_r |d|
    assert (np.abs(d).T @ np.abs(f)).max() < 2.0 ** 24 * 2.0 ** -10
    assert np.abs(d).sum(0).max() < 2.0 ** 24 * 2.0 ** -10
    # the cls | box | dim split: the columns either side of nc and 7 nc differ, so a one-column shift changes dW, db
    for b in (nc, 7 * nc):
        assert not np.array_equal(d[:, b - 1], d[:, b]) and not np.array_equal(W[b - 1], W[b]), b


@pytest.mark.parametrize("case", BOX_CASES, ids=lambda c: "R%d-K%d-nc%d-ms%g-gs%g" % c)
def test_box_exact_case_is_exact(case):
    R, K, nc, ms, gs = case
    box_exact_proof(R, K, nc, ms, gs)


def test_box_cases_cover_the_edges():
    cs = BOX_CASES
    small = {(R, K, nc) for R, K, nc, _, _ in cs if R in BOX_SMALL_RS}
    assert len(small) == len(BOX_SMALL_RS) * len(BOX_KS) * len(NCS)
    for R in BOX_LARGE_RS:
        assert {K for r, K, *_ in cs if r == R} == set(BOX_KS)
        assert {nc for r, _, nc, *_ in cs if r == R} == set(NCS)
        assert {(ms, gs) for r, _, _, ms, gs in cs if r == R} == set(SCALES)
    # K: the partial last 256-wide block (K % 256 != 0) and the full one; R: ordered_sum with no, one and seven tail
    # terms, below and above one full round of eight lanes
    assert {K % 256 for K in BOX_KS} >= {0, 1, 31, 255} and {K // 256 for K in BOX_KS} >= {0, 1, 8}
    assert {R % 8 for R in BOX_SMALL_RS + BOX_LARGE_RS} == {0, 1, 7} and min(BOX_SMALL_RS) < 8 < max(BOX_SMALL_RS)
    assert 12 * max(NCS) == 48                                            # nc = 4 fills box_tail_dx's dv[48]


# float32 restatements of the kernels' order --------------------------------------------------------------------
def _rto_add(a, b):
    """a + b in float64 rounded to odd: exactly representable results are exact, others keep a sticky last bit"""
    s = a + b
    bb = s - a
    e = (a - (s - bb)) + (b - bb)
    fix = (e != 0) & ((s.view(np.int64) & 1) == 0)
    return np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)


def madd(a, b, c, fma):
    """float32 a b + c: product rounded first, or fused (exact product, one rounding, via round-to-odd)"""
    a, b, c = (np.asarray(v, np.float32) for v in (a, b, c))
    if not fma:
        return (a * b).astype(np.float32) + c
    return _rto_add(a.astype(np.float64) * b.astype(np.float64), np.broadcast_to(c, np.broadcast(a, b, c).shape)
                    .astype(np.float64)).astype(np.float32)


def ordered_sum32(a, b=None, fma=False):
    """ordered_sum over the leading axis: lane r % 8 (the tail loop restarts at lane 0 on a multiple of 8)"""
    R = a.shape[0]
    shape = np.broadcast(a[0], b[0]).shape if b is not None else a.shape[1:]
    p = [np.zeros(shape, np.float32) for _ in range(8)]
    for r in range(R):
        j = r % 8
        p[j] = p[j] + a[r] if b is None else madd(a[r], b[r], p[j], fma)
    return ((p[0] + p[1]) + (p[2] + p[3])) + ((p[4] + p[5]) + (p[6] + p[7]))


def box_restated(d_cls, d_box, d_dim, fc7, w_cls, w_box, w_dim, ms, gs, fma):
    d = np.concatenate([d_cls, d_box, d_dim], 1)
    W = np.concatenate([w_cls, w_box, w_dim], 0)
    s = np.zeros(fc7.shape, np.float32)
    for o in range(d.shape[1]):
        s = madd(d[:, o:o + 1], W[o][None, :], s, fma)
    dz = np.where(fc7 > 0, (s * np.float32(ms)) * np.float32(gs), np.float32(0)).astype(np.float32)
    dw = ordered_sum32(d[:, :, None], fc7[:, None, :], fma)
    db = ordered_sum32(d)
    return {"dz": dz, "dw": dw, "db": db}


def worst_ratio(got, ref, bound):
    got = torch.as_tensor(np.asarray(got)).double() if not torch.is_tensor(got) else got.double()
    err = (got.to(ref.device) - ref).abs()
    return float((err / bound.clamp_min(1e-300)).max())


@pytest.mark.parametrize("case", BOX_BOUND_CASES, ids=lambda c: "R%d-K%d-nc%d" % c[:3])
def test_box_bound_sound_and_tight(case):
    R, K, nc, ms, gs = case
    ops = box_random(R, K, nc)
    ref, bound = box_ref(*ops, ms, gs)
    for fma in (False, True):
        got = box_restated(*ops, ms, gs, fma)
        for k in ref:
            assert worst_ratio(got[k], ref[k], bound[k]) <= 1.0, (k, fma)
        dz16 = torch.from_numpy(got["dz"].astype(np.float16).astype(np.float64))
        assert worst_ratio(dz16, ref["dz"].half().double(), fp16_bound(ref["dz"], bound["dz"])) <= 1.0 or \
            worst_ratio(dz16, ref["dz"], fp16_bound(ref["dz"], bound["dz"])) <= 1.0
    d = torch.from_numpy(np.concatenate(ops[:3], 1)).double()
    f = torch.from_numpy(ops[3]).double()
    r = R - 1                                   # the last RoI: in ordered_sum's tail when R % 8 != 0
    mut = {"drop": ref["dw"] - d[r][:, None] * f[r][None, :],
           "duplicate": ref["dw"] + d[r][:, None] * f[r][None, :],
           "neighbour row": ref["dw"] - d[r][:, None] * f[r][None, :] + torch.roll(d[r][:, None] * f[r][None, :], 1, 0)}
    for name, m in mut.items():
        assert worst_ratio(m, ref["dw"], bound["dw"]) > 1.0, name
    assert worst_ratio(ref["db"] - d[r], ref["db"], bound["db"]) > 1.0
    W = torch.from_numpy(np.concatenate(ops[4:], 0)).double()
    mask = (f > 0).double() * ms * gs
    one = d[:, :1] * W[:1] * mask                # the first output's term of every dz
    for m in (ref["dz"] - one, ref["dz"] + one, ref["dz"] - one + torch.roll(one, 1, 1)):
        assert worst_ratio(m, ref["dz"], bound["dz"]) > 1.0


# ------------------------------------------------------------------- sb_box_tail_scores' cls_score
SCORE_CASES = [(nc, K) for nc in NCS for K in (255, 256, 257, 2048)]


def score_bound(fc7, w, b):
    """cls_score[r][j] = sum_k fc7 w + b: per thread ceil(K/256) FMAs, a 5-level warp tree, 8 warp partials added in
    order, then the bias"""
    f, w, b = (torch.as_tensor(v).double() for v in (fc7, w, b))
    K = f.shape[1]
    ref = f @ w.t() + b
    return ref, (-(-K // 256) + 5 + 8 + 1 + SLACK) * U * (f.abs() @ w.abs().t() + b.abs())


def score_restated(fc7, w, b, fma):
    R, K = fc7.shape
    out = np.zeros((R, w.shape[0]), np.float32)
    for j in range(w.shape[0]):
        lane = np.zeros((R, 256), np.float32)
        for k0 in range(0, K, 256):
            n = min(256, K - k0)
            lane[:, :n] = madd(fc7[:, k0:k0 + n], w[j, k0:k0 + n][None, :], lane[:, :n], fma)
        v = lane.reshape(R, 8, 32)
        for o in (16, 8, 4, 2, 1):              # __shfl_xor tree: lane i adds lane i ^ o
            v = v + v[:, :, np.arange(32) ^ o]
        s = np.zeros(R, np.float32)
        for q in range(8):
            s = s + v[:, q, 0]
        out[:, j] = s + b[j]
    return out


def box_tail_weights(K, nc, exact, seed=0):
    rs = np.random.RandomState(3 + seed + K * 5 + nc)
    if exact:
        W = [(rs.randint(-8, 9, (n * nc, K)) * 2.0 ** -8).astype(np.float32) for n in (1, 6, 5)]
        b = [(rs.randint(-8, 9, n * nc) * 2.0 ** -8).astype(np.float32) for n in (1, 6, 5)]
    else:
        W = [(rs.standard_normal((n * nc, K)) * 2e-2).astype(np.float32) for n in (1, 6, 5)]
        b = [(rs.standard_normal(n * nc) * 1e-1).astype(np.float32) for n in (1, 6, 5)]
    return W[0], b[0], W[1], b[1], W[2], b[2]


@pytest.mark.parametrize("nc,K", [(1, 257), (4, 2048)])
def test_score_bound_sound_and_tight(nc, K):
    fc7 = box_random(33, K, nc)[3]
    w, b = box_tail_weights(K, nc, False)[:2]
    ref, bound = score_bound(fc7, w, b)
    for fma in (False, True):
        assert worst_ratio(score_restated(fc7, w, b, fma), ref, bound) <= 1.0
    f, wd = torch.from_numpy(fc7).double(), torch.from_numpy(w).double()
    one = f[:, -1:] * wd[:, -1][None, :]         # the last K element: the partial block's lane
    assert worst_ratio(ref - one, ref, bound) > 1.0 and worst_ratio(ref + one, ref, bound) > 1.0


def test_score_exact_cases_are_exact():
    for nc, K in SCORE_CASES:
        fc7 = box_exact(5, K, nc)[3]
        w, b = box_tail_weights(K, nc, True)[:2]
        s = np.abs(fc7.astype(np.float64)) @ np.abs(w.astype(np.float64)).T + np.abs(b)
        assert s.max() < 2.0 ** 24 * 2.0 ** -8                       # quantum 2^-8 (integer fc7, W k 2^-8)


# ================================================================================================ keypoint tail ====
KP_GS = [2, 4, 6, 28, 30, 62, 64]
KP_CS = [32, 64, 96, 256, 1024]
KP_RS = [1, 7, 8, 9, 17, 512, 513]
KP_SCALES = [1.0, 2.0 ** 10]


def kpts_cases():
    """(R, G, C, grad_scale): every (G, C) at R = 1 (grad_scale 1) and at R = 9 (2^10); every (R, G) at C = 32
    (grad_scale 1); every (R, C) at G = 6 (2^10).  So every pair of values of two dimensions appears."""
    out = []
    for G in KP_GS:
        for C in KP_CS:
            out += [(1, G, C, 1.0), (9, G, C, 2.0 ** 10)]
    for R in KP_RS:
        out += [(R, G, 32, 1.0) for G in KP_GS] + [(R, 6, C, 2.0 ** 10) for C in KP_CS]
    return sorted(set(out))


KP_CASES = kpts_cases()
KP_BOUND_CASES = [(9, 64, 32, 2.0 ** 10), (17, 30, 64, 1.0), (513, 6, 32, 2.0 ** 10), (8, 28, 96, 1.0)]


def _kpts_level(R, G):
    """operand magnitudes (up max, |w| / 2^-6 max, |d logits| / 2^-8 max) that keep R G^2-term sums exact"""
    n = R * G * G
    return (7, 8, 8) if n <= 40000 else (3, 4, 4) if n <= 300000 else (1, 2, 2) if n <= 1000000 else (1, 1, 1)


def kpts_exact_grads(R, G, C, seed=0):
    """w = k 2^-6, d logits = k 2^-8 -> w [6,C], d_kpts [R,4G], d_left [R,G], d_right [R,G] (float32)"""
    _, kw, kd = _kpts_level(R, G)
    rs = np.random.RandomState(4 + seed + R * 131 + G * 17 + C)
    w = (rs.randint(-kw, kw + 1, (6, C)) * 2.0 ** -6).astype(np.float32)
    dp = (rs.randint(-kd, kd + 1, (R, 6, G)) * 2.0 ** -8).astype(np.float32)
    return w, dp[:, :4].reshape(R, 4 * G).copy(), dp[:, 4].copy(), dp[:, 5].copy()


PHASE_DENSITY = (9, 7, 5, 3)          # tenths of the pixels of phase (y % 2) * 2 + x % 2 that may be positive


def kpts_exact_up(R, G, C, seed=0, device="cpu"):
    """up16 [R,G,G,C] fp16: integers 0..umax, a zero row and a zero column per RoI, a phase-dependent density of
    positives, and a few -1 and -0.0 entries (mask <= 0)"""
    umax = _kpts_level(R, G)[0]
    g = torch.Generator().manual_seed(5 + seed + R * 131 + G * 17 + C)
    u = torch.randint(1, umax + 1, (R, G, G, C), generator=g, dtype=torch.int16).to(device)
    q = torch.randint(0, 10, (R, G, G, C), generator=g, dtype=torch.int8).to(device)
    ph = (torch.arange(G, device=device) % 2)[:, None] * 2 + (torch.arange(G, device=device) % 2)[None, :]
    dens = torch.tensor(PHASE_DENSITY, device=device, dtype=torch.int8)[ph]             # [y,x]
    u = torch.where(q < dens[None, :, :, None], u, torch.zeros_like(u)).half()
    u[q == 0] = -1.0
    u[q == 1] = -0.0
    rr = torch.arange(R, device=device)
    u[rr, (rr * 5 + 1) % G] = 0                 # a zero row ...
    u[rr, :, (rr * 3 + 2) % G] = 0              # ... and a zero column per RoI
    return u


def kpts_random(R, G, C, seed=0, device="cpu"):
    g = torch.Generator().manual_seed(6 + seed + R * 131 + G * 17 + C)
    up = torch.randn(R, G, G, C, generator=g).half().to(device)
    w = (torch.randn(6, C, generator=g) * 0.05).numpy()
    dp = (torch.randn(R, 6, G, generator=g) * 1e-3).numpy()
    return up, w, dp[:, :4].reshape(R, 4 * G).copy(), dp[:, 4].copy(), dp[:, 5].copy()


def logit_grads(dkp, dl, dr):
    """[R,6,G] float64 torch from the three loss gradients"""
    dkp, dl, dr = (torch.as_tensor(v).double() for v in (dkp, dl, dr))
    R, G = dl.shape
    return torch.cat([dkp.view(R, 4, G), dl.view(R, 1, G), dr.view(R, 1, G)], 1)


def phase_major(full, swap=False):
    """[R,G,G,C] -> [R,G/2,G/2,4C], pixel (y, x) into channel block (y % 2) * 2 + x % 2 (x % 2 * 2 + y % 2 with swap)"""
    R, G, _, C = full.shape
    v = full.reshape(R, G // 2, 2, G // 2, 2, C)
    return (v.permute(0, 1, 3, 4, 2, 5) if swap else v.permute(0, 1, 3, 2, 4, 5)).reshape(R, G // 2, G // 2, 4 * C)


def kpts_ref(up, w, dp, gs):
    """float64 references and per-element bounds (torch, on up's device); dp [R,6,G] float64.
    g[r,x,c] = sum_k w dp: 6 FMAs; colsum: 4 interleaved lanes of G/4 adds and a 2-level tree; dW: G FMAs per RoI
    then ordered_sum over R; d deconv bias: G FMAs of g x (count of up > 0) then ordered_sum; db: G adds, ordered_sum,
    x G"""
    u = up.double()
    R, G, _, C = u.shape
    w = torch.as_tensor(w).to(u.device).double()
    dp = dp.to(u.device)
    g = torch.einsum("kc,rkx->rxc", w, dp)
    ga = torch.einsum("kc,rkx->rxc", w.abs(), dp.abs())
    on = (u > 0).double().sum(1)                                   # [R,x,C]
    cs, csa = u.sum(1), u.abs().sum(1)
    dr = R // 8 + (R % 8 > 0) + 3
    full = torch.where(u > 0, g[:, None].expand_as(u), torch.zeros_like(u))                 # +0 where masked
    ref = {"dup": phase_major(full * gs), "dw": torch.einsum("rkx,rxc->kc", dp, cs).reshape(-1),
           "db": dp.sum((0, 2)) * G, "db_up": (g * on).sum((0, 1))}
    b32 = (6 + SLACK) * U * gs * ga[:, None] * (u > 0).double()
    bound = {"dup": fp16_bound(ref["dup"], phase_major(b32)),
             "dw": ((G + 3) // 4 + 2 + G + dr + SLACK) * U * torch.einsum("rkx,rxc->kc", dp.abs(), csa).reshape(-1),
             "db": (G + dr + 1 + SLACK) * U * dp.abs().sum((0, 2)) * G,
             "db_up": (6 + G + dr + SLACK) * U * (ga * on).sum((0, 1))}
    return ref, bound


def kpts_restated(up, w, dp, gs, fma):
    """float32 numpy restatement of kpts_tail_bwd_kernel + kpts_tail_bwd_reduce_kernel"""
    u = up.float().numpy()
    R, G, _, C = u.shape
    w = np.asarray(w, np.float32)
    dp = np.asarray(dp, np.float32)
    aw = [np.zeros((R, C), np.float32) for _ in range(6)]
    ab = np.zeros((R, C), np.float32)
    full = np.zeros((R, G, G, C), np.float32)
    for x in range(G):
        g = np.zeros((R, C), np.float32)
        for k in range(6):
            g = madd(w[k][None, :], dp[:, k, x][:, None], g, fma)
        h = (g * np.float32(gs)).astype(np.float16).astype(np.float32)
        cs = [np.zeros((R, C), np.float32) for _ in range(4)]
        on = np.zeros((R, C), np.float32)
        for y in range(G):
            cs[y & 3] = cs[y & 3] + u[:, y, x]
            on += u[:, y, x] > 0
            full[:, y, x] = np.where(u[:, y, x] > 0, h, 0)
        colsum = (cs[0] + cs[1]) + (cs[2] + cs[3])
        for k in range(6):
            aw[k] = madd(dp[:, k, x][:, None], colsum, aw[k], fma)
        ab = madd(g, on, ab, fma)
    border = np.zeros((R, 6), np.float32)
    for x in range(G):
        border = border + dp[:, :, x]
    dw = np.stack([ordered_sum32(a) for a in aw], 0).reshape(-1)
    return {"dup": phase_major(torch.from_numpy(full)).numpy(), "dw": dw, "db": ordered_sum32(border) * np.float32(G),
            "db_up": ordered_sum32(ab)}


def kpts_exact_proof(R, G, C):
    umax = _kpts_level(R, G)[0]
    w, dkp, dl, dr = kpts_exact_grads(R, G, C)
    dp = logit_grads(dkp, dl, dr).numpy()
    assert _multiple_below(w, 2.0 ** -6) and _multiple_below(dp, 2.0 ** -8)
    ga = np.einsum("kc,rkx->rxc", np.abs(w.astype(np.float64)), np.abs(dp))         # |w| |dp| summed over k
    q = 2.0 ** -14
    assert ga.max() < 2.0 ** 24 * q                                    # g, its products and FMA partials
    assert G * umax < 2.0 ** 24                                        # colsum (integers)
    # dW: per RoI sum_x |dp| colsum, and over R (the reduce): bounded by sum_{r,x} |dp| G umax, quantum 2^-8
    assert (np.abs(dp).sum((0, 2)) * G * umax).max() < 2.0 ** 24 * 2.0 ** -8
    # d deconv bias: sum_{r,x} |g| on <= G sum_{r,x} |g|, quantum 2^-14
    assert (ga.sum((0, 1)) * G).max() < 2.0 ** 24 * q
    # db: border sums and the reduce (quantum 2^-8), then x G
    assert (np.abs(dp).sum((0, 2)) * G).max() < 2.0 ** 24 * 2.0 ** -8
    # dup16: g gs is exact in fp32 (a power-of-two scale) and finite in fp16
    assert ga.max() * q * 2.0 ** 10 < 65504
    return w, dp


@pytest.mark.parametrize("case", KP_CASES, ids=lambda c: "R%d-G%d-C%d-gs%g" % c)
def test_kpts_exact_case_is_exact(case):
    R, G, C, gs = case
    kpts_exact_proof(R, G, C)
    if R * G * G * C <= 1 << 20:
        up = kpts_exact_up(R, G, C)
        umax = _kpts_level(R, G)[0]
        u = up.float()
        assert bool((u == u.round()).all()) and float(u.max()) <= umax and float(u.min()) >= -1
        z = (u == 0).all(3)
        assert bool(z.all(2).any(1).all()) and bool(z.all(1).any(1).all())        # a zero row and column per RoI
        assert bool(((u == 0) & torch.signbit(u)).any()) or R * G * G * C < 4000
        # the four phases differ: swapping the phase bits of the dup index changes the result
        w, dp = kpts_exact_proof(R, G, C)
        g = torch.einsum("kc,rkx->rxc", torch.from_numpy(w).double(), torch.from_numpy(dp))
        fm = g[:, None] * (u > 0).double() * gs
        assert not torch.equal(phase_major(fm), phase_major(fm, swap=True))


def test_kpts_cases_cover_the_edges():
    cs = KP_CASES
    for a, b in ((0, 1), (0, 2), (1, 2), (0, 3), (1, 3), (2, 3)):
        vals = (KP_RS, KP_GS, KP_CS, KP_SCALES)
        assert {(c[a], c[b]) for c in cs} == {(x, y) for x in vals[a] for y in vals[b]}, (a, b)
    assert {R % 8 for R in KP_RS} >= {0, 1, 7}
    assert max(C for _, _, C, _ in cs) == 1024                        # a 1024-thread CTA


@pytest.mark.parametrize("case", KP_BOUND_CASES, ids=lambda c: "R%d-G%d-C%d" % c[:3])
def test_kpts_bound_sound_and_tight(case):
    R, G, C, gs = case
    up, w, dkp, dl, dr = kpts_random(R, G, C)
    dp = logit_grads(dkp, dl, dr)
    ref, bound = kpts_ref(up, w, dp, gs)
    for fma in (False, True):
        got = kpts_restated(up, w, dp.float().numpy(), gs, fma)
        for k in ref:
            assert worst_ratio(got[k], ref[k], bound[k]) <= 1.0, (k, fma)
    # a term dropped, duplicated or moved to the neighbouring row leaves the bound: the last RoI's x = G - 1 term
    u = up.double()
    r, x = R - 1, G - 1
    wd = torch.from_numpy(w).double()
    t_dw = (dp[r, :, x][:, None] * u[r, :, x].sum(0)[None, :]).reshape(-1)
    g = (wd * dp[r, :, x][:, None]).sum(0)
    t_bu = g * (u[r, :, x] > 0).double().sum(0)
    for name, ref_k, t in (("dw", ref["dw"], t_dw), ("db_up", ref["db_up"], t_bu)):
        for m in (ref_k - t, ref_k + t, ref_k - t + torch.roll(t, 1, 0)):
            assert worst_ratio(m, ref_k, bound[name]) > 1.0, name
    assert worst_ratio(ref["db"] - dp[r, :, x] * G, ref["db"], bound["db"]) > 1.0
    # a dup element with the neighbouring column's gradient
    shifted = phase_major(torch.roll(phase_major_inv(ref["dup"]), 1, 2))
    assert worst_ratio(shifted, ref["dup"], bound["dup"]) > 1.0


def phase_major_inv(ph):
    R, Gh, _, C4 = ph.shape
    C = C4 // 4
    return ph.view(R, Gh, Gh, 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(R, 2 * Gh, 2 * Gh, C)


def test_phase_major_round_trip():
    x = torch.arange(2 * 4 * 4 * 3, dtype=torch.float64).view(2, 4, 4, 3)
    ph = phase_major(x)
    assert torch.equal(phase_major_inv(ph), x)
    assert ph[0, 0, 1, 2 * 3 + 1] == x[0, 1, 2, 1]                 # pixel (1, 2): (0, 1), phase (1, 0) = block 2


# ================================================================================================ permute3 ====
PERM_SHAPES = [(3, 5, 7), (1, 7, 1), (4, 1, 9), (1, 1, 1), (4, 1031, 263)]
ORDERS = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)]


def permute_strides(dims, order):
    """the strides s of sb_permute3 that make dst = src.view(dims).permute(order).contiguous()"""
    od = [dims[a] for a in order]
    cs = [od[1] * od[2], od[2], 1]
    s = [0, 0, 0]
    for j, a in enumerate(order):
        s[a] = cs[j]
    return tuple(s)


def test_permute_cases():
    assert (4 * 1031 * 263) > GRID_CAP and passes(4 * 1031 * 263) == 2
    for dims in PERM_SHAPES[:3]:
        for order in ORDERS:
            s = permute_strides(dims, order)
            src = np.arange(np.prod(dims)).reshape(dims)
            dst = np.empty(np.prod(dims), np.int64)
            i0, i1, i2 = np.meshgrid(*[np.arange(d) for d in dims], indexing="ij")
            dst[(i0 * s[0] + i1 * s[1] + i2 * s[2]).ravel()] = src.ravel()
            assert np.array_equal(dst, np.transpose(src, order).ravel())


# ================================================================================================ chain ====
def synth_rois(R, B, H, W, seed=0):
    """R left / right RoIs [R,5] (image index, x1, y1, x2, y2) spread over B images: sizes from 8 px to the whole
    image, the right box shifted left by a disparity"""
    rs = np.random.RandomState(8 + seed + R)
    b = np.sort(np.arange(R) % B).astype(np.float32)
    w = rs.uniform(8, W - 2, R)
    h = rs.uniform(8, H - 2, R)
    x1 = rs.uniform(0, W - 1 - w)
    y1 = rs.uniform(0, H - 1 - h)
    rl = np.stack([b, x1, y1, x1 + w, y1 + h], 1)
    disp = np.minimum(rs.uniform(0, 40, R), x1)
    rr = rl.copy()
    rr[:, 1] -= disp
    rr[:, 3] -= disp
    return rl.astype(np.float32), rr.astype(np.float32)


def test_synth_rois_inside_every_image():
    for R, B in ((1, 1), (129, 2), (1024, 2)):
        rl, rr = synth_rois(R, B, 100, 333)
        assert rl.shape == (R, 5) and set(rl[:, 0].tolist()) == set(range(B))
        for r in (rl, rr):
            assert (r[:, 1] >= 0).all() and (r[:, 3] <= 332).all() and (r[:, 4] <= 99).all()
            assert (r[:, 3] - r[:, 1] >= 8).all()
