"""GPU: the backward of the pyramid RoIAlign (roi_align.cu, sb_roi_align_pyramid_backward), engine.roi_align_backward
and train.loss_gradients, the whole six-term training loss differentiated end to end.

Kernel against a float64 mirror, element by element.  The mirror reuses the forward mirror's geometry of
test_gpu_roi_heads (roi_geometry, axis_taps: the fp32 lattice coordinates rebuilt exactly, so h0, hr and the four fp64
tap weights are exact) and takes each RoI's level from the forward itself (a one-hot probe through
roi_align_pyramid_nhwc), so a RoI within an ulp of a level boundary is checked at the level the forward read.  It then
restates the kernel's arithmetic in two ways:

  fixed point  gl = ((G[i-1][j-1] + G[i-1][j]) + (G[i][j-1] + G[i][j])) in float64, times 2^(e-2) (exact), times w,
               rint, summed exactly in int64; dP + acc 2^-e in float64, rounded once to fp32.  e = 60 - ex - k with
               max|G| < 2^ex over every source of the call and T = sum R (P+1)^2 <= 2^k.  The kernel must match this
               bit for bit: the same roundings in the same order.
  exact        gl / 4 * w summed in float64 (no quantisation).  Per element, with n the number of contributions,
               S = sum over them of |w| (|a|+|b|+|c|+|d|) / 4 and q = 2^-e the fixed-point quantum:
                   |kernel - (dP + exact)| <= q n + 2^-40 (S + |dP|) + ulp32(kernel) / 2
               q n: each rint is off by at most q / 2; 2^-40 (S + |dP|): the float64 roundings of gl, gl w, the
               conversion and the add in the kernel, and the mirror's own float64 sum over at most 2^13 terms;
               ulp / 2: the final rounding to fp32.

Adjoint identity against the forward on the device, RoI by RoI: <pyramid_nhwc(F), G_r> = <F, backward(G_r)> in float64
within 2^-20 <|F|, S_r> + <|F|, q n_r>: the forward's output is within 2^-22 A of float64 (test_gpu_roi_heads) and
sum |G| A <= <|F|, S>; the backward's error is the bound above.  The level gradients sit in NaN-sentinel guard buffers.

End to end: train.loss_gradients against fp32 autograd (TF32 off) through oracle.model.trunk_fpn, rpn_head, a
differentiable pyramid RoIAlign over oracle.ops.roi_align_forward / roi_align_backward and roi_levels, the train-mode
heads of test_gpu_rcnn_backward with the engine's dropout masks, and rpn_losses + rcnn_losses, fed the engine's anchor
targets, sampled RoIs and targets; at 160x256 (B = 1 and 2, FIXED_BLOCKS 0 and 1) and 600x1987, with a non-uniform
uncert in three of the five cases.  Bars: losses and d total / d uncert 1e-3, RPN and box head 5e-3, trunk and keypoint
convs 1e-1, FPN 2e-2 and at most twice the oracle's own shift under fp16-rounded weights (printed beside it).
Every test prints its worst measured error against its bound.
"""
import collections
import math
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_roi_heads import IMAGE, PYRAMIDS, axis_taps, boundary_sweep, level_scale, level_sets, mixed_rois, \
    roi_geometry
from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200 import ops as G
from stereo_rcnn_b200 import train as TR
from stereo_rcnn_b200.synth import synth_pair, synth_train_gt

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
SENT32 = 0x7FA5A5A5
GUARD = 131
MODEL_TOL = 5e-3


# ------------------------------------------------------------------------------------------------------ mirror
def tap_count(sources):
    return sum(g.shape[0] * (g.shape[1] + 1) ** 2 for g, _, _, _ in sources)


def exponent(sources, C):
    """the kernel's fixed-point exponent e (None when every gradient is zero)"""
    m = max([float(g[..., c:c + C].abs().max()) if g.numel() else 0.0 for g, _, c, _ in sources])
    if m == 0.0:
        return None
    _, ex = math.frexp(m)                                    # m < 2^ex
    return 60 - ex - (tap_count(sources) - 1).bit_length()


def probe_levels(shapes, N, im_h, rois, P, boff):
    """the level the forward reads each RoI from (0..3), or -1 when every tap of the RoI is a zero tap"""
    probe = []
    for l, (h, w) in enumerate(shapes):
        f = torch.zeros(N, h, w, 4, device="cuda")
        f[..., l] = 1.0
        probe.append(f[boff:])
    r = torch.from_numpy(rois).cuda()
    out = G.roi_align_pyramid_nhwc(probe, im_h, r, P).double().sum((1, 2)).cpu()
    lv = out.argmax(1).numpy()
    return np.where(out.sum(1).numpy() > 0, lv, -1)


def mirror(shapes, N, C, im_h, sources, dp_in, chunk=1 << 21, e=None):
    """sources as ops.roi_align_pyramid_backward's; dp_in: 4 fp32 CPU tensors; e: the call's exponent when `sources`
    is only part of the call.
    -> dict(fixed: 4 fp32 [N,h,w,C] (the kernel's bits), exact: 4 float64 (dP + exact sum), n, S: per element, e)"""
    npix = [N * h * w for h, w in shapes]
    poff = np.concatenate([[0], np.cumsum(npix)])
    P_tot = int(poff[-1])
    acc = torch.zeros(P_tot, C, dtype=torch.int64)
    ex = torch.zeros(P_tot, C, dtype=torch.float64)
    S = torch.zeros(P_tot, C, dtype=torch.float64)
    cnt = torch.zeros(P_tot, dtype=torch.int64)
    e = exponent(sources, C) if e is None else e
    sc = 2.0 ** (e - 2) if e is not None else 0.0
    for g, rois_t, coff, boff in sources:
        R, P = g.shape[0], g.shape[1]
        if R == 0:
            continue
        L = P + 1
        rois = rois_t.cpu().numpy()
        lv = probe_levels(shapes, N, im_h, rois, P, boff)
        gs = g[..., coff:coff + C].double().cpu()
        step = max(1, chunk // (L * L * C))
        for r0 in range(0, R, step):
            sl = slice(r0, min(R, r0 + step))
            gp = torch.zeros(sl.stop - sl.start, P + 2, P + 2, C, dtype=torch.float64)
            gp[:, 1:P + 1, 1:P + 1] = gs[sl]
            a, b, c, d = gp[:, :-1, :-1], gp[:, :-1, 1:], gp[:, 1:, :-1], gp[:, 1:, 1:]
            gsum = (a + b) + (c + d)                             # [r, L, L, C]
            gabs = (a.abs() + b.abs()) + (c.abs() + d.abs())
            for l, (H, W) in enumerate(shapes):
                sel = np.nonzero(lv[sl] == l)[0]
                if sel.size == 0:
                    continue
                rr = rois[sl][sel]
                sw, sh, bw, bh = roi_geometry(rr, level_scale(H, im_h), L)
                _, h0, hr, hz = axis_taps(sh, bh, L, H)
                _, w0, wr, wz = axis_taps(sw, bw, L, W)
                img = rr[:, 0].astype(np.int64) + boff
                valid = ~(hz[:, :, None] | wz[:, None, :]) & ((img >= 0) & (img < N))[:, None, None]
                base = poff[l] + (img[:, None, None] * H + h0[:, :, None]) * W + w0[:, None, :]
                hr3, wr3 = hr[:, :, None], wr[:, None, :]
                vi = torch.from_numpy(valid.reshape(-1))
                gv = gsum[torch.from_numpy(sel)].reshape(-1, C)[vi]
                ga = gabs[torch.from_numpy(sel)].reshape(-1, C)[vi]
                for dofs, wt in ((0, (1. - hr3) * (1. - wr3)), (1, (1. - hr3) * wr3), (W, hr3 * (1. - wr3)),
                                 (W + 1, hr3 * wr3)):
                    idx = torch.from_numpy((base + dofs).reshape(-1)[valid.reshape(-1)])
                    w_ = torch.from_numpy(np.ascontiguousarray(wt).reshape(-1)[valid.reshape(-1)])[:, None]
                    acc.index_add_(0, idx, torch.round((gv * sc) * w_).long())
                    ex.index_add_(0, idx, gv * 0.25 * w_)
                    S.index_add_(0, idx, ga * 0.25 * w_.abs())
                    cnt.index_add_(0, idx, torch.ones(idx.numel(), dtype=torch.int64))
    out = dict(fixed=[], exact=[], n=[], S=[], e=e)
    for l, (h, w) in enumerate(shapes):
        sl = slice(int(poff[l]), int(poff[l + 1]))
        d0 = dp_in[l].double()
        if e is None:
            out["fixed"].append(dp_in[l].clone())
        else:
            out["fixed"].append((acc[sl].view(N, h, w, C).double() * 2.0 ** -e + d0).float())
        out["exact"].append(ex[sl].view(N, h, w, C) + d0)
        out["n"].append(cnt[sl].view(N, h, w, 1).double())
        out["S"].append(S[sl].view(N, h, w, C))
    return out


# ------------------------------------------------------------------------------------------------ device calls
def guarded_levels(shapes, N, C, init):
    """level gradients inside NaN-sentinel buffers, initialised to `init` (4 CPU tensors)"""
    bufs, views = [], []
    for (h, w), x in zip(shapes, init):
        n = N * h * w * C
        buf = torch.full((GUARD + n + GUARD,), SENT32, dtype=torch.int32, device="cuda")
        v = buf[GUARD:GUARD + n].view(torch.float32).view(N, h, w, C)
        v.copy_(x)
        bufs.append(buf)
        views.append(v)
    return bufs, views


def check_guards(bufs):
    for b in bufs:
        assert bool((b[:GUARD] == SENT32).all()) and bool((b[-GUARD:] == SENT32).all()), "written outside dP"


def run_backward(shapes, N, C, im_h, sources, init, nonfinite=None):
    bufs, views = guarded_levels(shapes, N, C, init)
    G.roi_align_pyramid_backward(views, im_h, sources, nonfinite=nonfinite)
    torch.cuda.synchronize()
    check_guards(bufs)
    return [v.cpu() for v in views]


def bits(t):
    return t.contiguous().view(torch.int32)


# ------------------------------------------------------------------------------------------------------- cases
def tiny_rois(R, pyr, seed):
    """RoIs of zero to one pixel at a handful of spots: every tap of a RoI in one bilinear cell, hundreds of taps per
    pixel"""
    im_h, im_w = IMAGE[pyr]
    rs = np.random.RandomState(seed)
    spots = np.stack([rs.uniform(0, im_w - 2, 4), rs.uniform(0, im_h - 2, 4)], 1)
    s = spots[rs.randint(0, 4, R)]
    wh = rs.uniform(0, 1, (R, 2)) * (rs.rand(R, 1) < 0.7)
    return np.concatenate([rs.randint(0, 2, (R, 1)), s, s + wh], 1).astype(F32)


# a source: (P, R, family, grad ld / coff ("dense" | "slice" | "box_l" | "box_r"), batch offset in units of B, scale)
Src = collections.namedtuple("Src", "P R fam lay side scale")
Case = collections.namedtuple("Case", "id pyr C B srcs dp")
CASES = [Case(*c) for c in (
    ("small-c4-p1", "small", 4, 2, (Src(1, 300, "mixed", "dense", 0, 1.0),), "zero"),
    ("small-c12-p2-right", "small", 12, 2, (Src(2, 300, "mixed", "slice", 1, 1.0),), "rand"),
    ("bench-c64-p7-two", "bench", 64, 2, (Src(7, 200, "mixed", "dense", 0, 1.0), Src(7, 200, "mixed", "slice", 1, 1.0)),
     "zero"),
    ("bench-c12-p8", "bench", 12, 2, (Src(8, 300, "mixed", "slice", 1, 1.0),), "rand"),
    ("small-c64-p9", "small", 64, 2, (Src(9, 200, "mixed", "dense", 0, 1.0),), "zero"),
    ("small-c512-p15", "small", 512, 2, (Src(15, 16, "mixed", "slice", 1, 1.0),), "rand"),
    ("bench-c4-p2-sweep", "bench", 4, 1, (Src(2, 18003, "sweep", "slice", 0, 1.0),), "zero"),
    ("bench-c256-engine", "bench", 256, 1, (Src(7, 128, "mixed", "box_l", 0, 1.0), Src(7, 128, "mixed", "box_r", 1, 1.0),
                                             Src(14, 128, "mixed", "dense", 0, 1.0)), "rand"),
    ("small-c12-p14-tiny", "small", 12, 2, (Src(14, 400, "tiny", "dense", 0, 1.0),), "zero"),
    ("small-c12-empty-source", "small", 12, 2, (Src(7, 0, "mixed", "dense", 0, 1.0), Src(7, 100, "mixed", "dense", 1, 1.0)),
     "rand"),
    # one source of gradients 2^-30 below the other's: there the quantum 2^-e shows in the fp32 bits
    ("small-c8-quantum", "small", 8, 2, (Src(14, 300, "tiny", "dense", 0, 1.0), Src(7, 300, "mixed", "dense", 1, 2 ** -30)),
     "zero"),
)]


def case_sources(c, dev="cuda", perm=False):
    """-> [(grad, rois, coff, boff)], with the RoIs of each source permuted (and their gradient rows) when perm"""
    seed = zlib.crc32(c.id.encode())
    gen = torch.Generator(device=dev).manual_seed(seed & 0x7FFFFFFF)
    out = []
    box = None
    for i, s in enumerate(c.srcs):
        if s.fam == "sweep":
            rois = np.concatenate([boundary_sweep(k) for k in range(3)])
        elif s.fam == "tiny":
            rois = tiny_rois(s.R, c.pyr, seed + i)
        else:
            rois = mixed_rois(s.R, c.pyr, seed + i) if s.R else np.zeros((0, 5), F32)
        rois[:, 0] = np.minimum(rois[:, 0], c.B - 1)
        if s.lay in ("box_l", "box_r"):                      # one [R,7,7,512] tensor, two slices
            if box is None:
                box = torch.randn(s.R, s.P, s.P, 2 * c.C, generator=gen, device=dev) * s.scale
            g, coff = box, 0 if s.lay == "box_l" else c.C
        else:
            ld = c.C + 8 if s.lay == "slice" else c.C
            g = torch.randn(rois.shape[0], s.P, s.P, ld, generator=gen, device=dev) * s.scale
            coff = 4 if s.lay == "slice" else 0
        r = torch.from_numpy(rois).to(dev)
        if perm and rois.shape[0]:
            p = torch.from_numpy(np.random.RandomState(i).permutation(rois.shape[0])).to(dev)
            g, r = g[p].contiguous(), r[p].contiguous()
        out.append((g, r, coff, s.side * c.B))
    return out


def case_init(c, shapes, N):
    gen = torch.Generator().manual_seed(zlib.crc32(c.id.encode()) & 0x7FFFFFFF)
    return [torch.randn(N, h, w, c.C, generator=gen) if c.dp == "rand" else torch.zeros(N, h, w, c.C)
            for h, w in shapes]


# ------------------------------------------------------------------------------------------------ 1. vs float64
@pytest.mark.parametrize("c", CASES, ids=[c.id for c in CASES])
def test_backward_vs_mirror(c, capsys):
    shapes, N, im_h = PYRAMIDS[c.pyr], 2 * c.B, IMAGE[c.pyr][0]
    srcs = case_sources(c)
    init = case_init(c, shapes, N)
    nf = torch.zeros(1, dtype=torch.int32, device="cuda")
    got = run_backward(shapes, N, c.C, im_h, srcs, init, nonfinite=nf)
    assert int(nf.item()) == 0
    m = mirror(shapes, N, c.C, im_h, srcs, init)
    q = 2.0 ** -m["e"]
    worst, differ, ncmax = 0.0, 0, 0
    for l in range(4):
        g = got[l]
        differ += int((bits(g) != bits(m["fixed"][l])).sum())
        ulp = (torch.nextafter(g.abs(), torch.tensor(math.inf)) - g.abs()).double()
        bound = q * m["n"][l] + 2.0 ** -40 * (m["S"][l] + init[l].double().abs()) + ulp / 2
        err = (g.double() - m["exact"][l]).abs()
        worst = max(worst, float((err / bound).max()))
        ncmax = max(ncmax, int(m["n"][l].max()))
    with capsys.disabled():
        print("%-26s e=%d taps=%d max contributions/element=%d  err/bound %.3e  bits differing from the "
              "fixed-point mirror %d" % (c.id, m["e"], tap_count(srcs), ncmax, worst, differ))
    assert worst <= 1.0
    assert differ == 0
    if c.id.endswith("tiny"):
        assert ncmax >= 200                                  # hundreds of taps on one pixel
    # determinism: a second call, and the RoIs of every source permuted with their gradient rows
    again = run_backward(shapes, N, c.C, im_h, srcs, init)
    permuted = run_backward(shapes, N, c.C, im_h, case_sources(c, perm=True), init)
    for l in range(4):
        assert torch.equal(bits(again[l]), bits(got[l])), "a repeated call differs"
        assert torch.equal(bits(permuted[l]), bits(got[l])), "permuting the RoIs changes the result"


def test_exponent_at_the_largest_tap_count(capsys):
    """T = 2^24 lattice taps in one call (65536 RoIs at P = 15, k = 24): the exponent still follows e = 60 - ex - k bit
    for bit.  A second source 2^-36 below the largest gradient writes its own image, where the quantum 2^-e reaches the
    fp32 result: the mirror at e matches it bit for bit, the mirror at e + 1 or e - 1 does not"""
    shapes, N, im_h, C = PYRAMIDS["small"], 2, IMAGE["small"][0], 4
    gen = torch.Generator(device="cuda").manual_seed(3)
    big = tiny_rois(65536 - 64, "small", 5)
    big[:, 0] = 0
    small = mixed_rois(64, "small", 6)
    small[:, 0] = 0
    srcs = [(torch.randn(big.shape[0], 15, 15, C, generator=gen, device="cuda"), torch.from_numpy(big).cuda(), 0, 0),
            (torch.randn(64, 15, 15, C, generator=gen, device="cuda") * 2.0 ** -36, torch.from_numpy(small).cuda(), 0,
             1)]
    assert tap_count(srcs) == 2 ** 24
    init = [torch.zeros(N, h, w, C) for h, w in shapes]
    got = run_backward(shapes, N, C, im_h, srcs, init)
    e = exponent(srcs, C)
    differ = {}
    for de in (-1, 0, 1):
        m = mirror(shapes, N, C, im_h, srcs[1:], init, e=e + de)
        differ[de] = sum(int((bits(got[l][1]) != bits(m["fixed"][l][1])).sum()) for l in range(4))
    assert all(bool(torch.isfinite(g).all()) for g in got)
    with capsys.disabled():
        print("largest tap count: T=2^24 e=%d; bits of the small source's image differing from the mirror at "
              "e-1, e, e+1: %s" % (e, [differ[d] for d in (-1, 0, 1)]))
    assert differ[0] == 0 and differ[1] > 0 and differ[-1] > 0


# ------------------------------------------------------------------------------------- 2. adjoint of the forward
def test_adjoint_identity_roi_by_roi(capsys):
    shapes, im_h, C, B = PYRAMIDS["bench"], IMAGE["bench"][0], 4, 1
    N = 2 * B
    rois = np.concatenate([boundary_sweep(k) for k in range(3)] + [mixed_rois(600, "bench", 21)])
    rois[:, 0] = 0
    lo, hi, _ = level_sets(rois)
    amb = np.nonzero(lo != hi)[0]
    pick = np.concatenate([amb[:40], rois.shape[0] - 600 + np.random.RandomState(2).choice(600, 40, replace=False)])
    gen = torch.Generator(device="cuda").manual_seed(8)
    F = [torch.randn(N, h, w, C, generator=gen, device="cuda") for h, w in shapes]
    Fa = [f.double().abs().cpu() for f in F]
    worst, n_amb = 0.0, 0
    for i in pick:
        for P, side in ((7, 1), (14, 0)):
            r = torch.from_numpy(rois[i:i + 1]).cuda()
            g = torch.randn(1, P, P, C, generator=gen, device="cuda")
            fwd = G.roi_align_pyramid_nhwc([f[side * B:] for f in F], im_h, r, P)
            lhs = float((fwd.double() * g.double()).sum())
            zero = [torch.zeros(N, h, w, C) for h, w in shapes]
            srcs = [(g, r, 0, side * B)]
            d = run_backward(shapes, N, C, im_h, srcs, zero)
            rhs = sum(float((f.double().cpu() * x.double()).sum()) for f, x in zip(F, d))
            m = mirror(shapes, N, C, im_h, srcs, zero)
            q =2.0 ** -m["e"] if m["e"] is not None else 0.0
            tol = sum(float((fa * (2.0 ** -20 * s + q * n)).sum()) for fa, s, n in zip(Fa, m["S"], m["n"]))
            assert abs(lhs - rhs) <= tol, (i, P, lhs, rhs, tol)
            worst = max(worst, abs(lhs - rhs) / tol if tol else 0.0)
        n_amb += int(lo[i] != hi[i])
    with capsys.disabled():
        print("adjoint identity: %d RoIs (%d ambiguous) x P in (7, 14): worst err/bound %.3e" % (len(pick), n_amb, worst))
    assert n_amb == amb.size >= 10


# ----------------------------------------------------------------------------------- 4. flags and degenerate calls
def test_nonfinite_flag_from_any_source_and_never_cleared():
    c = CASES[7]                                             # the engine layout: three sources
    shapes, N, im_h = PYRAMIDS[c.pyr], 2 * c.B, IMAGE[c.pyr][0]
    init = [torch.zeros(N, h, w, c.C) for h, w in shapes]
    for k in range(3):
        srcs = case_sources(c)
        g = srcs[k][0].clone()
        g[3, 1, 2, srcs[k][2] + 5] = float("inf")
        srcs[k] = (g,) + srcs[k][1:]
        nf = torch.zeros(1, dtype=torch.int32, device="cuda")
        got = run_backward(shapes, N, c.C, im_h, srcs, init, nonfinite=nf)
        assert int(nf.item()) == 1, k
        assert all(bool(torch.isnan(x).all()) for x in got), k
    nf = torch.ones(1, dtype=torch.int32, device="cuda")
    run_backward(shapes, N, c.C, im_h, case_sources(c), init, nonfinite=nf)
    assert int(nf.item()) == 1, "a set flag was cleared"
    print("an Inf in each of the three sources sets the flag; a set flag stays set")


def test_no_rois_leaves_dp_untouched_without_a_launch():
    shapes, N, C = PYRAMIDS["small"], 2, 8
    init = [torch.randn(N, h, w, C) for h, w in shapes]
    bufs, views = guarded_levels(shapes, N, C, init)
    torch.cuda.synchronize()
    n0 = G.launch_count()
    G.roi_align_pyramid_backward(views, 160.0, [(torch.zeros(0, 7, 7, C, device="cuda"),
                                                 torch.zeros(0, 5, device="cuda"), 0, 0)] * 3)
    torch.cuda.synchronize()
    assert G.launch_count() == n0
    check_guards(bufs)
    assert all(torch.equal(bits(v.cpu()), bits(x)) for v, x in zip(views, init))
    # all-zero gradients: dP unchanged bit for bit
    rois = torch.from_numpy(mixed_rois(50, "small", 1)).cuda()
    G.roi_align_pyramid_backward(views, 160.0, [(torch.zeros(50, 7, 7, C, device="cuda"), rois, 0, 0)])
    torch.cuda.synchronize()
    assert all(torch.equal(bits(v.cpu()), bits(x)) for v, x in zip(views, init))


# ------------------------------------------------------------------------------------- 5-7. the full training loss
def _small_hw():
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "forward_small.npz"))
    return int(g["H"]), int(g["W"])


def _words(shape, seed):
    w = np.random.RandomState(seed).randint(0, 2 ** 32, shape, dtype=np.uint64).astype(np.uint32)
    return torch.from_numpy(w.view(np.int32)).cuda()


@pytest.fixture(scope="module")
def step_case():
    from oracle import model as OM
    H, W = _small_hw()
    B = 1
    eng = E.StereoRCNNEngine(OM.make_state_dict(3), "cuda", precision="fp16")
    p = synth_pair(H, W, 7, 12)
    iml, imr = [torch.from_numpy(x[None]).cuda().contiguous() for x in p[:2]]
    gt = [torch.from_numpy(t).cuda() for t in synth_train_gt(B, 30, H, W, 7)[:5]]
    shapes = [[-(-H // s), -(-W // s)] for s in (4, 8, 16, 32, 64)]
    rpn_keys = _words((B, 3 * sum(h * w for h, w in shapes)), 8)
    keys = _words((B, 2030), 9)
    words = _words((B, 512), 10)
    dw = _words((2, 512, 2048), 11)
    return eng, iml, imr, gt, keys, words, rpn_keys, dw


def _run(sc, **kw):
    eng, iml, imr, gt, keys, words, rpn_keys, dw = sc
    r = TR.loss_gradients(eng, iml, imr, *gt, keys, words, rpn_keys, dropout_words=dw, **kw)
    out = (r[0].clone(), {k: v.clone() for k, v in r[1].items()}) + tuple(x.clone() for x in r[2:])
    torch.cuda.synchronize()
    return out + (int(eng.found_inf.item()),)


def test_loss_gradients_match_the_merged_chains(step_case, capsys):
    eng, iml, imr, gt, keys, words, rpn_keys, dw = step_case
    gs = 2.0 ** 12
    losses, got, fi = _run(step_case, grad_scale=gs)
    assert fi == 0
    names = [n for n, _ in E.trainable_trunk_fpn_params(1) + E.trainable_rpn_params() + E.trainable_rcnn_head_params()]
    assert sorted(got) == sorted(names) and losses.shape == (6,)
    l_rpn, g_rpn = TR.rpn_gradients(eng, iml, imr, *gt[:3], rpn_keys, grad_scale=gs)
    g_rpn = {k: v.clone() for k, v in g_rpn.items()}
    l_rcnn, g_rcnn, dpool = TR.rcnn_head_gradients(eng, iml, imr, *gt, keys, words, dropout_words=dw, grad_scale=gs)
    torch.cuda.synchronize()
    assert torch.equal(losses[:2], l_rpn) and torch.equal(losses[2:], l_rcnn)
    for n, _ in E.trainable_rpn_params():
        assert torch.equal(got[n], g_rpn[n]), n
    for n in g_rcnn:
        assert torch.equal(got[n], g_rcnn[n]), n
    # the trunk and the FPN: rpn_gradients' chain plus exactly the RoI path
    with torch.no_grad():
        im = torch.cat((iml, imr), 0)
        feats, st = eng.trunk_fpn(im, save_for_backward=True)
        cp, bbox, shapes, sr, score = eng.rpn(feats, 1, save_for_backward=True)
        lab = TR.anchor_targets(TR.generate_anchors(shapes, "cuda"), *gt[:3], tuple(iml.shape[2:]), rpn_keys)
        _, dc, db = TR.rpn_loss(score, bbox, *lab)
        _, dp = eng.rpn_backward(sr, dc, db, grad_scale=gs)
        rl, rr = G.proposal_layer(cp, bbox, TR._im_info(1, *iml.shape[2:], "cuda"), "TRAIN", shapes)
        tgt = TR.proposal_targets(rl, rr, gt[0], gt[1], gt[3], gt[4], keys, words)
        _, sh = eng.heads(feats, 1, tgt["rois_left"].view(-1, 5), tgt["rois_right"].view(-1, 5), float(iml.shape[2]),
                          save_for_backward=True, dropout_words=dw)
        eng.roi_align_backward(sh, dpool, dp)
        manual = eng.trunk_fpn_backward(st, dp, grad_scale=gs)
    torch.cuda.synchronize()
    rel = {}
    for n, _ in E.trainable_trunk_fpn_params(1):
        assert torch.equal(got[n], manual[n]), n
        rel[n] = float((got[n] - g_rpn[n]).double().norm() / g_rpn[n].double().norm())
    with capsys.disabled():
        print("loss_gradients vs the merged chains: RPN and heads bit-identical; trunk/FPN = rpn_gradients + the RoI "
              "path bit for bit; relative change from the RoI path: FPN %s, trunk max %.2e" % (
                  {k: "%.2e" % v for k, v in rel.items() if k.startswith("RCNN_smooth")},
                  max(v for k, v in rel.items() if k.startswith("RCNN_layer"))))
    assert all(rel[n] > 0 for n in rel if n.startswith(("RCNN_smooth", "RCNN_latlayer", "RCNN_toplayer")))


def test_loss_gradients_buffers_and_graph_capture(step_case):
    eng, iml, imr, gt, keys, words, rpn_keys, dw = step_case
    l0, a, fi = _run(step_case)
    assert fi == 0
    names = E.trainable_trunk_fpn_params(1) + E.trainable_rpn_params() + E.trainable_rcnn_head_params()
    bufs = {n: torch.full(s, float("nan"), device="cuda") for n, s in names}
    l1, b = TR.loss_gradients(eng, iml, imr, *gt, keys, words, rpn_keys, dropout_words=dw, grads=bufs)
    torch.cuda.synchronize()
    assert torch.equal(l0, l1)
    for n in a:
        assert b[n].data_ptr() == bufs[n].data_ptr(), n
        assert torch.equal(bufs[n], a[n]), n

    def step(x, y):
        return TR.loss_gradients(eng, x, y, *gt, keys, words, rpn_keys, dropout_words=dw)
    with torch.no_grad():
        runner = E.GraphRunner(step, [iml, imr])
        lg, out = runner()
        torch.cuda.synchronize()
    assert torch.equal(lg, l0)
    for n in a:
        assert torch.equal(out[n], a[n]), n


def test_loss_gradients_scaling_overflow_and_uncert(step_case, capsys):
    base_l, base, fi = _run(step_case)
    assert fi == 0
    # uncert = 14 everywhere: every gradient times exp(-14) ~ 8e-7; grad_scale 2^20 keeps the fp16 chains in range
    u14 = torch.full((6,), 14.0, device="cuda")
    lt, tiny, du, fi = _run(step_case, uncert=u14, grad_scale=2.0 ** 20)
    assert fi == 0 and torch.equal(lt, base_l)
    f = math.exp(-14.0)
    errs = {n: float((tiny[n].double() - base[n].double() * f).norm() / (base[n].double() * f).norm()) for n in base
            if float(base[n].abs().max()) > 0}
    worst = max(errs.items(), key=lambda kv: kv[1])
    with capsys.disabled():
        print("uncert 14, grad_scale 2^20 vs unscaled x exp(-14): worst %s %.2e" % worst)
    tol = lambda n: 1e-1 if n.startswith(("RCNN_layer", "RCNN_kpts")) else MODEL_TOL
    assert all(e < tol(n) for n, e in errs.items()), {n: e for n, e in errs.items() if e >= tol(n)}
    _, _, fi = _run(step_case, grad_scale=2.0 ** 40)
    assert fi == 1
    _, _, fi = _run(step_case)
    assert fi == 0
    # d total / d uncert = 1 - L exp(-u) for all six terms
    u = torch.tensor([0.3, -0.2, 0.1, 0.0, 0.5, -0.4], device="cuda")
    l1, _, du, _ = _run(step_case, uncert=u)
    L_, uc = l1.cpu().double().numpy(), u.cpu().double().numpy()
    np.testing.assert_allclose(du.cpu().numpy(), 1 - L_ * np.exp(-uc), rtol=1e-5)


def test_flag_set_by_the_heads_survives_the_chain(step_case):
    """uncert[2:6] = -40 multiplies only the R-CNN loss gradients by e^40: the heads' fp16 chain overflows while the RPN
    part stays finite, and the flag set there is still set when loss_gradients returns.  heads_backward itself keeps a
    flag with clear_found_inf=False and clears it by default"""
    eng = step_case[0]
    u = torch.tensor([0.0, 0.0, -40.0, -40.0, -40.0, -40.0], device="cuda")
    _, _, _, fi = _run(step_case, uncert=u, grad_scale=2.0 ** 8)
    assert fi == 1
    _, _, fi = _run(step_case)
    assert fi == 0
    _, iml, imr, gt, keys, words, _, _ = step_case
    with torch.no_grad():
        feats = eng.trunk_fpn(torch.cat((iml, imr), 0))
        cp, bb, shapes = eng.rpn(feats, 1)
        rl, rr = G.proposal_layer(cp, bb, TR._im_info(1, *iml.shape[2:], "cuda"), "TRAIN", shapes)
        tgt = TR.proposal_targets(rl, rr, gt[0], gt[1], gt[3], gt[4], keys, words)
        out, sh = eng.heads(feats, 1, tgt["rois_left"].view(-1, 5), tgt["rois_right"].view(-1, 5), float(iml.shape[2]),
                            save_for_backward=True)
        d = [torch.zeros_like(out[k]) for k in ("cls_score", "bbox_pred", "dim_orien_pred", "kpts_pred",
                                                "left_border_pred", "right_border_pred")]
        eng.found_inf.fill_(1)
        eng.heads_backward(sh, *d, clear_found_inf=False)
        kept = int(eng.found_inf.item())
        eng.heads_backward(sh, *d)
        cleared = int(eng.found_inf.item())
    assert kept == 1 and cleared == 0


# ------------------------------------------------------------------------ 6. end to end against fp32 autograd
LOSS_TOL = 1e-3
DEEP_TOL = 1e-1        # the trunk and the keypoint chain (DESIGN 6: fp16 forward rounding and ReLU-mask flips)
# the FPN now also receives the R-CNN losses' pooled gradients, which carry the keypoint chain's fp16 error (DESIGN 6):
# looser than the RPN-only 5e-3, and held to twice the oracle's own shift under fp16-rounded weights, which the test
# measures and prints beside it
FPN_TOL = 2e-2
UNCERT = (0.3, -0.2, 0.1, 0.0, 0.5, -0.4)
THR = int(np.ceil(E.DROPOUT_P * 2.0 ** 32))


class _LevelRoIAlign(torch.autograd.Function):
    """oracle.ops.roi_align_forward / roi_align_backward on one NCHW level at an L x L lattice (CPU C kernels)"""

    @staticmethod
    def forward(ctx, feat, rois, L, scale):
        from oracle import ops as O
        ctx.rois, ctx.shape, ctx.L, ctx.scale, ctx.dev = rois, tuple(feat.shape), L, scale, feat.device
        return torch.from_numpy(O.roi_align_forward(feat.detach().cpu().numpy(), rois, L, L, scale)).to(feat.device)

    @staticmethod
    def backward(ctx, g):
        from oracle import ops as O
        d = O.roi_align_backward(g.detach().cpu().numpy(), ctx.rois, ctx.shape, ctx.L, ctx.L, ctx.scale)
        return torch.from_numpy(d).to(ctx.dev), None, None, None


def _pyramid_roi_feat(feats, rois, im_h, P):
    """differentiable PyramidRoI_Feat (stereo_rcnn.py:110-139) as oracle.ops.pyramid_roi_feat: feats = NCHW P2..P5,
    rois [R,5] numpy -> [R,C,P,P]"""
    from oracle import ops as O
    lv = O.roi_levels(rois)
    parts, order = [], []
    for i in range(4):
        idx = np.nonzero(lv == i + 2)[0]
        if idx.size == 0:
            continue
        scale = np.float32(feats[i].shape[2] / float(im_h))
        x = _LevelRoIAlign.apply(feats[i], np.ascontiguousarray(rois[idx]), P + 1, scale)
        parts.append(((x[..., :-1, :-1] + x[..., :-1, 1:]) + (x[..., 1:, :-1] + x[..., 1:, 1:])) * 0.25)
        order.append(idx)
    inv = torch.from_numpy(np.argsort(np.concatenate(order))).to(feats[0].device)
    return torch.cat(parts, 0)[inv]


def _oracle_loss(sd, im, B, rpn_tgt, tgt, words, names, fixed_uncert, weights16=False):
    """fp32 autograd (TF32 off) of the six-term loss: oracle.model.trunk_fpn -> rpn_head -> the pyramid RoIAlign above
    on the engine's sampled RoIs -> the train-mode heads of test_gpu_rcnn_backward (the engine's dropout masks) ->
    rpn_losses + rcnn_losses.  -> (losses [6], {name: grad}, d total / d uncert or None)"""
    from oracle import model as OM
    from oracle import train_targets as T
    dev = "cuda"
    sdd = {k: v.to(dev) for k, v in sd.items()}
    if weights16:
        sdd = {k: (v.half().float() if k.endswith("weight") and v.dim() >= 2 else v) for k, v in sdd.items()}
    for n in names:
        sdd[n] = sdd[n].clone().requires_grad_(True)
    u = torch.tensor(fixed_uncert, dtype=torch.float32, requires_grad=True) if fixed_uncert else None
    H = im.shape[2]
    rl, rr = tgt["rois_left"].reshape(-1, 5).numpy(), tgt["rois_right"].reshape(-1, 5).numpy()
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.enable_grad():
            f = OM.trunk_fpn(im.to(dev), sdd)
            lvl = ("p2", "p3", "p4", "p5", "p6")
            _, bbox_r, _, score = OM.rpn_head([f[k][:B] for k in lvl], [f[k][B:] for k in lvl], sdd)
            lc, lb = T.rpn_losses(score.cpu(), bbox_r.cpu(), *[t.cpu() for t in rpn_tgt])
            left, right = [f[k][:B] for k in lvl[:4]], [f[k][B:] for k in lvl[:4]]
            pb = torch.cat([_pyramid_roi_feat(left, rl, H, 7), _pyramid_roi_feat(right, rr, H, 7)], 1)
            pk = _pyramid_roi_feat(left, rl, H, 14)
            R = pb.shape[0]
            w = words.cpu().numpy().view(np.uint32).astype(np.int64) >= THR
            keep = [torch.from_numpy(w[i]).float().to(dev).view(R, 2048, 1, 1) * 1.25 for i in range(2)]
            x = F.relu(F.conv2d(pb, sdd["RCNN_top.0.weight"], sdd["RCNN_top.0.bias"], stride=7)) * keep[0]
            x = F.relu(F.conv2d(x, sdd["RCNN_top.3.weight"], sdd["RCNN_top.3.bias"])) * keep[1]
            fc7 = x.mean(3).mean(2)
            cls = F.linear(fc7, sdd["RCNN_cls_score.weight"], sdd["RCNN_cls_score.bias"])
            bbox = F.linear(fc7, sdd["RCNN_bbox_pred.weight"], sdd["RCNN_bbox_pred.bias"])
            dim = F.linear(fc7, sdd["RCNN_dim_orien_pred.weight"], sdd["RCNN_dim_orien_pred.bias"])
            y = pk
            for k in range(0, 12, 2):
                y = F.relu(F.conv2d(y, sdd["RCNN_kpts.%d.weight" % k], sdd["RCNN_kpts.%d.bias" % k], padding=1))
            y = F.relu(F.conv_transpose2d(y, sdd["RCNN_kpts.12.weight"], sdd["RCNN_kpts.12.bias"], stride=2))
            ka = F.conv2d(y, sdd["kpts_class.weight"], sdd["kpts_class.bias"]).sum(2)
            g = ka.shape[2]
            losses = [lc, lb] + list(T.rcnn_losses(cls.cpu(), bbox.cpu(), dim.cpu(), ka[:, :4].reshape(-1, 4 * g).cpu(),
                                                   ka[:, 4].cpu(), ka[:, 5].cpu(), tgt))
            if u is None:
                total = sum(losses)
            else:
                total = sum(l * torch.exp(-u[i]) + u[i] for i, l in enumerate(losses))
            leaves = [sdd[n] for n in names] + ([u] if u is not None else [])
            gr = torch.autograd.grad(total, leaves)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    ref = {n: t.detach().cpu() for n, t in zip(names, gr)}
    return [float(l.detach()) for l in losses], ref, (gr[-1].detach() if u is not None else None)


def _oracle_tol(n):
    if n.startswith(("RCNN_layer", "RCNN_kpts.")):
        return DEEP_TOL
    if n.startswith(("RCNN_smooth", "RCNN_latlayer", "RCNN_toplayer")):
        return FPN_TOL
    return MODEL_TOL


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / max(float(b.norm()), 1e-300))


OCASES = [(160, 256, 1, 0, True), (160, 256, 1, 1, False), (160, 256, 2, 0, False), (160, 256, 2, 1, True),
          (600, 1987, 1, 1, True)]


@pytest.mark.parametrize("H,W,B,fb,use_u", OCASES, ids=["%dx%d-b%d-fb%d%s" % (c[:4] + ("-uncert" if c[4] else "",))
                                                         for c in OCASES])
def test_loss_gradients_vs_oracle(H, W, B, fb, use_u, capsys):
    from oracle import model as OM
    if (H, W) == (160, 256):
        H, W = _small_hw()
    sd = OM.make_state_dict(3)
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    seed = 7 + B + fb
    ps = [synth_pair(H, W, seed + b, 12) for b in range(B)]
    im = torch.from_numpy(np.stack([p[0] for p in ps] + [p[1] for p in ps], 0)).contiguous().cuda()
    gl, gr, gm, dim, kp, _ = [torch.from_numpy(t).cuda() for t in synth_train_gt(B, 30, H, W, seed)]
    shapes = [[-(-H // s), -(-W // s)] for s in (4, 8, 16, 32, 64)]
    rpn_keys = _words((B, 3 * sum(h * w for h, w in shapes)), seed + 1)
    keys, words = _words((B, 2030), seed + 2), _words((B, 512), seed + 3)
    dw = _words((2, B * 512, 2048), seed + 4)
    u = torch.tensor(UNCERT, device="cuda") if use_u else None
    r = TR.loss_gradients(eng, im[:B], im[B:], gl, gr, gm, dim, kp, keys, words, rpn_keys, dropout_words=dw, uncert=u,
                          fixed_blocks=fb, grad_scale=2.0 ** 12)
    torch.cuda.synchronize()
    assert int(eng.found_inf.item()) == 0
    losses, got = r[0].cpu().tolist(), {k: v.cpu() for k, v in r[1].items()}
    # the targets and sampled RoIs the engine used, for the oracle
    with torch.no_grad():
        feats = eng.trunk_fpn(torch.cat((im[:B], im[B:]), 0))
        cp, bb, shp = eng.rpn(feats, B)
        rpn_tgt = TR.anchor_targets(TR.generate_anchors(shp, "cuda"), gl, gr, gm, (H, W), rpn_keys)
        rl, rr = G.proposal_layer(cp, bb, TR._im_info(B, H, W, "cuda"), "TRAIN", shp)
        tgt = {k: v.cpu() for k, v in TR.proposal_targets(rl, rr, gl, gr, dim, kp, keys, words).items()}
    du = r[2].cpu().double() if use_u else None
    del eng, feats, r
    torch.cuda.empty_cache()
    names = [n for n, _ in E.trainable_trunk_fpn_params(fb) + E.trainable_rpn_params() + E.trainable_rcnn_head_params()]
    assert sorted(got) == sorted(names)
    ol, ref, odu = _oracle_loss(sd, im.cpu(), B, rpn_tgt, tgt, dw, names, UNCERT if use_u else None)
    _, ref16, _ = _oracle_loss(sd, im.cpu(), B, rpn_tgt, tgt, dw, names, UNCERT if use_u else None, weights16=True)
    label = "%dx%d B=%d fixed_blocks=%d uncert=%s" % (H, W, B, fb, use_u)
    errs = {n: _rel(got[n], ref[n]) for n in names}
    shift = {n: _rel(ref16[n], ref[n]) for n in names}

    def group(d, pre):
        v = [e for n, e in d.items() if n.startswith(pre)]
        return "%.2e .. %.2e" % (min(v), max(v)) if v else "-"
    groups = (("trunk", "RCNN_layer"), ("FPN", ("RCNN_smooth", "RCNN_latlayer", "RCNN_toplayer")),
              ("RPN", "RCNN_rpn."), ("box head", ("RCNN_top.", "RCNN_cls", "RCNN_bbox", "RCNN_dim")),
              ("kpts convs", "RCNN_kpts."), ("kpts_class", "kpts_class"))
    with capsys.disabled():
        print("\n%s: losses %s vs oracle %s" % (label, ["%.6g" % x for x in losses], ["%.6g" % x for x in ol]))
        for g, pre in groups:
            print("  %-10s relative L2 vs oracle %s   oracle fp16-weights shift %s" % (g, group(errs, pre),
                                                                                        group(shift, pre)))
        if du is not None:
            print("  d total / d uncert %s vs oracle %s" % (du.numpy().round(6).tolist(),
                                                          odu.double().numpy().round(6).tolist()))
    for a, b in zip(losses, ol):
        assert abs(a - b) <= LOSS_TOL * abs(b), (a, b)
    if du is not None:
        Le = np.array(ol) * np.exp(-np.array(UNCERT))
        assert np.all(np.abs(du.numpy() - odu.double().numpy()) <= LOSS_TOL * np.abs(Le) + 1e-6)
    bad = {n: e for n, e in errs.items() if not e < _oracle_tol(n)}
    assert not bad, bad
    fpn = [n for n in names if n.startswith(("RCNN_smooth", "RCNN_latlayer", "RCNN_toplayer"))]
    assert max(errs[n] for n in fpn) <= 2 * max(shift[n] for n in fpn)
