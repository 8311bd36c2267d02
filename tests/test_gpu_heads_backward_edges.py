"""GPU: the R-CNN heads' backward kernels (heads_bwd.cu) at their edges, on the builders of test_heads_backward_edges.py,
and engine.heads_backward at two images per step.

* every kernel case twice (bit-identical runs), every output and workspace inside NaN-sentinel guard bands;
* exact-arithmetic cases bit for bit against float64 (fp16 outputs: the single rounding of the exact value), random
  cases per element against the a-priori bounds of the CPU file;
* sb_dropout_words over its grid-stride pass and at its threshold; sb_kpts_logits across the block tail;
  sb_box_tail_backward over R, K, nc and both scales; sb_kpts_tail_backward over G, C, R and grad_scale with a workspace
  of exactly sb_kpts_tail_backward_workspace bytes; sb_permute3 in all six orders; sb_box_tail_scores against
  sb_box_tail; the non-finite flag from each upstream gradient, from dz16, from dW and from the keypoint reduce alone;
* heads_backward layer by layer against float64 at B = 2 (R = 1024, dropout on and off) and at R = 1 and 129, and the
  per-RoI gradients and saved activations bit-identical under a permutation of the RoIs and for a prefix of them.
Every test prints its worst per-element error / bound per tensor."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import model as OM
from stereo_rcnn_b200 import engine as EN
from stereo_rcnn_b200 import lib as _l
from stereo_rcnn_b200 import ops as G

import test_heads_backward_edges as E
from test_gpu_rcnn_backward import KERNEL_TOL, _heads_backward_ref, _pairs, _small_hw, _words, guarded, l2_err

pytestmark = pytest.mark.gpu
F16, F32 = torch.float16, torch.float32


def vp(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int16 if t.dtype == F16 else torch.int32)


def same(a, b):
    return a.dtype == b.dtype and torch.equal(bits(a), bits(b))


def report(label, ratios):
    print("%s worst error / bound: %s" % (label, ", ".join("%s %.3f" % kv for kv in ratios.items())))
    assert all(r <= 1.0 for r in ratios.values()), ratios


def cuda(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


# ================================================================================================ dropout ====
@pytest.mark.parametrize("half", [True, False])
@pytest.mark.parametrize("p", E.DROP_PS)
@pytest.mark.parametrize("n", E.DROP_NS)
def test_dropout_words(n, p, half):
    x, words = E.dropout_case(n, p, half)
    ref = E.dropout_ref(x, words, p)
    w = torch.from_numpy(words.view(np.int32)).cuda()
    runs = []
    for _ in range(2):
        v, check = guarded((n,), F16 if half else F32)
        v.copy_(torch.from_numpy(x))
        G.dropout_words_(v, w, p)
        torch.cuda.synchronize()
        check()
        runs.append(v.cpu().numpy())
    assert E.same_bits(runs[0], ref)
    assert np.array_equal(runs[0].view(np.uint8), runs[1].view(np.uint8))


def test_dropout_words_empty_launches_nothing():
    L = _l.load()
    torch.cuda.synchronize()
    n0 = G.launch_count()
    assert L.sb_dropout_words(None, 0, 0, None, 0.2, G.stream_ptr()) == 0
    assert G.launch_count() == n0


# ================================================================================================ kpts_logits ====
@pytest.mark.parametrize("Gd", E.LOGIT_GS)
@pytest.mark.parametrize("R", E.LOGIT_RS)
def test_kpts_logits(R, Gd):
    L = _l.load()
    a = E.logits_case(R, Gd)
    ref = [torch.from_numpy(r) for r in E.logits_ref(a)]
    (src,) = cuda(a)
    runs = []
    for _ in range(2):
        outs = [guarded(s, F32) for s in ((R, 4 * Gd), (R, Gd), (R, Gd))]
        assert L.sb_kpts_logits(vp(src), R, Gd, *[vp(o[0]) for o in outs], G.stream_ptr()) == 0
        torch.cuda.synchronize()
        for o in outs:
            o[1]()
        runs.append([o[0].cpu() for o in outs])
    for got, want, name in zip(runs[0], ref, ("kpts_pred", "left", "right")):
        assert same(got, want), name
    assert all(same(a_, b_) for a_, b_ in zip(*runs))


# ================================================================================================ box tail ====
def run_box(ops_np, ms, gs, nf=None):
    """sb_box_tail_backward into guarded outputs -> {dz, dz16, dw [12nc,K], db [12nc]}"""
    L = _l.load()
    d_cls, d_box, d_dim, fc7, w_cls, w_box, w_dim = cuda(*ops_np)
    R, K = fc7.shape
    nc = d_cls.shape[1]
    outs = [guarded(s, F32) for n in (1, 6, 5) for s in ((n * nc, K), (n * nc,))]
    dz16, c16 = guarded((R, K), F16)
    dz32, c32 = guarded((R, K), F32)
    rc = L.sb_box_tail_backward(vp(d_cls), vp(d_box), vp(d_dim), vp(fc7), R, K, nc, vp(w_cls), vp(w_box), vp(w_dim),
                                ms, gs, *[vp(o[0]) for o in outs], vp(dz16), vp(dz32), vp(nf), G.stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    for o in outs:
        o[1]()
    c16()
    c32()
    return {"dz": dz32.clone(), "dz16": dz16.clone(), "dw": torch.cat([outs[i][0] for i in (0, 2, 4)], 0),
            "db": torch.cat([outs[i][0] for i in (1, 3, 5)], 0)}


def _box_twice(ops_np, ms, gs):
    a, b = run_box(ops_np, ms, gs), run_box(ops_np, ms, gs)
    assert all(same(a[k], b[k]) for k in a)
    return a


@pytest.mark.parametrize("case", E.BOX_CASES, ids=lambda c: "R%d-K%d-nc%d-ms%g-gs%g" % c)
def test_box_tail_backward(case):
    R, K, nc, ms, gs = case
    # exact: every fp32 output equals float64, dz16 its single rounding, +0 wherever fc7 <= 0 (-0.0 included)
    ops = E.box_exact(R, K, nc)
    got = _box_twice(ops, ms, gs)
    ref, _ = E.box_ref(*[torch.from_numpy(a).cuda() for a in ops], ms, gs)
    for k in ("dz", "dw", "db"):
        assert torch.equal(got[k].double(), ref[k]), k
    assert same(got["dz16"], ref["dz"].float().half())
    off = torch.from_numpy(ops[3]).cuda() <= 0
    assert bool((bits(got["dz"])[off] == 0).all()) and bool((bits(got["dz16"])[off] == 0).all())
    # random: per element inside the bound
    ops = E.box_random(R, K, nc)
    got = _box_twice(ops, ms, gs)
    ref, bound = E.box_ref(*[torch.from_numpy(a).cuda() for a in ops], ms, gs)
    ratios = {k: E.worst_ratio(got[k], ref[k], bound[k]) for k in ("dz", "dw", "db")}
    ratios["dz16"] = E.worst_ratio(got["dz16"], ref["dz"], E.fp16_bound(ref["dz"], bound["dz"]))
    off = torch.from_numpy(ops[3]).cuda() <= 0
    assert bool((bits(got["dz"])[off] == 0).all()) and bool((bits(got["dz16"])[off] == 0).all())
    report("box_tail_backward R=%d K=%d nc=%d" % (R, K, nc), ratios)


# ================================================================================================ keypoint tail ====
def run_kpts(up, w, dkp, dl, dr, gs, nf=None):
    """sb_kpts_tail_backward through lib with guarded outputs and a guarded workspace of exactly the advertised size
    -> {dup, dw, db, db_up, ws}"""
    L = _l.load()
    R, Gd, _, C = up.shape
    nb = L.sb_kpts_tail_backward_workspace(R, C)
    assert nb == R * (7 * C + 8) * 4
    ws, cw = guarded((nb // 4,), F32)
    dup, cd = guarded((R, Gd // 2, Gd // 2, 4 * C), F16)
    outs = [guarded((n,), F32) for n in (6 * C, 6, C)]
    rc = L.sb_kpts_tail_backward(vp(up), R, Gd, C, vp(w), vp(dkp), vp(dl), vp(dr), gs, vp(dup),
                                 *[vp(o[0]) for o in outs], vp(nf), vp(ws), nb, G.stream_ptr())
    assert rc == 0
    torch.cuda.synchronize()
    for c in [cw, cd] + [o[1] for o in outs]:
        c()
    return {"dup": dup.clone(), "dw": outs[0][0].clone(), "db": outs[1][0].clone(), "db_up": outs[2][0].clone(),
            "ws": ws.clone()}


def _kpts_twice(up, w, dkp, dl, dr, gs):
    a, b = run_kpts(up, w, dkp, dl, dr, gs), run_kpts(up, w, dkp, dl, dr, gs)
    assert all(same(a[k], b[k]) for k in a)
    return a


def _column_invariant(dup, up):
    """dup16 is the same for every y of a column wherever up > 0, and +0 wherever up <= 0"""
    full = E.phase_major_inv(dup.float()).float()
    on = up > 0
    hi = torch.where(on, full, torch.full_like(full, -float("inf"))).amax(1)
    lo = torch.where(on, full, torch.full_like(full, float("inf"))).amin(1)
    any_on = on.any(1)
    assert torch.equal(hi[any_on], lo[any_on])
    assert bool((bits(E.phase_major_inv(dup))[~on] == 0).all())


@pytest.mark.parametrize("case", E.KP_CASES, ids=lambda c: "R%d-G%d-C%d-gs%g" % c)
def test_kpts_tail_backward(case):
    R, Gd, C, gs = case
    w, dkp, dl, dr = E.kpts_exact_grads(R, Gd, C)
    up = E.kpts_exact_up(R, Gd, C).cuda()
    wc, dkpc, dlc, drc = cuda(w, dkp, dl, dr)
    got = _kpts_twice(up, wc, dkpc, dlc, drc, gs)
    ref, _ = E.kpts_ref(up, wc, E.logit_grads(dkpc, dlc, drc), gs)
    for k in ("dw", "db", "db_up"):
        assert torch.equal(got[k].double(), ref[k]), k
    assert same(got["dup"], ref["dup"].float().half())
    _column_invariant(got["dup"], up)
    if R * Gd * Gd * C > 1 << 25:
        return
    up, w, dkp, dl, dr = E.kpts_random(R, Gd, C, device="cuda")
    wc, dkpc, dlc, drc = cuda(w, dkp, dl, dr)
    got = _kpts_twice(up, wc, dkpc, dlc, drc, gs)
    ref, bound = E.kpts_ref(up, wc, E.logit_grads(dkpc, dlc, drc), gs)
    ratios = {k: E.worst_ratio(got[k], ref[k], bound[k]) for k in ("dup", "dw", "db", "db_up")}
    ratios["db[5] (right border)"] = E.worst_ratio(got["db"][5:], ref["db"][5:], bound["db"][5:])
    _column_invariant(got["dup"], up)
    report("kpts_tail_backward R=%d G=%d C=%d gs=%g" % case, ratios)


# ================================================================================================ permute3 ====
@pytest.mark.parametrize("order", E.ORDERS)
@pytest.mark.parametrize("dims", E.PERM_SHAPES)
def test_permute3(dims, order):
    L = _l.load()
    n = int(np.prod(dims))
    src = torch.randn(n, generator=torch.Generator().manual_seed(n)).cuda()
    want = src.view(*dims).permute(*order).contiguous().view(-1)
    runs = []
    for _ in range(2):
        dst, check = guarded((n,), F32)
        assert L.sb_permute3(vp(src), *dims, *E.permute_strides(dims, order), vp(dst), G.stream_ptr()) == 0
        torch.cuda.synchronize()
        check()
        runs.append(dst.clone())
    assert same(runs[0], want) and same(runs[0], runs[1])


# ================================================================================================ box_tail_scores ====
@pytest.mark.parametrize("nc,K", E.SCORE_CASES)
def test_box_tail_scores_matches_box_tail(nc, K):
    L = _l.load()
    R = 33
    for exact in (True, False):
        fc7 = (E.box_exact if exact else E.box_random)(R, K, nc)[3]
        ws = E.box_tail_weights(K, nc, exact)
        fc7c, *wc = cuda(fc7, *ws)
        a = [guarded((R, n * nc), F32) for n in (1, 6, 5)]
        b = [guarded((R, n * nc), F32) for n in (1, 6, 5, 1)]
        assert L.sb_box_tail(vp(fc7c), R, K, nc, *[vp(t) for t in wc], *[vp(o[0]) for o in a], G.stream_ptr()) == 0
        assert L.sb_box_tail_scores(vp(fc7c), R, K, nc, *[vp(t) for t in wc], *[vp(o[0]) for o in b],
                                    G.stream_ptr()) == 0
        torch.cuda.synchronize()
        for o in a + b:
            o[1]()
        for x, y, name in zip(a, b, ("cls_prob", "bbox_pred", "dim_orien")):
            assert same(x[0], y[0]), name
        ref, bound = E.score_bound(fc7c, wc[0], wc[1])
        if exact:
            assert torch.equal(b[3][0].double(), ref)
        else:
            report("cls_score nc=%d K=%d" % (nc, K), {"cls_score": E.worst_ratio(b[3][0], ref, bound)})


# ================================================================================================ non-finite flag ====
def _flag(v=0):
    return torch.full((1,), v, dtype=torch.int32, device="cuda")


@pytest.mark.parametrize("which", [0, 1, 2])
def test_flag_nan_in_one_box_gradient(which):
    ops = list(E.box_random(9, 257, 2))
    ops[which] = ops[which].copy()
    ops[which][4 % ops[which].shape[0], -1] = np.nan
    nf = _flag()
    run_box(ops, 1.25, 1.0, nf)
    assert int(nf.item()) == 1


@pytest.mark.parametrize("which", [0, 1, 2])
def test_flag_nan_in_one_kpts_gradient(which):
    up, w, dkp, dl, dr = E.kpts_random(9, 28, 64, device="cuda")
    g = [dkp.copy(), dl.copy(), dr.copy()]
    g[which][3, -1] = np.nan
    nf = _flag()
    run_kpts(up, *cuda(w, *g), 1.0, nf)
    assert int(nf.item()) == 1


def test_flag_clean_stays_and_is_never_cleared():
    ops = E.box_random(9, 257, 2)
    up, w, dkp, dl, dr = E.kpts_random(9, 28, 64, device="cuda")
    for v in (0, 1):
        nf = _flag(v)
        run_box(ops, 1.25, 2.0 ** 12, nf)
        run_kpts(up, *cuda(w, dkp, dl, dr), 2.0 ** 10, nf)
        assert int(nf.item()) == v


def test_flag_dz16_overflow_with_finite_dz32():
    ops = E.box_random(9, 257, 2)
    ref, _ = E.box_ref(*[torch.from_numpy(a).double() for a in ops], 1.0, 1.0)
    gs = 2.0 ** int(np.ceil(np.log2(1e5 / float(ref["dz"].abs().max()))))
    nf = _flag()
    got = run_box(ops, 1.0, gs, nf)
    assert bool(torch.isfinite(got["dz"]).all()) and float(got["dz"].abs().max()) > 65520
    assert bool(torch.isinf(got["dz16"].float()).any()) and int(nf.item()) == 1


def test_flag_dw_overflow_with_finite_dz():
    R, K, nc = 4, 256, 1
    d = [np.full((R, n * nc), 1e20, np.float32) for n in (1, 6, 5)]
    W = [np.full((n * nc, K), 1e-30, np.float32) for n in (1, 6, 5)]
    fc7 = np.full((R, K), 1e20, np.float32)
    nf = _flag()
    got = run_box([d[0], d[1], d[2], fc7, W[0], W[1], W[2]], 1.0, 1.0, nf)
    assert bool(torch.isfinite(got["dz"]).all()) and bool(torch.isfinite(got["dz16"].float()).all())
    assert bool(torch.isfinite(got["db"]).all()) and bool(torch.isinf(got["dw"]).all())
    assert int(nf.item()) == 1


def test_flag_kpts_reduce_overflow_only():
    """per-RoI partials finite, their sum over the two RoIs not: only kpts_tail_bwd_reduce raises the flag"""
    R, Gd, C = 2, 2, 32
    up = torch.full((R, Gd, Gd, C), 4.0, dtype=F16, device="cuda")          # colsum 8
    w = torch.zeros(6, C, device="cuda")                                    # g = 0: dup16 and db_up stay 0
    dkp = torch.full((R, 4 * Gd), 2e37, device="cuda")                      # per RoI dW = 2 x 2e37 x 8 = 3.2e38
    dl, dr = torch.full((R, Gd), 2e37, device="cuda"), torch.full((R, Gd), 2e37, device="cuda")
    nf = _flag()
    got = run_kpts(up, w, dkp, dl, dr, 1.0, nf)
    part = got["ws"].view(R, 7 * C + 8)[:, :7 * C + 6]
    assert bool(torch.isfinite(part).all()) and float(part.abs().max()) > 3e38
    assert bool(torch.isinf(got["dw"]).all()) and bool(torch.isfinite(got["db"]).all())
    assert bool((got["dup"].float() == 0).all()) and int(nf.item()) == 1


# ================================================================================================ the chain ====
@pytest.fixture(scope="module")
def sd():
    return OM.make_state_dict(3)


@pytest.fixture(scope="module")
def chain(sd):
    H, W = _small_hw()
    eng = EN.StereoRCNNEngine(sd, "cuda", precision="fp16")
    with torch.no_grad():
        feats = {B: eng.trunk_fpn(_pairs(H, W, B, 5).cuda()) for B in (1, 2)}
    return eng, feats, H, W


def _forward(chain, B, rl, rr, words):
    eng, feats, H, _ = chain
    with torch.no_grad():
        return eng.heads(feats[B], B, rl, rr, float(H), save_for_backward=True, dropout_words=words)


def _upstream(out, seed):
    g = torch.Generator().manual_seed(seed)
    return [(torch.randn(*out[k].shape, generator=g) * 1e-2).cuda()
            for k in ("cls_score", "bbox_pred", "dim_orien_pred", "kpts_pred", "left_border_pred", "right_border_pred")]


# the conv weight gradients (sb_conv_wgrad / conv_wgrad_acc, held to their own order in test_gpu_wgrad.py) reduce over
# R x 196 pixels for the keypoint convs: at R = 1024 and random upstream gradients their relative L2 error against
# float64 reaches 3.8e-5 (RCNN_kpts.10.weight), which the 2e-5 bar of the single-image test does not allow for
WGRAD_OUT = {"RCNN_top.%d.%s" % (i, s) for i in (0, 3) for s in ("weight", "bias")} | \
    {"RCNN_kpts.%d.%s" % (i, s) for i in range(0, 12, 2) for s in ("weight", "bias")} | {"RCNN_kpts.12.weight"}
WGRAD_TOL = 1e-4


@pytest.mark.parametrize("B,R,dropout", [(2, 1024, False), (2, 1024, True), (1, 1, False), (2, 129, True)])
def test_heads_backward_vs_float64_from_state_dict(chain, sd, B, R, dropout):
    eng, _, H, W = chain
    rl, rr = cuda(*E.synth_rois(R, B, H, W))
    words = _words((2, R, 2048), 40 + R) if dropout else None
    out, saved = _forward(chain, B, rl, rr, words)
    d = _upstream(out, R)
    gs = 2.0 ** 10
    got, dpool = eng.heads_backward(saved, *d, grad_scale=gs)
    got = {k: v.clone() for k, v in got.items()}
    torch.cuda.synchronize()
    assert int(eng.found_inf.item()) == 0
    with torch.no_grad():
        ref, rpool, mid = _heads_backward_ref(eng, sd, saved, d, gs)
    errs = {n: l2_err(got[n], ref[n]) for n in ref}
    errs.update({"d" + k: l2_err(dpool[k], rpool[k]) for k in rpool})
    errs.update({k: l2_err(a, b) for k, (a, b) in mid.items()})
    print("heads_backward B=%d R=%d dropout=%s relative L2: worst %s" % (B, R, dropout, max(errs.items(),
                                                                                         key=lambda kv: kv[1])))
    bar = {n: WGRAD_TOL if R >= 1024 and n in WGRAD_OUT else KERNEL_TOL for n in errs}
    assert all(e < bar[n] for n, e in errs.items()), errs
    # per element: the three linears, kpts_class and the deconv bias against their a-priori bounds
    keep = 1.25 if dropout else 1.0
    w_cls, _, w_box, _, w_dim, _ = eng.fc
    bref, bb = E.box_ref(d[0], d[1], d[2], saved.fc7.view(R, -1), w_cls, w_box, w_dim, keep, gs)
    nc = d[0].shape[1]
    gw = torch.cat([got[n + ".weight"].view(-1, 2048) for n in ("RCNN_cls_score", "RCNN_bbox_pred",
                                                                  "RCNN_dim_orien_pred")], 0)
    gb = torch.cat([got[n + ".bias"] for n in ("RCNN_cls_score", "RCNN_bbox_pred", "RCNN_dim_orien_pred")], 0)
    assert gw.shape == (12 * nc, 2048)
    with torch.no_grad():
        kref, kb = E.kpts_ref(saved.up, eng.kpts_class[0], E.logit_grads(*d[3:]), gs)
    ratios = {"linears.weight": E.worst_ratio(gw, bref["dw"], bb["dw"]),
              "linears.bias": E.worst_ratio(gb, bref["db"], bb["db"]),
              "kpts_class.weight": E.worst_ratio(got["kpts_class.weight"].view(-1), kref["dw"], kb["dw"]),
              "kpts_class.bias": E.worst_ratio(got["kpts_class.bias"], kref["db"], kb["db"]),
              "RCNN_kpts.12.bias": E.worst_ratio(got["RCNN_kpts.12.bias"], kref["db_up"], kb["db_up"])}
    report("heads_backward B=%d R=%d dropout=%s" % (B, R, dropout), ratios)


def test_heads_backward_per_roi_invariance(chain):
    """pooled gradients and saved activations of a RoI do not depend on the other RoIs or on their order"""
    _, _, H, W = chain
    R, B = 1024, 2
    rl, rr = E.synth_rois(R, B, H, W)
    words = _words((2, R, 2048), 77)
    out, _ = _forward(chain, B, *cuda(rl, rr), words)
    d = _upstream(out, 78)
    perm = torch.from_numpy(np.random.RandomState(79).permutation(R)).cuda()
    keys = ("pooled_box", "pooled_kpts", "top0", "fc7", "up")

    def run(idx):
        rli, rri = cuda(rl, rr)
        o, s = _forward(chain, B, rli[idx].contiguous(), rri[idx].contiguous(), words[:, idx].contiguous())
        g, p = chain[0].heads_backward(s, *[t[idx].contiguous() for t in d], grad_scale=2.0 ** 10)
        res = {k: getattr(s, k).clone() for k in keys}
        res.update({"kpts%d" % i: t.clone() for i, t in enumerate(s.kpts)})
        res.update({"d " + k: v.clone() for k, v in p.items()})
        torch.cuda.synchronize()
        return res
    every = torch.arange(R, device="cuda")
    a = run(every)
    b = run(perm)
    c = run(every[:37])
    inv = torch.argsort(perm)
    for k in a:
        assert same(a[k], b[k][inv]), k
        assert same(a[k][:37], c[k]), k
    print("per-RoI invariance over %d tensors: bit-identical under a permutation and for the first 37 RoIs" % len(a))
