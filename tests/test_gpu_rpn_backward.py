"""GPU: backward of the stereo RPN (sb_rpn_head_scores, sb_rpn_head_grad, sb_conv_wgrad_acc, engine.rpn_backward,
train.rpn_gradients).

Kernels against float64 on the fp16-rounded operands they read (relative L2 < 2e-5, the bar of test_wgrad_exact);
rpn_backward alone against float64 with the engine's own ReLU masks; the RPN loss differentiated end to end against
fp32 autograd through oracle.model.trunk_fpn + rpn_head + oracle.train_targets.rpn_losses (the measured worst error
per tensor is printed)."""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import model as OM
from oracle import train_targets as T
from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200 import lib as _l
from stereo_rcnn_b200 import ops as G
from stereo_rcnn_b200 import train as TR
from stereo_rcnn_b200.synth import synth_pair, synth_train_gt

pytestmark = pytest.mark.gpu

KERNEL_TOL = 2e-5
MODEL_TOL = 5e-3          # FPN and RPN parameters
TRUNK_TOL = 1e-1          # trunk convs: fp16 ReLU-mask flips, see test_gpu_backward.py
LOSS_TOL = 1e-3
GRAD_SCALE = 2.0 ** 14    # the RPN loss gradients are ~1e-3 / 512: keep the deep trunk out of fp16's subnormals
SENT32 = 0x7FA5A5A5       # NaN bit patterns: bytes a kernel must not write
SENT16 = 0x7E55
LEVELS = ("p2", "p3", "p4", "p5", "p6")
SB_EINVAL = -22


def l2_err(a, b):
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    return float((a - b).norm() / max(float(b.norm()), 1e-300))


def h16(t):
    return t.half().double()


def nchw(t):
    return t.permute(0, 3, 1, 2)


def _small_hw():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "forward_small.npz"))
    return int(g["H"]), int(g["W"])


def _pairs(H, W, B, seed=5):
    """[2B,3,H,W]: the B left images, then the B right images"""
    ps = [synth_pair(H, W, seed + b, 12) for b in range(B)]
    return torch.from_numpy(np.stack([p[0] for p in ps] + [p[1] for p in ps], 0)).contiguous()


@pytest.fixture(scope="module")
def sd():
    return OM.make_state_dict(3)


# ---------------------------------------------------------------- 1. the training-mode forward
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("forks", [True, False])
def test_rpn_forward_unchanged_with_save(sd, B, forks):
    H, W = _small_hw()
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16", forks=forks)
    with torch.no_grad():
        feats = eng.trunk_fpn(_pairs(H, W, B).cuda())
        cp0, bb0, sh0 = eng.rpn(feats, B)
        cp1, bb1, sh1, saved, score = eng.rpn(feats, B, save_for_backward=True)
    torch.cuda.synchronize()
    assert sh0 == sh1
    assert torch.equal(cp0, cp1) and torch.equal(bb0, bb1)
    P = saved.offs[-1]
    ref = saved.head[:, :, 0:6].reshape(B, 3 * P, 2)          # each pixel's six raw scores as three pairs
    assert score.shape == (B, 3 * P, 2) and torch.equal(score, ref)
    for i, (h, w) in enumerate(sh1):
        assert saved.cats[i].shape == (B, h, w, 1024) and saved.cats[i].dtype == torch.float16
        assert saved.levels[i].data_ptr() == feats[LEVELS[i] + "_16"].data_ptr()


def test_rpn_save_requires_fp16(sd):
    eng = E.StereoRCNNEngine(sd, "cuda", precision="tf32")
    with pytest.raises(ValueError):
        eng.rpn({}, 1, save_for_backward=True)


# ---------------------------------------------------------------- 2. packing the head gradient
@pytest.mark.parametrize("B,P", [(1, 2720), (2, 37), (1, 1)])
def test_rpn_head_grad_packing(B, P):
    L = _l.load()
    g = torch.Generator().manual_seed(1)
    d_cls = torch.randn(B, 3 * P, 2, generator=g)
    d_box = torch.randn(B, 3 * P, 6, generator=g)
    gs = 8.0
    n, lead, tail = B * P * 64, 64 * 5, 64 * 7
    b16 = torch.full((lead + n + tail,), SENT16, dtype=torch.int16, device="cuda")
    b32 = torch.full((lead + n + tail,), SENT32, dtype=torch.int32, device="cuda")
    o16 = b16[lead:lead + n].view(torch.float16).view(B, P, 64)
    o32 = b32[lead:lead + n].view(torch.float32).view(B, P, 64)
    dc, db = d_cls.cuda(), d_box.cuda()
    G.check(L.sb_rpn_head_grad(G.ptr(dc), G.ptr(db), B, P, gs, G.ptr(o16), G.ptr(o32), G.stream_ptr()),
            "sb_rpn_head_grad")
    torch.cuda.synchronize()
    ref = torch.zeros(B, P, 64)
    ref[:, :, 0:6] = gs * d_cls.view(B, P, 6)
    ref[:, :, 6:24] = gs * d_box.view(B, P, 18)
    assert torch.equal(o32.cpu(), ref)
    assert torch.equal(o16.cpu(), ref.half())
    for buf, s in ((b16, SENT16), (b32, SENT32)):
        assert bool((buf[:lead] == s).all()) and bool((buf[lead + n:] == s).all()), "written past [B,P,64]"
    a16, a32 = G.rpn_head_grad(d_cls.cuda(), d_box.cuda(), B, P, gs)
    assert torch.equal(a16.cpu(), ref.half()) and torch.equal(a32.cpu(), ref)


# ---------------------------------------------------------------- 3. the strided, accumulating weight gradient
def _ref_wgrad(dy, x, k):
    """float64 dW [Cout,Cin,k,k] of a k x k (pad k // 2) conv: sum over pixels of dy x (both NHWC)"""
    Cout, Cin = dy.shape[3], x.shape[3]
    wd = torch.zeros(Cout, Cin, k, k, dtype=torch.float64, requires_grad=True)
    (F.conv2d(nchw(x.double()), wd, padding=k // 2) * nchw(dy.double())).sum().backward()
    return wd.grad


@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("coff", [0, 512])
def test_wgrad_acc_strided_dy(k, coff):
    """dY = one channel half of a [N,h,w,1024] gradient (the RPN_Conv layout), X dense"""
    N, Hh, Ww, Cin, Cout = 2, 9, 70, 256, 512
    g = torch.Generator().manual_seed(2)
    wide = torch.randn(N, Hh, Ww, 1024, generator=g)
    x = torch.relu(torch.randn(N, Hh, Ww, Cin, generator=g))
    w16, w32 = wide.half().cuda(), wide.cuda()
    dw = torch.empty(Cout, Cin, k, k, device="cuda")
    db = torch.empty(Cout, device="cuda")
    G.conv_wgrad_acc(w16[..., coff:coff + Cout], x.half().cuda(), k, dw, db=db, dy32=w32[..., coff:coff + Cout],
                     grad_scale=4.0)
    torch.cuda.synchronize()
    dy = wide[..., coff:coff + Cout]
    assert l2_err(dw, _ref_wgrad(h16(dy), h16(x), k) / 4.0) < KERNEL_TOL
    assert l2_err(db, dy.double().sum((0, 1, 2)) / 4.0) < 1e-6


@pytest.mark.parametrize("k", [1, 3])
def test_wgrad_acc_accumulates_segments(k):
    """a sum over segments of different N x H x W, one of fewer pixels than a 64-pixel K-block, with a BN scale"""
    segs = [(2, 13, 70), (1, 3, 5), (1, 1, 1), (2, 6, 9)]
    Cin, Cout = 128, 192
    g = torch.Generator().manual_seed(3)
    scale = torch.rand(Cout, generator=g) + 0.5
    dw = torch.full((Cout, Cin, k, k), float("nan"), device="cuda")
    db = torch.full((Cout,), float("nan"), device="cuda")
    ref_w = torch.zeros(Cout, Cin, k, k, dtype=torch.float64)
    ref_b = torch.zeros(Cout, dtype=torch.float64)
    for i, (n, hh, ww) in enumerate(segs):
        dy = torch.randn(n, hh, ww, Cout, generator=g)
        x = torch.relu(torch.randn(n, hh, ww, Cin, generator=g))
        G.conv_wgrad_acc(dy.half().cuda(), x.half().cuda(), k, dw, db=db, dy32=dy.cuda(), scale=scale.cuda(),
                         grad_scale=2.0, accumulate=i > 0)
        ref_w += _ref_wgrad(h16(dy), h16(x), k) * scale.double().view(-1, 1, 1, 1) / 2.0
        ref_b += dy.double().sum((0, 1, 2)) / 2.0
    torch.cuda.synchronize()
    assert l2_err(dw, ref_w) < KERNEL_TOL
    assert l2_err(db, ref_b) < 1e-6


def test_wgrad_acc_row_split():
    """the fused RPN head: Cout = 64 (rows 24..63 padding), rows 0..5 -> one tensor, 6..23 -> another"""
    g = torch.Generator().manual_seed(4)
    dy = torch.randn(1, 11, 37, 64, generator=g)
    x = torch.relu(torch.randn(1, 11, 37, 1024, generator=g))
    lo, hi = torch.empty(6, 1024, 1, 1, device="cuda"), torch.empty(18, 1024, 1, 1, device="cuda")
    blo, bhi = torch.empty(6, device="cuda"), torch.empty(18, device="cuda")
    G.conv_wgrad_acc(dy.half().cuda(), x.half().cuda(), 1, lo, db=blo, dy32=dy.cuda(), rows=24, split=6, dw_hi=hi,
                     db_hi=bhi)
    torch.cuda.synchronize()
    ref = _ref_wgrad(h16(dy), h16(x), 1)
    assert l2_err(lo, ref[0:6]) < KERNEL_TOL and l2_err(hi, ref[6:24]) < KERNEL_TOL
    rb = dy.double().sum((0, 1, 2))
    assert l2_err(blo, rb[0:6]) < 1e-6 and l2_err(bhi, rb[6:24]) < 1e-6


@pytest.mark.parametrize("case", [(2, 19, 33, 64, 256, 1), (2, 13, 70, 256, 256, 3), (1, 5, 9, 64, 64, 1)])
def test_wgrad_acc_dense_equals_conv_wgrad(case):
    N, Hh, Ww, Cin, Cout, k = case
    g = torch.Generator().manual_seed(5)
    dy = torch.randn(N, Hh, Ww, Cout, generator=g).cuda()
    x = torch.relu(torch.randn(N, Hh, Ww, Cin, generator=g)).half().cuda()
    scale = (torch.rand(Cout, generator=g) + 0.5).cuda()
    a = [torch.empty(Cout, Cin, k, k, device="cuda"), torch.empty(Cout, device="cuda")]
    b = [torch.empty(Cout, Cin, k, k, device="cuda"), torch.empty(Cout, device="cuda")]
    G.conv_wgrad(dy.half(), x, k, a[0], scale=scale, grad_scale=8.0, dy32=dy, db=a[1])
    G.conv_wgrad_acc(dy.half(), x, k, b[0], db=b[1], dy32=dy, scale=scale, grad_scale=8.0)
    torch.cuda.synchronize()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_wgrad_acc_rejects_invalid_arguments():
    """every refusal returns SB_EINVAL before any launch"""
    L = _l.load()
    N, Hh, Ww, Cin, Cout, k = 1, 4, 8, 64, 128, 3
    dy = torch.zeros(N, Hh, Ww, 1024, dtype=torch.float16, device="cuda")
    x = torch.zeros(N, Hh, Ww, Cin + 8, dtype=torch.float16, device="cuda")
    dw = torch.zeros(Cout, Cin, k, k, device="cuda")
    nb = L.sb_conv_wgrad_acc_workspace(N, Hh, Ww, Cin, Cout, k)
    ws = torch.zeros(nb + 64, dtype=torch.uint8, device="cuda")
    vp = lambda t, off=0: ctypes.c_void_p(t.data_ptr() + off)

    def call(dy_p=None, dy_ld=1024, x_p=None, x_ld=Cin + 8, cin=Cin, cout=Cout, nbytes=nb, ws_p=None, rows=Cout,
             split=Cout):
        return L.sb_conv_wgrad_acc(dy_p or vp(dy), dy_ld, x_p or vp(x), x_ld, N, Hh, Ww, cin, cout, k, None, 1.0, None,
                                   0, 0, rows, split, vp(dw), None, None, None, None, ws_p or vp(ws), nbytes,
                                   G.stream_ptr())
    torch.cuda.synchronize()
    n0 = G.launch_count()
    bad = {"misaligned dY": call(dy_p=vp(dy, 8)), "misaligned X": call(x_p=vp(x, 2)),
           "misaligned workspace": call(ws_p=vp(ws, 4)), "dY ld < Cout": call(dy_ld=120),
           "X ld < Cin": call(x_ld=56), "ld % 8": call(dy_ld=1020), "Cin % 64": call(cin=72, x_ld=72),
           "Cout % 64": call(cout=96), "short workspace": call(nbytes=nb - 1),
           "split > rows": call(rows=24, split=30), "rows > Cout": call(rows=Cout + 64),
           "split < rows without dw_hi": call(rows=24, split=6)}
    assert G.launch_count() == n0
    assert all(rc == SB_EINVAL for rc in bad.values()), bad
    assert call() == 0


# ---------------------------------------------------------------- 4. rpn_backward alone against float64
def _rpn_backward_ref(eng, saved, d_cls, d_box):
    """float64: heads and RPN_Conv on the engine's fp16 operands (fp16-rounded weights, saved cat, fp16 P levels), the
    ReLU replaced by the saved mask cat > 0; d cat rounded to fp16 where the kernels read it as an fp16 operand"""
    B, offs = saved.B, saved.offs
    wh = eng._bwd_src["rpn_heads"][0][:24, :, 0, 0].half().double()          # [24,1024]
    wc = eng._bwd_src["RCNN_rpn.RPN_Conv"][0].half().double()                # [512,256,3,3]
    P = offs[-1]
    dx = torch.zeros(B, P, 24, dtype=torch.float64)       # exact: the bias gradients read the fp32 twin
    dx[:, :, 0:6] = d_cls.cpu().double().view(B, P, 6)
    dx[:, :, 6:24] = d_box.cpu().double().view(B, P, 18)
    dh = h16(dx)
    g_head = torch.zeros(24, 1024, dtype=torch.float64)
    b_head = torch.zeros(24, dtype=torch.float64)
    g_conv = torch.zeros(512, 256, 3, 3, dtype=torch.float64)
    b_conv = torch.zeros(512, dtype=torch.float64)
    dps = {}
    for i, (h, w) in enumerate(saved.shapes):
        cat = saved.cats[i].cpu().double()                                   # [B,h,w,1024]
        d = dh[:, offs[i]:offs[i + 1]].reshape(B, h, w, 24)
        g_head += torch.einsum("bhwo,bhwi->oi", d, cat)
        b_head += dx[:, offs[i]:offs[i + 1]].sum((0, 1))
        dcat = (d @ wh) * (cat > 0).double()
        f = saved.levels[i].cpu().double()
        dp = torch.zeros(2 * B, h, w, 256, dtype=torch.float64)
        for side in range(2):
            dy = dcat[..., side * 512:(side + 1) * 512]
            g_conv += _ref_wgrad(h16(dy), f[side * B:(side + 1) * B], 3)
            b_conv += dy.sum((0, 1, 2))
            dp[side * B:(side + 1) * B] = F.conv_transpose2d(nchw(h16(dy)), wc, padding=1).permute(0, 2, 3, 1)
        dps[LEVELS[i]] = dp
    grads = {"RCNN_rpn.RPN_Conv.weight": g_conv, "RCNN_rpn.RPN_Conv.bias": b_conv,
             "RCNN_rpn.RPN_cls_score.weight": g_head[0:6].view(6, 1024, 1, 1),
             "RCNN_rpn.RPN_cls_score.bias": b_head[0:6],
             "RCNN_rpn.RPN_bbox_pred_left_right.weight": g_head[6:24].view(18, 1024, 1, 1),
             "RCNN_rpn.RPN_bbox_pred_left_right.bias": b_head[6:24]}
    return grads, dps


@pytest.mark.parametrize("B", [1, 2])
def test_rpn_backward_vs_float64(sd, B):
    H, W = _small_hw()
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    with torch.no_grad():
        feats = eng.trunk_fpn(_pairs(H, W, B).cuda())
        _, _, shapes, saved, score = eng.rpn(feats, B, save_for_backward=True)
    A = score.shape[1]
    g = torch.Generator().manual_seed(6)
    d_cls = torch.randn(B, A, 2, generator=g) * 1e-2
    d_box = torch.randn(B, A, 6, generator=g) * 1e-2
    got, dps = eng.rpn_backward(saved, d_cls.cuda(), d_box.cuda())
    torch.cuda.synchronize()
    assert int(eng.found_inf.item()) == 0
    assert sorted(got) == sorted(n for n, _ in E.trainable_rpn_params())
    ref, rdp = _rpn_backward_ref(eng, saved, d_cls, d_box)
    errs = {n: l2_err(got[n], ref[n]) for n in ref}
    errs.update({"d" + k: l2_err(dps[k], rdp[k]) for k in LEVELS})
    print("rpn_backward B=%d vs float64: %s" % (B, ", ".join("%s %.2e" % kv for kv in sorted(errs.items()))))
    for k in LEVELS:
        assert dps[k].shape == feats[k].shape and dps[k].dtype == torch.float32 and dps[k].is_contiguous()
    assert all(e < KERNEL_TOL for e in errs.values()), errs


# ---------------------------------------------------------------- 5. the RPN loss end to end against the oracle
def _keys(B, A, seed):
    w = np.random.RandomState(seed).randint(0, 2 ** 32, (B, A), dtype=np.uint64).astype(np.uint32)
    return torch.from_numpy(w.view(np.int32)).cuda()


def _device_targets(shapes, gt, H, W, keys):
    anchors = TR.generate_anchors(shapes, "cuda")
    return TR.anchor_targets(anchors, *[torch.from_numpy(t).cuda() for t in gt[:3]], (H, W), keys)


def _oracle(sd, im, B, targets, fixed_blocks, device, weights16=False):
    """fp32 autograd (TF32 off) through oracle trunk_fpn + rpn_head + rpn_losses -> (losses, {name: grad});
    weights16 rounds every conv weight to fp16 first (the sensitivity experiment)"""
    names = [n for n, _ in E.trainable_trunk_fpn_params(fixed_blocks) + E.trainable_rpn_params()]
    sdd = {k: v.to(device) for k, v in sd.items()}
    if weights16:
        sdd = {k: (v.half().float() if k.endswith("weight") and v.dim() == 4 else v) for k, v in sdd.items()}
    for n in names:
        sdd[n] = sdd[n].clone().requires_grad_(True)
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.enable_grad():
            f = OM.trunk_fpn(im.to(device), sdd)
            _, bbox, _, score = OM.rpn_head([f[k][:B] for k in LEVELS], [f[k][B:] for k in LEVELS], sdd)
            lc, lb = T.rpn_losses(score.cpu(), bbox.cpu(), *[t.cpu() for t in targets])     # CPU-built targets
            gr = torch.autograd.grad(lc + lb, [sdd[n] for n in names])
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    return (float(lc.detach()), float(lb.detach())), {n: t.detach().cpu() for n, t in zip(names, gr)}


def _tol(n):
    return TRUNK_TOL if n.startswith("RCNN_layer") else MODEL_TOL


def _check(got, ref, label):
    worst = sorted(((l2_err(got[n], ref[n]), n) for n in ref), reverse=True)
    print("%s: relative L2 error per tensor: %s" % (label, ", ".join("%s %.2e" % (n, e) for e, n in worst)))
    bad = [(n, e) for e, n in worst if not e < _tol(n)]
    assert not bad, bad


def _end_to_end(sd, H, W, B, fixed_blocks, device, seed=7, eng=None):
    eng = eng or E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    im = _pairs(H, W, B, seed)
    gt = synth_train_gt(B, 30, H, W, seed)
    shapes = [[-(-H // s), -(-W // s)] for s in (4, 8, 16, 32, 64)]
    keys = _keys(B, 3 * sum(h * w for h, w in shapes), seed + 1)
    g = [torch.from_numpy(t).cuda() for t in gt[:3]]
    imc = im.cuda()
    losses, got = TR.rpn_gradients(eng, imc[:B], imc[B:], *g, keys, fixed_blocks=fixed_blocks, grad_scale=GRAD_SCALE)
    got = {k: v.cpu() for k, v in got.items()}
    losses = losses.cpu()
    assert int(eng.found_inf.item()) == 0
    names = [n for n, _ in E.trainable_trunk_fpn_params(fixed_blocks) + E.trainable_rpn_params()]
    assert sorted(got) == sorted(names)
    targets = [t.cpu() for t in _device_targets(shapes, gt, H, W, keys)]
    assert float((targets[0] == 1).sum()) > 0
    del eng
    torch.cuda.empty_cache()
    rl, ref = _oracle(sd, im, B, targets, fixed_blocks, device)
    label = "%dx%d B=%d fixed_blocks=%d" % (H, W, B, fixed_blocks)
    print("%s: losses %s vs oracle %s" % (label, losses.tolist(), rl))
    for a, b in zip(losses.tolist(), rl):
        assert abs(a - b) <= LOSS_TOL * abs(b), (a, b)
    _check(got, ref, label)
    return im, targets, ref


@pytest.mark.parametrize("fixed_blocks", [0, 1, 2, 3])
def test_rpn_gradients_small_vs_oracle(sd, fixed_blocks):
    H, W = _small_hw()
    _end_to_end(sd, H, W, 1, fixed_blocks, "cpu")


def test_rpn_gradients_small_b2_vs_oracle(sd):
    H, W = _small_hw()
    _end_to_end(sd, H, W, 2, 1, "cpu", seed=9)


def test_rpn_gradients_benchmark_size_vs_oracle(sd):
    """the benchmarked 600x1987 pair; the oracle in fp32 (TF32 off) on the GPU.  Also prints how far rounding only the
    oracle's conv weights to fp16 moves its own gradients (the sensitivity the fp16 forward's mask flips bring)"""
    im, targets, ref = _end_to_end(sd, 600, 1987, 1, 1, "cuda", seed=3)
    _, ref16 = _oracle(sd, im, 1, targets, 1, "cuda", weights16=True)
    worst = sorted(((l2_err(ref16[n], ref[n]), n) for n in ref), reverse=True)
    print("oracle with fp16-rounded weights vs fp32: %s" % ", ".join("%s %.2e" % (n, e) for e, n in worst[:12]))
    print("  RPN: %s" % ", ".join("%s %.2e" % (n, e) for e, n in worst if n.startswith("RCNN_rpn")))


# ---------------------------------------------------------------- 6. determinism, capture, gradient scaling
@pytest.fixture(scope="module")
def step_case(sd):
    H, W = _small_hw()
    B = 1
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    im = _pairs(H, W, B, 7).cuda()
    gt = [torch.from_numpy(t).cuda() for t in synth_train_gt(B, 30, H, W, 7)[:3]]
    shapes = [[-(-H // s), -(-W // s)] for s in (4, 8, 16, 32, 64)]
    keys = _keys(B, 3 * sum(h * w for h, w in shapes), 8)
    return eng, im[:B].contiguous(), im[B:].contiguous(), gt, keys


def test_rpn_gradients_deterministic_into_given_buffers_and_graph_capturable(step_case):
    eng, iml, imr, gt, keys = step_case
    l0, a = TR.rpn_gradients(eng, iml, imr, *gt, keys, grad_scale=GRAD_SCALE)
    a = {k: v.clone() for k, v in a.items()}
    l0 = l0.clone()
    names = E.trainable_trunk_fpn_params(1) + E.trainable_rpn_params()
    bufs = {n: torch.full(s, float("nan"), device="cuda") for n, s in names}
    l1, b = TR.rpn_gradients(eng, iml, imr, *gt, keys, grads=bufs, grad_scale=GRAD_SCALE)
    torch.cuda.synchronize()
    assert torch.equal(l0, l1)
    for n in a:
        assert b[n].data_ptr() == bufs[n].data_ptr(), n
        assert torch.equal(a[n], b[n]), n

    def step(x, y):
        return TR.rpn_gradients(eng, x, y, *gt, keys, grad_scale=GRAD_SCALE)
    with torch.no_grad():
        runner = E.GraphRunner(step, [iml, imr])
        lg, out = runner()
        torch.cuda.synchronize()
    assert torch.equal(lg, l0)
    for n in a:
        assert torch.equal(out[n], a[n]), n


def test_rpn_gradients_with_uncertainty_weights(step_case):
    """the multi-task weights of trainval_net.py:214-219: gradients scale by exp(-uncert[i]), d total / d uncert"""
    eng, iml, imr, gt, keys = step_case
    u = torch.tensor([0.3, -0.2, 0.1, 0.0, 0.5, -0.4], device="cuda")
    l0, a = TR.rpn_gradients(eng, iml, imr, *gt, keys, grad_scale=GRAD_SCALE)
    a = {k: v.clone() for k, v in a.items()}
    l1, b, du = TR.rpn_gradients(eng, iml, imr, *gt, keys, uncert=u, grad_scale=GRAD_SCALE)
    torch.cuda.synchronize()
    assert torch.equal(l0, l1)
    lc, lb = [float(v) for v in l0.cpu()]
    uc = u.cpu().double().numpy()
    np.testing.assert_allclose(du.cpu().numpy(), [1 - lc * np.exp(-uc[0]), 1 - lb * np.exp(-uc[1])], rtol=1e-5)
    # the score head's gradient comes from the class loss only, the box head's from the box loss only.  The biases
    # read the fp32 head gradient; the weights read its fp16 rounding, which the factor exp(-u) moves by up to an ulp
    for head, i in (("RCNN_rpn.RPN_cls_score", 0), ("RCNN_rpn.RPN_bbox_pred_left_right", 1)):
        f = float(np.exp(-uc[i]))
        assert l2_err(b[head + ".bias"], a[head + ".bias"] * f) < 1e-6, head
        assert l2_err(b[head + ".weight"], a[head + ".weight"] * f) < 1e-3, head


def test_grad_scale_and_overflow_flag_survive_the_chain(step_case):
    eng, iml, imr, gt, keys = step_case
    with torch.no_grad():
        f, st = eng.trunk_fpn(torch.cat((iml, imr), 0), save_for_backward=True)
        _, _, _, sr, score = eng.rpn(f, 1, save_for_backward=True)
    g = torch.Generator().manual_seed(10)
    d_cls = (torch.randn(score.shape, generator=g) * 1e-3).cuda()
    d_box = (torch.randn(1, score.shape[1], 6, generator=g) * 1e-3).cuda()

    def chain(dc, db, gs):
        r, dp = eng.rpn_backward(sr, dc, db, grad_scale=gs)
        r = {k: v.clone() for k, v in r.items()}
        r.update({k: v.clone() for k, v in
                  eng.trunk_fpn_backward(st, dp, grad_scale=gs, clear_found_inf=False).items()})
        torch.cuda.synchronize()
        return r, int(eng.found_inf.item())
    base, fi = chain(d_cls, d_box, 1.0)
    assert fi == 0
    tiny, fi = chain(d_cls * 1e-6, d_box * 1e-6, 2.0 ** 20)
    assert fi == 0
    errs = {n: l2_err(tiny[n], base[n] * 1e-6) for n in base}
    print("grad_scale 2^20 on 1e-6 gradients vs unscaled: worst %s" % (max(errs.items(), key=lambda kv: kv[1]),))
    assert all(e < _tol(n) for n, e in errs.items()), errs
    # an fp16 overflow inside the RPN part: the trunk backward that follows must not clear the flag
    _, fi = chain(d_cls, d_box, 2.0 ** 40)
    assert fi == 1
    _, fi = chain(d_cls, d_box, 1.0)
    assert fi == 0
    # the same through the composed call
    TR.rpn_gradients(eng, iml, imr, *gt, keys, grad_scale=2.0 ** 40)
    torch.cuda.synchronize()
    assert int(eng.found_inf.item()) == 1
    TR.rpn_gradients(eng, iml, imr, *gt, keys, grad_scale=GRAD_SCALE)
    torch.cuda.synchronize()
    assert int(eng.found_inf.item()) == 0
