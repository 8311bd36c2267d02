"""GPU: backward of the trunk + FPN (sb_conv2d_tc_dgrad, sb_conv_wgrad, sb_fpn_grad_combine, engine.trunk_fpn_backward).

Per kernel: operands rounded to fp16 first, then compared with float64 torch (relative L2 < 2e-5), so that kernel
defects are separated from rounding noise.  End to end: every returned gradient against torch fp32 autograd through
oracle.model.trunk_fpn (relative L2 < 5e-3 for the FPN, 1e-1 for the trunk; the measured worst error per tensor is
printed).  That bar is loose because fp16 flips ReLU masks; the wiring between the kernels is held to the kernel bar
by test_gpu_trunk_backward_replay.py, which replays every layer in float64 from the engine's own recorded operands
and masks (fp32 data gradients relative L2 < 2e-5, weight gradients element by element within the wgrad bound)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import model as OM
from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200 import ops as G
from stereo_rcnn_b200.synth import synth_pair

pytestmark = pytest.mark.gpu

KERNEL_TOL = 2e-5
MODEL_TOL = 5e-3          # FPN convs (measured worst 6.7e-4 at 600x1987)
# Trunk convs miss 5e-3: measured 1.1e-2 (layer-4 conv3, first in the chain) growing to 7.4e-2 further down.  The
# kernels are exact to 2e-5 on fp16 operands (tests above) and the FPN gradients, which pass no ReLU, agree to 7e-4,
# so the spread grows with the number of ReLU masks crossed: the fp16 forward differs from fp32 by ~1e-3, which flips
# the masks of near-zero pre-activations, and each flipped element changes the gradient by its full value.  The fp32
# oracle shows the same sensitivity by itself: rounding only its conv weights to fp16 moves its trunk gradients by
# 9.7e-3 .. 5.7e-2 (worst again layer-3 conv1) and its FPN gradients by 5.1e-4 (600x1987 pair, fixed_blocks=1).
TRUNK_TOL = 1e-1
# dP ~ 1e-3 leaves the deeper trunk gradients in fp16's subnormal range; a training loop scales them up (GradScaler),
# and so do the oracle comparisons
GRAD_SCALE = 2.0 ** 14


def l2_err(a, b):
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    return float((a - b).norm() / max(float(b.norm()), 1e-300))


def h16(t):
    """round to fp16 and back: the operand values the kernels see"""
    return t.half().float()


def nchw(t):
    return t.permute(0, 3, 1, 2)


# (N, H, W, Cin, Cout, k) -- shape classes of the trunk + FPN
WGRAD_CASES = [
    (2, 19, 33, 64, 256, 1),        # 1x1 (layer-1 conv3 / downsample)
    (2, 10, 17, 1024, 256, 1),      # lateral 1x1
    (2, 13, 70, 256, 256, 3),       # 3x3 at 256 (smooth / layer-3 conv2), rows longer than one 64-pixel K-block
    (1, 9, 20, 512, 512, 3),        # 3x3 at 512 (layer-4 conv2)
    (2, 7, 9, 64, 128, 3),          # Cin / Cout not multiples of the 128 tile
    (2, 5, 7, 256, 64, 1),          # Cout = 64: half of the 128-row dY tile is zero-fill (layer-1 conv1)
    (2, 6, 9, 64, 64, 3),           # Cin = Cout = 64
    (1, 1, 1, 64, 128, 1),          # a single pixel: one K-block of 63 zero-filled rows, one bias chunk
    (1, 1, 1, 128, 64, 3),          # a single pixel, 3x3: eight of nine taps read only the halo
    (1, 3, 64, 64, 128, 3),         # W = 64: one full 64-pixel chunk per row
    (1, 3, 65, 128, 64, 3),         # W = 65: a second chunk of one pixel per row
    (1, 5, 9, 64, 64, 1),           # N*H*W = 45 < 64: fewer pixels than one K-block and than the bias chunks
    (2, 7, 9, 64, 192, 1),          # Cout = 192: the second m-tile is half empty
]


def wgrad_plan(N, H, W, Cin, Cout, k, sms):
    """conv_wgrad.cu plan(): -> (K-blocks, K-blocks per split, splits)"""
    num_kb = N * H * -(-W // 64) if k == 3 else -(-(N * H * W) // 64)
    tiles = -(-Cout // 128) * k * k * -(-Cin // 128)
    splits = max(1, min(-(-2 * sms // tiles), num_kb // 8))
    kbs = -(-num_kb // splits)
    return num_kb, kbs, -(-num_kb // kbs)


@pytest.mark.parametrize("case", WGRAD_CASES)
def test_wgrad_exact(case):
    _check_wgrad(case)


@pytest.mark.parametrize("split", ["short_last", "single"])
def test_wgrad_split_tails(split):
    """the K-split tails of plan(), found for this device's SM count: a last split shorter than the others (the
    fixed-order reduction over splits must include it), and a single split"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for m in range(64 * 12 + 1, 64 * 400):
        case = (1, 1, m, 128, 128, 1)
        num_kb, kbs, splits = wgrad_plan(*case, sms)
        if m % 64 and (num_kb % kbs and splits > 1 if split == "short_last" else splits == 1 and num_kb > 8):
            break
    else:
        pytest.fail("no shape with a %s split" % split)
    print("wgrad split %s: M = %d, %d K-blocks, %d per split, %d splits" % (split, m, num_kb, kbs, splits))
    _check_wgrad(case)


def _check_wgrad(case):
    N, H, W, Cin, Cout, k = case
    g = torch.Generator().manual_seed(1)
    dy = torch.randn(N, H, W, Cout, generator=g)
    x = torch.relu(torch.randn(N, H, W, Cin, generator=g))
    scale = torch.rand(Cout, generator=g) + 0.5
    dw = torch.empty(Cout, Cin, k, k, device="cuda")
    db = torch.empty(Cout, device="cuda")
    G.conv_wgrad(dy.half().cuda(), x.half().cuda(), k, dw, scale=scale.cuda(), grad_scale=4.0, dy32=dy.cuda(), db=db)
    torch.cuda.synchronize()
    xd = nchw(h16(x)).double().requires_grad_(False)
    wd = torch.zeros(Cout, Cin, k, k, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(xd, wd, padding=k // 2)
    (y * nchw(h16(dy)).double()).sum().backward()
    ref = wd.grad * scale.double().view(-1, 1, 1, 1) / 4.0
    assert l2_err(dw, ref) < KERNEL_TOL, l2_err(dw, ref)
    assert l2_err(db, dy.double().sum((0, 1, 2)) / 4.0) < 1e-6


# (N, H, W, Cin_forward, Cout_forward, k, stride) -- dgrad = the forward conv on transposed weights
DGRAD_CASES = [
    (2, 19, 33, 64, 256, 1, 1),
    (2, 21, 23, 256, 128, 1, 2),     # strided 1x1: scatter to the even positions through out_strides
    (2, 13, 40, 256, 256, 3, 1),
    (1, 9, 20, 512, 512, 3, 1),
    (2, 10, 17, 1024, 256, 1, 1),    # lateral 1x1
    (1, 5, 13, 64, 256, 1, 1),       # forward Cin = 64: the 64-wide masked variant; M = 65
    (1, 11, 23, 64, 256, 1, 2),      # ... strided (M = 72 at the strided pixels)
    (3, 1, 43, 64, 128, 1, 1),       # M = 129: a last m-tile of one row
    (1, 1, 1, 128, 64, 1, 1),        # a single pixel
    (1, 9, 17, 64, 64, 3, 1),        # 3x3 patches with a one-row tail
]
SENT32 = 0x7FA5A5A5                  # NaN bit pattern: bytes the data gradient must not write


@pytest.mark.parametrize("case", DGRAD_CASES)
@pytest.mark.parametrize("epi", ["plain", "mask_residual"])
def test_dgrad_exact_on_restated_weights(case, epi):
    N, H, W, Cin, Cout, k, stride = case
    g = torch.Generator().manual_seed(2)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    w = torch.randn(Cout, Cin, k, k, generator=g) / (Cin * k * k) ** 0.5
    s = torch.rand(Cout, generator=g) + 0.5
    dy = torch.randn(N, Ho, Wo, Cout, generator=g)
    # the data gradient's weights, as the engine packs them: [Cin][kh][kw][Cout] fp16, taps flipped, scale folded in
    w16 = (w * s.view(-1, 1, 1, 1)).flip(2, 3).permute(1, 2, 3, 0).contiguous().half()
    ws = w16.float().permute(3, 0, 1, 2).flip(2, 3)                     # the fp16-rounded s * w actually used
    ref = F.conv_transpose2d(nchw(h16(dy)).double(), ws.double(), stride=stride, padding=k // 2,
                             output_padding=(H - 1 - (Ho - 1) * stride))
    ref = ref.permute(0, 2, 3, 1)
    # the output inside a sentinel-filled buffer with guard rows: every pixel of the (strided) output written, every
    # other byte -- the odd positions of a strided scatter included -- left alone
    lead, n = 5 * Cin, N * H * W * Cin
    buf = torch.full((lead + n + 7 * Cin,), SENT32, dtype=torch.int32, device="cuda")
    out = buf[lead:lead + n].view(torch.float32).view(N, H, W, Cin)
    res = mask = None
    if epi == "mask_residual":
        res_cpu = torch.randn(N, Ho, Wo, Cin, generator=g) if k == 1 else None
        mask_cpu = torch.randn(N, H, W, Cin, generator=g).half()
        res = res_cpu.cuda() if res_cpu is not None else None
        mask = mask_cpu.cuda()
        if res_cpu is not None:
            full = torch.zeros(N, H, W, Cin, dtype=torch.float64)
            full[:, ::stride, ::stride] = res_cpu.double()
            ref = ref + full
        ref = torch.where(mask_cpu.float() > 0, ref, torch.zeros_like(ref))
    d = G.conv_desc(dy.half().cuda(), w16.cuda(), out, Cout, Cin, k, k, 1, k // 2, Ho, Wo, residual=res,
                    out_strides=(H * W * Cin, stride * W * Cin, stride * Cin))
    G.conv2d_dgrad(d, mask)
    torch.cuda.synchronize()
    written = torch.zeros(N, H, W, Cin, dtype=torch.bool, device="cuda")
    written[:, ::stride, ::stride] = True
    untouched = torch.cat([buf[:lead], buf[lead:lead + n][~written.view(-1)], buf[lead + n:]])
    assert bool((untouched == SENT32).all()), "bytes outside the data gradient were written"
    got = out[:, ::stride, ::stride]
    assert bool(torch.isfinite(got).all()), "elements of the data gradient were not written"
    ref = ref[:, ::stride, ::stride]
    assert l2_err(got, ref) < KERNEL_TOL, l2_err(got, ref)


@pytest.mark.parametrize("shape", [((2, 38, 125), (2, 19, 63)), ((1, 75, 249), (1, 38, 125)), ((2, 5, 3), (2, 3, 2))])
def test_upsample_transpose_matches_autograd(shape):
    (N, TH, TW), (_, H, W) = shape
    C = 256
    g = torch.Generator().manual_seed(3)
    dt = torch.randn(N, TH, TW, C, generator=g)
    src = torch.zeros(N, C, H, W, requires_grad=True)
    F.interpolate(src, size=(TH, TW), mode="bilinear", align_corners=True).backward(nchw(dt))
    got = G.upsample_transpose(dt.cuda(), H, W)
    torch.cuda.synchronize()
    assert l2_err(got, src.grad.permute(0, 2, 3, 1)) < 1e-6


def test_fpn_grad_combine_with_p6():
    g = torch.Generator().manual_seed(4)
    dp = torch.randn(2, 19, 63, 256, generator=g)
    dt = torch.randn(2, 38, 125, 256, generator=g)
    dp6 = torch.randn(2, 10, 32, 256, generator=g)
    o32, o16 = G.fpn_grad_combine(dp.cuda(), dt=dt.cuda(), dp6=dp6.cuda(), scale=8.0)
    torch.cuda.synchronize()
    ref = 8.0 * dp.double() + G.upsample_transpose(dt.cuda(), 19, 63).cpu().double()
    ref[:, ::2, ::2] += 8.0 * dp6.double()
    assert l2_err(o32, ref) < 1e-6
    assert torch.equal(o16.cpu(), o32.cpu().half())


# ---------------------------------------------------------------- trunk + FPN against the oracle
def _pair(H, W, seed=5):
    left, right = synth_pair(H, W, seed, 12)
    return torch.from_numpy(np.concatenate([left[None], right[None]], 0)).contiguous()


def _d_feats(feats, seed=11):
    g = torch.Generator().manual_seed(seed)
    return {k: torch.randn(feats[k].shape, generator=g) * 1e-3 for k in ("p2", "p3", "p4", "p5", "p6")}


def _oracle_grads(sd, im, d_nhwc, fixed_blocks, device):
    """fp32 autograd through oracle.model.trunk_fpn (TF32 off) -> {name: grad}"""
    names = [n for n, _ in E.trainable_trunk_fpn_params(fixed_blocks)]
    sdd = {k: v.to(device) for k, v in sd.items()}
    for n in names:
        sdd[n] = sdd[n].clone().requires_grad_(True)
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.enable_grad():
            f = OM.trunk_fpn(im.to(device), sdd)
            loss = sum((f[k] * nchw(d_nhwc[k]).to(device)).sum() for k in d_nhwc)
            gr = torch.autograd.grad(loss, [sdd[n] for n in names])
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    return {n: t.detach().cpu() for n, t in zip(names, gr)}


def _small_hw():
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "forward_small.npz"))
    return int(g["H"]), int(g["W"])


@pytest.fixture(scope="module")
def small_run():
    H, W = _small_hw()
    sd = OM.make_state_dict(3)
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    im = _pair(H, W)
    with torch.no_grad():
        feats, saved = eng.trunk_fpn(im.cuda(), save_for_backward=True)
    d = _d_feats(feats)
    return sd, eng, im, feats, saved, d


def _check_against_oracle(got, ref, label):
    worst = sorted(((l2_err(got[n], ref[n]), n) for n in ref), reverse=True)
    print("%s: relative L2 error per tensor: %s" % (label, ", ".join("%s %.2e" % (n, e) for e, n in worst)))
    bad = [(n, e) for e, n in worst if not e < (TRUNK_TOL if n.startswith("RCNN_layer") else MODEL_TOL)]
    assert not bad, bad


@pytest.mark.parametrize("fixed_blocks", [0, 1, 2, 3])
def test_trunk_fpn_backward_small_vs_oracle(small_run, fixed_blocks):
    sd, eng, im, feats, saved, d = small_run
    got = eng.trunk_fpn_backward(saved, {k: v.cuda() for k, v in d.items()}, fixed_blocks=fixed_blocks,
                                 grad_scale=GRAD_SCALE)
    torch.cuda.synchronize()
    names = [n for n, _ in E.trainable_trunk_fpn_params(fixed_blocks)]
    assert sorted(got) == sorted(names)
    assert int(eng.found_inf.item()) == 0
    ref = _oracle_grads(sd, im, d, fixed_blocks, "cpu")
    _check_against_oracle(got, ref, "small fixed_blocks=%d" % fixed_blocks)


def test_trunk_fpn_backward_benchmark_size_vs_oracle():
    """the benchmarked 600x1987 pair; the oracle graph runs in fp32 (TF32 off) on the GPU through torch"""
    sd = OM.make_state_dict(3)
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    im = _pair(600, 1987, seed=3)
    with torch.no_grad():
        feats, saved = eng.trunk_fpn(im.cuda(), save_for_backward=True)
    d = _d_feats(feats, seed=12)
    got = eng.trunk_fpn_backward(saved, {k: v.cuda() for k, v in d.items()}, fixed_blocks=1, grad_scale=GRAD_SCALE)
    got = {k: v.cpu() for k, v in got.items()}
    assert int(eng.found_inf.item()) == 0
    del saved, feats
    torch.cuda.empty_cache()
    ref = _oracle_grads(sd, im, d, 1, "cuda")
    _check_against_oracle(got, ref, "600x1987 fixed_blocks=1")


def test_grad_scale_and_overflow_flag(small_run):
    sd, eng, im, feats, saved, d = small_run
    base = {k: v.clone() for k, v in eng.trunk_fpn_backward(saved, {k: v.cuda() for k, v in d.items()}).items()}
    tiny = {k: (v * 1e-6).cuda() for k, v in d.items()}
    got = eng.trunk_fpn_backward(saved, tiny, grad_scale=2.0 ** 20)
    torch.cuda.synchronize()
    assert int(eng.found_inf.item()) == 0
    for n in base:
        assert l2_err(got[n], base[n] * 1e-6) < MODEL_TOL, n
    eng.trunk_fpn_backward(saved, {k: v.cuda() for k, v in d.items()}, grad_scale=2.0 ** 40)
    torch.cuda.synchronize()
    assert int(eng.found_inf.item()) == 1
    eng.trunk_fpn_backward(saved, {k: v.cuda() for k, v in d.items()})
    torch.cuda.synchronize()
    assert int(eng.found_inf.item()) == 0


def test_backward_deterministic_into_given_buffers_and_graph_capturable(small_run):
    sd, eng, im, feats, saved, d = small_run
    dc = {k: v.cuda() for k, v in d.items()}
    a = {k: v.clone() for k, v in eng.trunk_fpn_backward(saved, dc).items()}
    bufs = {n: torch.full(s, float("nan"), device="cuda") for n, s in E.trainable_trunk_fpn_params(1)}
    b = eng.trunk_fpn_backward(saved, dc, grads=bufs)
    torch.cuda.synchronize()
    for n in a:
        assert b[n].data_ptr() == bufs[n].data_ptr()
        assert torch.equal(a[n], b[n]), n

    def step(x):
        f, s = eng.trunk_fpn(x, save_for_backward=True)
        return eng.trunk_fpn_backward(s, dc)
    with torch.no_grad():
        runner = E.GraphRunner(step, [im.cuda()])
        out = runner()
        torch.cuda.synchronize()
    for n in a:
        assert torch.equal(out[n], a[n]), n
