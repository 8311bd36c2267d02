"""CPU: which convolutions the tensor-core kernel takes (sb_conv2d_tc_supported, pure host logic), and that nothing
else runs an fp16 descriptor.  Descriptors carry fake, 16-byte-aligned device addresses: no call here launches.

Every rule of supported() in conv_tc.cu has one rejected row and an accepted neighbour that differs from it in the
one field the rule reads, so a rule that is dropped or widened fails a row."""
import ctypes

import pytest
import torch

from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import ops as G

BASE = 0x7f0000000000          # fake device addresses, 1 MB apart
A_IN, A_W, A_OUT, A_OUT16, A_RES, A_UP, A_SC, A_SH = (BASE + i * (1 << 20) for i in range(8))


@pytest.fixture(scope="module")
def lib():
    from stereo_rcnn_b200 import build
    build.build()
    return L.load()


def desc(f16=True, N=2, H=5, W=7, Cin=64, Cout=96, k=1, res=False, ups=False, twin=None, ld=None, **kw):
    """a dense NHWC conv descriptor the kernel accepts; kw overrides fields after the defaults are set"""
    d = L.ConvDesc()
    d.in_, d.wgt = A_IN, A_W
    d.out = A_OUT
    d.out16 = A_OUT16 if (f16 if twin is None else twin) else None
    d.in_dtype = 1 if f16 else 0
    d.scale, d.shift = A_SC, A_SH
    d.residual = A_RES if res else None
    d.up_src = A_UP if ups else None
    d.N, d.H, d.W, d.Cin, d.Cout, d.kh, d.kw = N, H, W, Cin, Cout, k, k
    d.stride, d.pad, d.Ho, d.Wo = 1, k // 2, H, W
    d.in_ld = Cin
    d.res_ld = Cout if res else 0
    d.UH, d.UW = ((H + 1) // 2, (W + 1) // 2) if ups else (0, 0)
    ld = Cout if ld is None else ld
    d.out_n_stride, d.out_h_stride, d.out_w_stride = H * W * ld, W * ld, ld
    for name, v in kw.items():
        setattr(d, name, v)
    return d


def rows(d):
    d.out_h_stride = d.Wo * d.out_w_stride + 8 * d.out_w_stride      # pixel rows with a gap after every image row
    d.out_n_stride = d.Ho * d.out_h_stride
    return d


# (id, descriptor, accepted)
CASES = [
    ("base_f16", desc(), True),
    ("base_tf32", desc(f16=False, Cin=32), True),
    # K-step of 64 fp16 / 32 fp32 channels
    ("cin32_f16", desc(Cin=32), False),
    ("cin96_f16", desc(Cin=96), False),
    ("cin128_f16", desc(Cin=128), True),
    ("cin48_tf32", desc(f16=False, Cin=48), False),
    ("cin96_tf32", desc(f16=False, Cin=96), True),
    ("in_dtype2", desc(in_dtype=2), False),
    ("in_ld_f16_not8", desc(Cin=64, in_ld=68), False),
    ("in_ld_f16_8", desc(Cin=64, in_ld=72), True),
    ("in_ld_tf32_not4", desc(f16=False, Cin=32, in_ld=34), False),
    ("in_ld_tf32_4", desc(f16=False, Cin=32, in_ld=36), True),
    # rows at least Cin wide: a shorter row would read the next pixel's channels
    ("in_ld_short_f16", desc(Cin=128, in_ld=120), False),
    ("in_ld_full_f16", desc(Cin=128, in_ld=128), True),
    ("in_ld_short_tf32", desc(f16=False, Cin=64, in_ld=60), False),
    ("in_ld_full_tf32", desc(f16=False, Cin=64, in_ld=64), True),
    ("no_outputs", desc(out=None, twin=False), False),
    ("twin_only", desc(out=None), True),
    ("fp32_only", desc(twin=False), True),
    ("null_in", desc(in_=None), False),
    ("null_wgt", desc(wgt=None), False),
    # Cout
    ("cout_not4", desc(Cout=98), False),
    ("cout_4", desc(Cout=4), True),
    ("cout_2052", desc(Cout=2052), False),
    ("cout_2048", desc(Cout=2048), True),
    # kernel shape, padding, stride
    ("k3_pad1", desc(k=3), True),
    ("k3_pad0", desc(k=3, pad=0), False),
    ("k1_pad1", desc(k=1, pad=1), False),
    ("k5_pad2", desc(k=5), False),
    ("k1x3", desc(kw=3), False),
    ("stride2", desc(stride=2, Ho=3, Wo=4), False),
    ("stride1_ho_ne_h", desc(Ho=4), False),
    # residual: flat 1x1 rows only, never with an upsample
    ("res_k1", desc(res=True), True),
    ("res_k3", desc(res=True, k=3), False),
    ("res_up", desc(res=True, ups=True), False),
    ("up_k3", desc(ups=True, k=3), True),
    ("up_k1", desc(ups=True), True),
    ("res_ld_not4", desc(res=True, res_ld=98), False),
    ("res_ld_wide", desc(res=True, res_ld=104), True),
    ("res_misaligned", desc(res=True, residual=A_RES + 8), False),
    ("res_aligned16", desc(res=True, residual=A_RES + 16), True),
    # alignment of every pointer and stride
    ("in_misaligned", desc(in_=A_IN + 8), False),
    ("in_aligned16", desc(in_=A_IN + 16), True),
    ("wgt_misaligned", desc(wgt=A_W + 8), False),
    ("wgt_aligned16", desc(wgt=A_W + 16), True),
    ("out_misaligned", desc(out=A_OUT + 8), False),
    ("out_aligned16", desc(out=A_OUT + 16), True),
    ("out16_misaligned4", desc(out16=A_OUT16 + 4), False),
    ("out16_aligned8", desc(out16=A_OUT16 + 8), True),
    ("scale_misaligned", desc(scale=A_SC + 8), False),
    ("scale_null", desc(scale=None), True),
    ("shift_misaligned", desc(shift=A_SH + 4), False),
    ("shift_null", desc(shift=None), True),
    ("up_misaligned", desc(ups=True, up_src=A_UP + 8), False),
    ("up_aligned16", desc(ups=True, up_src=A_UP + 16), True),
    ("out_coff_not4", desc(ld=104, out_coff=2), False),
    ("out_coff_4", desc(ld=104, out_coff=4), True),
    ("w_stride_not4", desc(out_w_stride=98, out_h_stride=7 * 98, out_n_stride=35 * 98), False),
    ("w_stride_4", desc(out_w_stride=100, out_h_stride=7 * 100, out_n_stride=35 * 100), True),
    ("h_stride_not4", desc(out_h_stride=7 * 96 + 2, out_n_stride=5 * (7 * 96 + 2)), False),
    ("h_stride_4", desc(out_h_stride=7 * 96 + 4, out_n_stride=5 * (7 * 96 + 4)), True),
    ("n_stride_not4", desc(out_n_stride=35 * 96 + 2), False),
    ("n_stride_4", desc(out_n_stride=35 * 96 + 4), True),
    # 32-bit index ranges
    ("out_index_2g", desc(N=2, out_n_stride=1 << 30), False),
    ("out_index_1g", desc(N=2, out_n_stride=(1 << 30) - 4096), True),
    ("up_index_2g", desc(ups=True, N=1, Cout=256, UH=4096, UW=4096), False),
    ("up_index_1g", desc(ups=True, N=1, Cout=256, UH=2048, UW=2048), True),
    ("pixels_2g", desc(N=1, H=65536, W=32768, out_n_stride=0, out_h_stride=0, out_w_stride=0), False),
    ("pixels_1g", desc(N=1, H=32768, W=32768, out_n_stride=0, out_h_stride=0, out_w_stride=0), True),
    # TMA residual epilogue (fp16 forward): output pixels are rows of one pitch, the twin 16-byte addressable
    ("tma_res_gapped_rows_f16", rows(desc(res=True)), False),
    ("tma_res_gapped_rows_tf32", rows(desc(f16=False, Cin=32, res=True)), True),
    ("tma_res_gapped_rows_no_res", rows(desc()), True),
    ("tma_res_gapped_images_f16", desc(res=True, out_n_stride=35 * 96 + 96), False),
    ("tma_res_single_image_any_n_stride", desc(res=True, N=1, out_n_stride=35 * 96 + 96), True),
    ("tma_res_single_row_any_h_stride", desc(res=True, H=1, out_h_stride=7 * 96 + 96), True),
    ("tma_res_wide_rows_coff", desc(res=True, ld=136, out_coff=32), True),
    ("tma_res_twin_w_stride_not8", desc(res=True, ld=100), False),
    ("tma_res_fp32_only_w_stride_4", desc(res=True, ld=100, twin=False), True),
    ("tma_res_twin_coff_not8", desc(res=True, ld=104, out_coff=4), False),
    ("tma_res_twin_coff_8", desc(res=True, ld=104, out_coff=8), True),
    ("tma_res_twin_misaligned", desc(res=True, out16=A_OUT16 + 8), False),
    ("tma_res_twin_aligned16", desc(res=True, out16=A_OUT16 + 16), True),
    ("no_res_twin_coff_4", desc(ld=104, out_coff=4), True),
    # ... and the twin's rows a whole number of 16-byte units (the bulk store wrote past Cout = 36 otherwise)
    ("tma_res_twin_cout_not8", desc(res=True, Cout=36, ld=48, out_coff=8), False),
    ("tma_res_twin_cout_8", desc(res=True, Cout=40, ld=48, out_coff=8), True),
    ("tma_res_fp32_only_cout_not8", desc(res=True, Cout=36, ld=48, out_coff=8, twin=False), True),
    ("no_res_twin_cout_not8", desc(Cout=36, ld=48, out_coff=8), True),
]


@pytest.mark.parametrize("name,d,ok", CASES, ids=[c[0] for c in CASES])
def test_tc_supported_rules(lib, name, d, ok):
    assert lib.sb_conv2d_tc_supported(ctypes.byref(d)) == (1 if ok else 0), name


def test_simt_rejects_fp16_descriptors_before_launch(lib):
    """the SIMT kernel reads fp32 operands and writes the fp32 output only; an fp16 descriptor or a twin is refused
    with SB_EINVAL (-22) before any launch (no device is needed to get the answer)"""
    for d in (desc(), rows(desc(res=True)), desc(f16=False, Cin=32, twin=True), desc(out=None)):
        assert lib.sb_conv2d_simt(ctypes.byref(d), None) == -22


def test_simt_rejects_short_rows_before_launch(lib):
    """an fp32 descriptor whose input rows are narrower than Cin is refused with SB_EINVAL before any launch"""
    d = desc(f16=False, Cin=32, in_ld=28)
    assert lib.sb_conv2d_simt(ctypes.byref(d), None) == -22


def test_auto_dispatch_raises_for_rejected_fp16(lib):
    """conv2d(desc, "auto") never hands an fp16 descriptor to the SIMT kernel"""
    for d in (rows(desc(res=True)), desc(Cin=96), desc(stride=2, Ho=3, Wo=4)):
        assert lib.sb_conv2d_tc_supported(ctypes.byref(d)) == 0
        with pytest.raises(L.SbError):
            G.conv2d(d, "auto")


def test_conv_desc_residual_pitch_from_strides():
    """res_ld is the residual's pixel pitch, not its channel count; a residual whose pixels are not rows of one
    pitch is refused"""
    N, H, W, C = 2, 3, 5, 32
    x = torch.zeros(N, H, W, 64, dtype=torch.float16)
    w = torch.zeros(C, 1, 1, 64, dtype=torch.float16)
    out = torch.zeros(N, H, W, C)
    big = torch.zeros(N, H, W, C + 8)
    d = G.conv_desc(x, w, out, 64, C, 1, 1, 1, 0, H, W, residual=big[..., :C])
    assert d.res_ld == C + 8 and d.residual == big.data_ptr()
    d = G.conv_desc(x, w, out, 64, C, 1, 1, 1, 0, H, W, residual=big[..., 8:])
    assert d.res_ld == C + 8 and d.residual == big.data_ptr() + 32
    d = G.conv_desc(x, w, out, 64, C, 1, 1, 1, 0, H, W, residual=torch.zeros(N, H, W, C))
    assert d.res_ld == C
    # one image of a batch: still flat rows
    d = G.conv_desc(x[:1], w, out[:1], 64, C, 1, 1, 1, 0, H, W, residual=torch.zeros(2, H, W, C)[1:])
    assert d.res_ld == C
    # 1x1 images (an FC as a conv): an NCHW tensor permuted to NHWC has arbitrary strides on its size-1 dimensions
    x1 = torch.zeros(4, 1, 1, 64, dtype=torch.float16)
    r1 = torch.zeros(4, C + 8, 1, 1).permute(0, 2, 3, 1)[..., :C]
    d = G.conv_desc(x1, w, torch.zeros(4, 1, 1, C), 64, C, 1, 1, 1, 0, 1, 1, residual=r1)
    assert d.res_ld == C + 8
    for bad in (torch.zeros(N, H, W + 1, C)[:, :, :W], torch.zeros(N, H + 1, W, C)[:, :H],
                torch.zeros(N, H, W, 2 * C)[..., ::2]):
        with pytest.raises(AssertionError):
            G.conv_desc(x, w, out, 64, C, 1, 1, 1, 0, H, W, residual=bad)
