"""GPU: the 3x3 convolution on flat 128-pixel tiles loaded by TMA im2col (sb_conv2d_tc_rows) against the same
descriptor on 8x16 patches (sb_conv2d_tc), bit for bit.

Per output pixel both paths feed the tensor core the same A values in the same K order (tap-major, then Cin chunks)
and run the same epilogue, so every output byte must match: torch.equal on the fp32 and fp16 buffers, guard bands
included (the patch path itself is held to float64 by test_gpu_conv_tc.py).  The cases put tiles across row and image
boundaries, use maps of one row, one column and one pixel, the keypoint-head shape [300, 14, 14], last m-tiles of
1, 64, 65, 127 and 128 rows, Cout tails at tile widths 32 / 64 / 128 / 256, and the dense, channel-slice, RPN L|R
concat (image n -> channel offset 512 n) and deconv-scatter output layouts.  The traced launch has the flat tile
count ceil(M / 128) * ceil(Cout / BN), the result does not depend on the grid size (max_ctas 1 and 3) or, for
Cout >= 256, on the tile width, and descriptors outside the entry point's domain are SB_EINVAL with nothing written."""
import collections
import ctypes
import zlib

import pytest
import torch

from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import ops as G

pytestmark = pytest.mark.gpu

SENT32 = 0x7FA5A5A5            # NaN bit patterns the kernels never produce
SENT16 = 0x7E5A
BM = 128
SB_EINVAL = -22
Case = collections.namedtuple("Case", "id N H W Cin Cout layout outs relu env")


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def pick_bn(cout, m_tiles, env):
    """conv_tc.cu pick_block_n + SB_TC_BLOCK_N"""
    if cout <= 32:
        bn = 32
    elif cout <= 64:
        bn = 64
    elif cout < 256:
        bn = 128
    else:
        sms = num_sms()
        t128, t256 = m_tiles * -(-cout // 128), m_tiles * -(-cout // 256)
        bn = 256 if -(-t256 // sms) * 1024 <= -(-t128 // sms) * 512 else 128
    return env if env in (128, 256) and cout >= 256 else bn


def _cases():
    out = []

    def add(N, H, W, Cin, Cout, layout, outs, relu, env=None):
        cid = "%dx%dx%d-c%d-co%d-%s-%s%s%s" % (N, H, W, Cin, Cout, layout, outs, "-relu" if relu else "",
                                              "" if env is None else "-bn%d" % env)
        out.append(Case(cid, N, H, W, Cin, Cout, layout, outs, relu, env))

    # last m-tile of 1, 64, 65, 127, 128 rows, tiles across row and image boundaries, Cout tails at every width
    add(3, 1, 43, 64, 24, "dense", "both", True)            # M = 129: last tile 1 row; H = 1
    add(3, 8, 8, 64, 40, "slice", "f16", False)             # M = 192: 64 rows; three images in a tile
    add(1, 1, 193, 128, 100, "scatter", "f32", True)        # M = 193: 65 rows; one row across tiles
    add(5, 3, 17, 64, 260, "slice", "both", False, 256)     # M = 255: 127 rows; image boundaries inside tiles
    add(1, 16, 16, 192, 36, "dense", "both", True)          # M = 256: 128 rows
    add(2, 70, 1, 64, 64, "dense", "f32", False)            # W = 1
    add(4, 1, 1, 64, 132, "slice", "both", True)            # 1x1 images
    add(3, 5, 13, 64, 516, "scatter", "both", True, 256)    # M = 195: 3 images of 65 px across 2 tiles
    add(2, 37, 29, 128, 200, "dense", "f16", True)          # M = 2146: 98 rows
    add(1, 9, 17, 64, 32, "scatter", "f16", False)          # M = 153, full 32-wide tile
    add(2, 19, 63, 512, 512, "dense", "f16", True)          # layer 4 conv2 of one pair
    add(2, 23, 31, 256, 512, "lrcat", "f16", True)          # RPN_Conv, L and R in one launch
    add(2, 11, 9, 256, 512, "lrcat", "both", False, 128)
    add(300, 14, 14, 256, 256, "dense", "both", True)       # keypoint head, fp32 + fp16 outputs
    add(300, 14, 14, 256, 256, "dense", "f16", True, 128)
    add(7, 14, 14, 256, 256, "scatter", "f16", True)        # a few RoIs of the head into a deconv-like scatter
    return out


CASES = _cases()


def layout_of(kind, N, Ho, Wo, Cout):
    """-> (elements, base, coff, (n, h, w) strides) of an output inside a guard-banded buffer"""
    lead, trail = 3, 5
    if kind == "dense":
        ld, coff = Cout, 0
        st, ext, off = (Ho * Wo * ld, Wo * ld, ld), N * Ho * Wo * ld, 0
    elif kind == "slice":             # channel slice of wider rows
        coff = 8
        ld = -(-(Cout + coff + 4) // 8) * 8
        st, ext, off = (Ho * Wo * ld, Wo * ld, ld), N * Ho * Wo * ld, 0
    elif kind == "lrcat":             # RPN L|R concat: one [Ho, Wo, N * Cout] map, image n at channel n * Cout
        ld, coff = N * Cout, 0
        st, ext, off = (Cout, Wo * ld, ld), Ho * Wo * ld, 0
    else:                             # odd pixels of a 2Ho x 2Wo image: the 2x2 deconv scatter
        ld, coff = Cout, 0
        st, ext = (4 * Ho * Wo * ld, 2 * 2 * Wo * ld, 2 * ld), N * 4 * Ho * Wo * ld
        off = (2 * Wo + 1) * ld
    return lead * ld + ext + trail * ld, lead * ld + off, coff, st


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_rows_match_patches(case, monkeypatch):
    c = case
    g = torch.Generator().manual_seed(zlib.crc32(c.id.encode()))
    dev = "cuda"
    N, H, W, Cin, Cout = c.N, c.H, c.W, c.Cin, c.Cout
    M = N * H * W
    x = torch.randn(N, H, W, Cin, generator=g).half().to(dev)
    w = (torch.randn(Cout, 3, 3, Cin, generator=g) / (3 * Cin ** 0.5)).half().to(dev)
    scale = (torch.rand(Cout, generator=g) + 0.5).to(dev)
    shift = torch.randn(Cout, generator=g).to(dev)
    S, base, coff, st = layout_of(c.layout, N, H, W, Cout)
    want32, want16 = c.outs in ("both", "f32"), c.outs in ("both", "f16")
    buf32 = torch.empty(S, dtype=torch.int32, device=dev)
    buf16 = torch.empty(S, dtype=torch.int16, device=dev)
    idx = (base + coff + torch.arange(N, device=dev).view(-1, 1, 1, 1) * st[0] +
           torch.arange(H, device=dev).view(1, -1, 1, 1) * st[1] + torch.arange(W, device=dev).view(1, 1, -1, 1) * st[2] +
           torch.arange(Cout, device=dev).view(1, 1, 1, -1)).reshape(-1)
    lib = L.load()

    def launch(rows, env=None, max_ctas=0):
        buf32.fill_(SENT32)
        buf16.fill_(SENT16)
        if env is None:
            monkeypatch.delenv("SB_TC_BLOCK_N", raising=False)
        else:
            monkeypatch.setenv("SB_TC_BLOCK_N", str(env))
        o32 = buf32.view(torch.float32)[base:] if want32 else None
        o16 = buf16.view(torch.float16)[base:] if want16 else None
        d = G.conv_desc(x, w, o32, Cin, Cout, 3, 3, 1, 1, H, W, scale=scale, shift=shift, relu=c.relu, out_coff=coff,
                        out_strides=st, out16=o16, max_ctas=max_ctas)
        if rows:
            G.conv2d_rows(d)
        else:
            assert G.conv2d(d, "tc") == "tc"
        torch.cuda.synchronize()
        return buf32.clone(), buf16.clone()

    m_tiles = -(-M // BM)
    bn = pick_bn(Cout, m_tiles, c.env)
    tiles = m_tiles * -(-Cout // bn)
    tbuf = torch.zeros(lib.sb_conv_trace_bytes(16), dtype=torch.uint8, device=dev)
    assert lib.sb_conv_trace(ctypes.c_void_p(tbuf.data_ptr()), 16) == 0
    launches = []                      # expected (BLOCK_N, max_ctas) of every traced rows launch
    try:
        p32, p16 = launch(False, env=c.env)
        r32, r16 = launch(True, env=c.env)
        launches.append((bn, 0))
        same = []
        if tiles <= 400:
            for mc in (1, 3):
                same.append(("max_ctas=%d" % mc, launch(True, env=c.env, max_ctas=mc)))
                launches.append((bn, mc))
        if Cout >= 256:
            other = 128 if bn == 256 else 256
            same.append(("BLOCK_N=%d" % other, launch(True, env=other)))
            launches.append((other, 0))
        infos = []
        for i in range(lib.sb_conv_trace_count()):
            v = (ctypes.c_int * 12)()
            assert lib.sb_conv_trace_info(i, v) == 0
            infos.append(list(v))
    finally:
        lib.sb_conv_trace(None, 0)
        monkeypatch.delenv("SB_TC_BLOCK_N", raising=False)

    # the first traced launch is the patch path; the rest are rows launches with the flat tile count
    assert len(infos) == 1 + len(launches), (infos, launches)
    for v, (b, mc) in zip(infos[1:], launches):
        assert v == [Cin, Cout, 3, M, b, m_tiles * -(-Cout // b), 9 * Cin // 64, 0, 0, 1, mc, N], (c.id, v)

    # every logical element written (the patch path is checked against float64 elsewhere)
    if want32:
        assert bool((r32[idx] != SENT32).all()), "fp32 output: elements not written"
    if want16:
        assert bool((r16[idx] != SENT16).all()), "fp16 twin: elements not written"
    assert torch.equal(r32, p32), (c.id, "fp32 output differs from the patch path")
    assert torch.equal(r16, p16), (c.id, "fp16 twin differs from the patch path")
    for name, (s32, s16) in same:
        assert torch.equal(s32, r32), (c.id, name, "fp32")
        assert torch.equal(s16, r16), (c.id, name, "twin")
    print("%-48s tiles %d -> %d (BN %d) | %s" % (c.id, N * -(-H // 8) * -(-W // 16) * -(-Cout // bn), tiles, bn,
                                                  ", ".join(n for n, _ in same)))


def test_case_list_covers_the_edges():
    assert {(c.N * c.H * c.W) % BM or BM for c in CASES} >= {1, 64, 65, 127, 128}
    assert any(c.H == 1 and c.W > 1 for c in CASES) and any(c.W == 1 and c.H > 1 for c in CASES)
    assert any(c.H == 1 and c.W == 1 for c in CASES)
    assert any((c.N, c.H, c.W, c.Cin, c.Cout) == (300, 14, 14, 256, 256) for c in CASES)
    # a tile that holds pixels of two images, and one that starts inside a row
    assert any(c.N > 1 and c.H * c.W % BM and c.N * c.H * c.W > BM for c in CASES)
    assert {c.layout for c in CASES} == {"dense", "slice", "lrcat", "scatter"}
    assert {c.outs for c in CASES} == {"both", "f32", "f16"} and {c.relu for c in CASES} == {True, False}


def test_cout_tails_at_every_width():
    """each tile width 32 / 64 / 128 / 256 has a case whose Cout is not a multiple of it (the width depends on the
    SM count)"""
    widths = {}
    for c in CASES:
        bn = pick_bn(c.Cout, -(-(c.N * c.H * c.W) // BM), c.env)
        widths.setdefault(bn, []).append(c.Cout % bn != 0)
    assert all(any(widths.get(bn, [])) for bn in (32, 64, 128, 256)), widths


def test_rows_rejects_outside_its_domain():
    """SB_EINVAL before any launch (nothing written) for a residual, an upsample source, TF32 operands, a 1x1 conv,
    a stride-2 conv, and for what sb_conv2d_tc itself rejects (Cin % 64 != 0)"""
    dev = "cuda"
    lib = L.load()
    N, H, W, C = 1, 6, 10, 64
    x16 = torch.randn(N, H, W, C, device=dev).half()
    x32 = torch.randn(N, H, W, C, device=dev)
    w16 = torch.randn(C, 3, 3, C, device=dev).half()
    w32 = torch.randn(C, 3, 3, C, device=dev)
    w1 = torch.randn(C, 1, 1, C, device=dev).half()
    res = torch.randn(N, H, W, C, device=dev)
    up = torch.randn(N, 3, 5, C, device=dev)
    out = torch.full((N, H, W, C), 7.0, device=dev)
    x48 = torch.randn(N, H, W, 48, device=dev).half()
    w48 = torch.randn(C, 3, 3, 48, device=dev).half()
    descs = {
        "residual": G.conv_desc(x16, w16, out, C, C, 3, 3, 1, 1, H, W, residual=res),
        "up_src": G.conv_desc(x16, w16, out, C, C, 3, 3, 1, 1, H, W, up_src=up),
        "tf32": G.conv_desc(x32, w32, out, C, C, 3, 3, 1, 1, H, W),
        "1x1": G.conv_desc(x16, w1, out, C, C, 1, 1, 1, 0, H, W),
        "stride2": G.conv_desc(x16, w16, out, C, C, 3, 3, 2, 1, H // 2, W // 2),
        "cin48": G.conv_desc(x48, w48, out, 48, C, 3, 3, 1, 1, H, W),
    }
    for name, d in descs.items():
        assert lib.sb_conv2d_tc_rows(ctypes.byref(d), L.stream_ptr()) == SB_EINVAL, name
    assert lib.sb_conv2d_tc_rows(None, L.stream_ptr()) == SB_EINVAL
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())
