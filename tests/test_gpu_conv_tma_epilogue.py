"""GPU: the plain TMA epilogue of the tensor-core conv kernel (conv_tc.cu) against the register epilogue, bit for bit.

fp16-operand forward convs without a residual or an upsample-add, on flat output rows (1x1, and 3x3 through the rows
entry), store their outputs through the per-warpgroup ring of 64-row x 32-column slots by TMA whenever the output is
a 2-D [ld, M] map (tma_epilogue_layout_ok).  The reference is the same descriptor through the data-gradient entry
with an all-ones mask, which runs the register epilogue (cooperative) and leaves every value as it is.  Each case runs
one tile per CTA (cooperative), about two tiles per CTA (ping-pong where the width allows) and three CTAs (the ring
wraps many times); the whole guard-banded output buffers must be identical.

The cases cover 32/64/128/256-wide tiles, fp32-only, fp16-only and both outputs, M tails (also a last tile whose
second 64-row half is empty) and Cout tails, a channel slice, the RPN_Conv L|R half at channel offset 512 and the
flat-row 3x3 entry.  Layouts the rule rejects (a deconv phase's strided pixels, a twin with Cout % 8 != 0) must run
the register epilogue and give the same bits."""
import collections
import ctypes
import math
import zlib

import pytest
import torch

from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import ops as G
from test_gpu_conv_tc import BM, SENT16, SENT32, layout_of, num_sms, pick_bn

pytestmark = pytest.mark.gpu

W_SCHED = 7                    # per-CTA trace word: schedule (1: ping-pong)

Case = collections.namedtuple("Case", "id k N H W Cin Cout env layout outs")
CASES = [
    Case("k1-bn32-f16-wg1-empty", 1, 1, 10, 70, 64, 32, None, "dense", "f16"),       # M = 700: last tile 60 rows
    Case("k1-bn32-f32-cout24", 1, 1, 13, 77, 128, 24, None, "slice", "f32"),
    Case("k1-bn64-both-cout40", 1, 2, 9, 61, 192, 40, None, "slice", "both"),
    Case("k1-bn64-f32", 1, 1, 17, 45, 320, 64, None, "dense", "f32"),
    Case("k1-bn128-f16-cout96", 1, 1, 19, 53, 512, 96, None, "dense", "f16"),      # chunk 3 past Cout
    Case("k1-bn128-both", 1, 1, 20, 50, 64, 128, None, "dense", "both"),
    Case("k1-bn128-f16-slice", 1, 2, 5, 83, 256, 200, None, "slice", "f16"),
    Case("k1-bn256-f16", 1, 1, 10, 70, 256, 512, 256, "dense", "f16"),
    Case("k1-bn256-both-cout328", 1, 1, 9, 61, 512, 328, 256, "dense", "both"),   # 3 operand stages, Cout tail
    Case("k1-bn256-f32", 1, 1, 21, 38, 128, 256, 256, "slice", "f32"),
    Case("k3-rows-bn64-both", 3, 1, 19, 53, 64, 64, None, "dense", "both"),
    Case("k3-rows-bn128-f16", 3, 2, 7, 45, 64, 128, None, "slice", "f16"),
    Case("k3-rows-bn256-rpn-half", 3, 1, 15, 49, 256, 512, 256, "rpn", "f16"),      # RPN_Conv R half: coff 512
    # layouts the rule rejects: register epilogue
    Case("k1-bn64-scatter-reject", 1, 1, 11, 70, 64, 64, None, "scatter1", "both"),
    Case("k1-bn64-cout36-twin-reject", 1, 1, 11, 70, 64, 36, None, "slice", "f16"),
    Case("k3-rows-bn128-scatter-reject", 3, 1, 9, 40, 64, 128, None, "scatter1", "f16"),
]


def layout(kind, N, Ho, Wo, Cout):
    if kind == "rpn":             # channels [512, 1024) of 1024-wide rows, the R half of the RPN_Conv concat
        lead, trail, ld, coff = 3, 5, 1024, 512
        return lead * ld + N * Ho * Wo * ld + trail * ld, lead * ld, coff, (Ho * Wo * ld, Wo * ld, ld)
    return layout_of(kind, N, Ho, Wo, Cout)


def tma_expected(c, want32, want16, bn, tiles, grid):
    if c.layout == "scatter1" or (want16 and c.Cout % 8):
        return False
    # a 128-wide TMA epilogue with an fp32 box has no ping-pong twin: with a second tile per CTA the register one runs
    return not (want32 and bn == 128 and tiles > grid)


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_tma_epilogue_matches_register_epilogue(case, monkeypatch):
    c = case
    g = torch.Generator().manual_seed(zlib.crc32(c.id.encode()))
    dev = "cuda"
    N, H, W, Cin, Cout, k = c.N, c.H, c.W, c.Cin, c.Cout, c.k
    x = torch.randn(N, H, W, Cin, generator=g).half().to(dev)
    w = (torch.randn(Cout, k, k, Cin, generator=g) / math.sqrt(k * k * Cin)).half().to(dev)
    scale = (torch.rand(Cout, generator=g) + 0.5).to(dev)
    shift = torch.randn(Cout, generator=g).to(dev)
    S, base, coff, st = layout(c.layout, N, H, W, Cout)
    want32, want16 = c.outs in ("both", "f32"), c.outs in ("both", "f16")
    buf32 = torch.empty(S, dtype=torch.int32, device=dev)
    buf16 = torch.empty(S, dtype=torch.int16, device=dev)
    ones = torch.ones(S, dtype=torch.float16, device=dev)
    if c.env is None:
        monkeypatch.delenv("SB_TC_BLOCK_N", raising=False)
    else:
        monkeypatch.setenv("SB_TC_BLOCK_N", str(c.env))

    m_tiles = -(-(N * H * W) // BM)
    bn = pick_bn(Cout, m_tiles, c.env, False)
    tiles = m_tiles * -(-Cout // bn)
    sms = num_sms()
    grids = [min(tiles, sms), -(-tiles // 2), 3]

    def launch(entry, max_ctas=0):
        buf32.fill_(SENT32)
        buf16.fill_(SENT16)
        o32 = buf32.view(torch.float32)[base:] if want32 else None
        o16 = buf16.view(torch.float16)[base:] if want16 else None
        d = G.conv_desc(x, w, o32, Cin, Cout, k, k, 1, k // 2, H, W, scale=scale, shift=shift, relu=False,
                        out_coff=coff, out_strides=st, out16=o16, max_ctas=max_ctas)
        if entry == "dgrad":
            G.conv2d_dgrad(d, ones[base:])
        elif k == 3:
            G.conv2d_rows(d)
        else:
            assert G.conv2d(d, "tc") == "tc"
        torch.cuda.synchronize()
        return buf32.clone(), buf16.clone()

    lib = L.load()
    tbuf = torch.zeros(lib.sb_conv_trace_bytes(len(grids) + 1) // 8, dtype=torch.int64, device=dev)
    assert lib.sb_conv_trace(ctypes.c_void_p(tbuf.data_ptr()), len(grids) + 1) == 0
    try:
        ref32, ref16 = launch("dgrad")
        outs = [launch("fwd", mc) for mc in grids]
        infos, epis = [], []
        for i in range(lib.sb_conv_trace_count()):
            v = (ctypes.c_int * 12)()
            assert lib.sb_conv_trace_info(i, v) == 0
            infos.append(list(v))
            epis.append(lib.sb_conv_trace_epilogue(i))
    finally:
        lib.sb_conv_trace(None, 0)
    # (the reference of a 3x3 runs on 8x16 patches: the data-gradient entry has no flat-row tiles)
    assert [(v[4], v[5], v[10]) for v in infos[1:]] == [(bn, tiles, mc) for mc in grids]
    assert epis[0] == 0, "the data-gradient entry runs the register epilogue"
    tr = tbuf.view(len(grids) + 1, -1, 16).cpu()
    for i, mc in enumerate(grids):
        grid = min(tiles, mc)
        assert epis[i + 1] == int(tma_expected(c, want32, want16, bn, tiles, grid)), (c.id, mc)
        pp = tiles > grid and bn <= 128
        assert bool((tr[i + 1, :grid, W_SCHED] == int(pp)).all()), (c.id, mc)

    # the reference wrote every logical element
    n_i = torch.arange(N, device=dev).view(-1, 1, 1, 1) * st[0]
    h_i = torch.arange(H, device=dev).view(1, -1, 1, 1) * st[1]
    w_i = torch.arange(W, device=dev).view(1, 1, -1, 1) * st[2]
    idx = (base + coff + n_i + h_i + w_i + torch.arange(Cout, device=dev).view(1, 1, 1, -1)).reshape(-1)
    written = torch.zeros(S, dtype=torch.bool, device=dev)
    written[idx] = True
    if want32:
        assert bool((ref32[~written] == SENT32).all()) and bool(torch.isfinite(ref32.view(torch.float32)[idx]).all())
    if want16:
        assert bool((ref16[~written] == SENT16).all()) and bool(torch.isfinite(ref16.view(torch.float16)[idx]).all())

    for mc, (o32, o16) in zip(grids, outs):
        assert torch.equal(o32, ref32), "%s: fp32 output with max_ctas=%d differs from the register epilogue" % (c.id, mc)
        assert torch.equal(o16, ref16), "%s: fp16 output with max_ctas=%d differs from the register epilogue" % (c.id, mc)
