"""GPU: the TMA residual epilogue's per-warpgroup ring of column chunks (conv_tc.cu) over launches of many tiles per
CTA, against the register residual epilogue (sb_conv2d_tc_dgrad without a mask on the same descriptor), by
torch.equal on the whole guard-banded output buffers.

A CTA steps its ring through every chunk of every tile it runs, so a grid of 1 to 7 CTAs wraps the ring many times,
with the ring's slot count (4 at 128-wide tiles, 3 at 64 and 32) out of step with the chunks per tile (4, 2, 1).
Every case ends on an M tail; most leave the second warpgroup without rows in the last m-tile (<= 64 rows), and the
Cout tails leave chunks partly or wholly past Cout.  The first case is the layer-3 conv3 shape of one stereo pair
(M = 2 x 38 x 125, 256 -> 1024): 600 tiles on one CTA."""
import ctypes
import math

import pytest
import torch

from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import ops as G
from test_gpu_conv_tc import BM, SENT16, SENT32, layout_of, pick_bn

pytestmark = pytest.mark.gpu

# (N, H, W, Cin, Cout, max_ctas, output layout, outputs)
CASES = [
    (2, 38, 125, 256, 1024, 1, "dense", "both"),     # layer 3 conv3: 75 m-tiles x 8, last m-tile 28 rows
    (2, 38, 125, 256, 1024, 7, "slice", "both"),
    (1, 19, 63, 512, 200, 1, "dense", "both"),       # 10 m-tiles (last 45 rows) x 2; chunk 6 holds 8 columns
                                                     # of Cout, chunk 7 none
    (2, 19, 63, 512, 2048, 5, "dense", "f16"),       # layer 4 conv3: 19 m-tiles (last 90 rows) x 16
    (1, 13, 89, 64, 40, 1, "slice", "both"),         # 64-wide: 10 m-tiles, last 5 rows; chunk 1 is 8 columns
    (3, 38, 37, 1024, 64, 3, "dense", "f32"),        # 64-wide: 33 m-tiles, last 122 rows
    (3, 11, 37, 64, 24, 1, "slice", "both"),         # 32-wide: 10 m-tiles, last 69 rows, 24 of 32 columns
    (3, 13, 89, 1024, 32, 2, "dense", "f16"),        # 32-wide: 28 m-tiles, last 15 rows
]


def _id(c):
    N, H, W, Cin, Cout, mc, layout, outs = c
    return "%dx%dx%d-c%d-co%d-ctas%d-%s-%s" % (N, H, W, Cin, Cout, mc, layout, outs)


@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_residual_ring_matches_register_epilogue(case):
    N, H, W, Cin, Cout, max_ctas, layout, outs = case
    dev = "cuda"
    g = torch.Generator().manual_seed(1000 * Cout + Cin + max_ctas)
    M = N * H * W
    m_tiles = -(-M // BM)
    bn = pick_bn(Cout, m_tiles, None, True)
    x = torch.randn(N, H, W, Cin, generator=g).half().to(dev)
    w = (torch.randn(Cout, 1, 1, Cin, generator=g) / math.sqrt(Cin)).half().to(dev)
    scale = (torch.rand(Cout, generator=g) + 0.5).to(dev)
    shift = torch.randn(Cout, generator=g).to(dev)
    res = torch.randn(N, H, W, Cout, generator=g).to(dev)

    S, base, coff, st = layout_of(layout, N, H, W, Cout)
    want32, want16 = outs in ("both", "f32"), outs in ("both", "f16")
    buf32 = torch.empty(S, dtype=torch.int32, device=dev)
    buf16 = torch.empty(S, dtype=torch.int16, device=dev)

    def launch(entry):
        buf32.fill_(SENT32)
        buf16.fill_(SENT16)
        o32 = buf32.view(torch.float32)[base:] if want32 else None
        o16 = buf16.view(torch.float16)[base:] if want16 else None
        d = G.conv_desc(x, w, o32, Cin, Cout, 1, 1, 1, 0, H, W, scale=scale, shift=shift, residual=res,
                        out_coff=coff, out_strides=st, out16=o16, max_ctas=max_ctas)
        if entry == "dgrad":
            G.conv2d_dgrad(d, None)
        else:
            assert G.conv2d(d, "tc") == "tc"
        torch.cuda.synchronize()
        return buf32.clone(), buf16.clone()

    lib = L.load()
    tbuf = torch.zeros(lib.sb_conv_trace_bytes(4), dtype=torch.uint8, device=dev)
    assert lib.sb_conv_trace(ctypes.c_void_p(tbuf.data_ptr()), 4) == 0
    try:
        ring32, ring16 = launch("tc")
        reg32, reg16 = launch("dgrad")
        infos = []
        for i in range(lib.sb_conv_trace_count()):
            v = (ctypes.c_int * 12)()
            assert lib.sb_conv_trace_info(i, v) == 0
            infos.append(list(v))
    finally:
        lib.sb_conv_trace(None, 0)

    # both launches ran the tile width and grid the case claims: the first on the TMA epilogue (fp16 forward)
    tiles = m_tiles * -(-Cout // bn)
    assert [(v[4], v[5], v[9], v[10]) for v in infos] == [(bn, tiles, 1, max_ctas), (bn, tiles, 3, max_ctas)]
    assert tiles >= 10 * max_ctas, "the case must run many tiles per CTA"

    # the register epilogue wrote every logical element (and the ring path must match it byte for byte)
    n_i = torch.arange(N, device=dev).view(-1, 1, 1, 1) * st[0]
    h_i = torch.arange(H, device=dev).view(1, -1, 1, 1) * st[1]
    w_i = torch.arange(W, device=dev).view(1, 1, -1, 1) * st[2]
    idx = (base + coff + n_i + h_i + w_i + torch.arange(Cout, device=dev).view(1, 1, 1, -1)).reshape(-1)
    if want32:
        assert bool(torch.isfinite(reg32.view(torch.float32)[idx]).all())
    if want16:
        assert bool(torch.isfinite(reg16.view(torch.float16)[idx]).all())
    assert torch.equal(ring32, reg32), "fp32 output differs from the register epilogue"
    assert torch.equal(ring16, reg16), "fp16 twin differs from the register epilogue"
