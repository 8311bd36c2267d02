"""GPU: the ping-pong schedule of the tensor-core conv kernel (conv_tc.cu) against the cooperative one, bit for bit.

Under the ping-pong schedule a CTA's j-th tile belongs to consumer warpgroup j & 1, which computes all 128 rows.  The
host picks it for fp16 operands with the register epilogue and tiles of at most 128 columns (64 with the
upsample-add) whenever some CTA gets a second tile.  Each case launches one descriptor with
max_ctas = tiles (one tile per CTA: cooperative), then again with max_ctas chosen so that CTAs get 2 tiles, 3 tiles,
and mixed 1 / 2 tiles (most CTAs' second warpgroup without a tile).  Every output element sums the same K-steps in
the same order either way, so the output buffers -- NaN-sentinel guard bands included -- must be identical.

The cases cover num_k_blocks of 1, 3, 5, 8, 9, 10 and 18 against each width's stage count (9 at 32 columns, 8 at 64,
6 at 128), M tails inside the last tile, Cout tails, flat rows, 8x16 patches, the flat-row 3x3 entry
(sb_conv2d_tc_rows), the upsample-add, fp32 and fp16 outputs, channel offsets and strided (scattered) outputs.  The per-CTA trace words show which schedule each launch ran and how many tiles each
warpgroup computed."""
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
BM, TW, TH = 128, 16, 8
TRACE_WORDS, TRACE_CTAS = 16, 304
W_SCHED, W_TILES = 7, 14       # per-CTA trace words: schedule (1: ping-pong), tiles of warpgroups 0 and 1

Case = collections.namedtuple("Case", "id entry k N H W Cin Cout up layout outs relu")
CASES = [
    # flat 1x1 rows: num_k_blocks 1 / 3 / 5 / 8 / 9 / 10 at each width, M and Cout tails
    Case("k1-kb1-bn128", "tc", 1, 1, 20, 50, 64, 128, None, "dense", "both", True),
    Case("k1-kb3-bn128-cout100", "tc", 1, 2, 9, 61, 192, 100, None, "slice", "f16", False),
    Case("k1-kb5-bn64", "tc", 1, 1, 17, 45, 320, 64, None, "dense", "f32", True),
    Case("k1-kb1-bn32-cout28", "tc", 1, 1, 13, 77, 64, 28, None, "slice", "both", False),
    Case("k1-kb10-bn64-cout40", "tc", 1, 1, 15, 51, 640, 40, None, "slice", "both", True),
    Case("k1-kb8-bn128-cout76", "tc", 1, 2, 5, 83, 512, 76, None, "dense", "f16", False),
    Case("k1-kb9-bn128-scatter", "tc", 1, 1, 11, 70, 576, 128, None, "scatter1", "both", True),
    Case("k1-kb9-bn32", "tc", 1, 1, 9, 99, 576, 32, None, "dense", "f16", True),
    # 3x3 on 8x16 patches (right and bottom patch tails)
    Case("k3-patch-kb9-bn128", "tc", 3, 1, 20, 37, 64, 128, None, "dense", "both", True),
    Case("k3-patch-kb9-bn64-cout48", "tc", 3, 2, 9, 30, 64, 48, None, "slice", "f16", False),
    # 3x3 on flat 128-pixel rows (TMA im2col)
    Case("k3-rows-kb9-bn128-cout96", "rows", 3, 1, 19, 53, 64, 96, None, "dense", "both", True),
    Case("k3-rows-kb18-bn32", "rows", 3, 1, 14, 61, 128, 32, None, "slice", "f32", False),
    Case("k3-rows-kb9-bn64", "rows", 3, 2, 7, 45, 64, 64, None, "scatter1", "both", True),
    # FPN lateral: 1x1 + bilinear upsample-add (patches); ping-pong at 64 columns, cooperative at 128
    Case("up-kb8-bn64", "tc", 1, 1, 21, 38, 512, 64, (11, 19), "dense", "both", False),
    Case("up-kb9-bn32-cout20", "tc", 1, 1, 17, 50, 576, 20, (9, 25), "slice", "f32", False),
    Case("up-kb3-bn64", "tc", 1, 1, 21, 38, 192, 64, (11, 19), "dense", "both", False),
    Case("up-kb8-bn128-cooperative", "tc", 1, 1, 21, 38, 512, 128, (11, 19), "dense", "both", False),
]


def block_n(cout):
    return 32 if cout <= 32 else 64 if cout <= 64 else 128        # conv_tc.cu pick_block_n below 256 columns


def pingpong_ok(bn, up):
    return bn <= (64 if up else 128)


def layout_of(kind, N, Ho, Wo, Cout):
    """-> (elements, base, coff, (n, h, w) strides) of an output inside a guard-banded buffer"""
    lead, trail = 3, 5
    if kind == "dense":
        ld, coff = Cout, 0
        st, ext, off = (Ho * Wo * ld, Wo * ld, ld), N * Ho * Wo * ld, 0
    elif kind == "slice":             # channel slice of wider rows (the RPN L|R concat)
        coff = 8
        ld = -(-(Cout + coff + 4) // 8) * 8
        st, ext, off = (Ho * Wo * ld, Wo * ld, ld), N * Ho * Wo * ld, 0
    else:                             # pixel (1, 1) of every 2x2 block of a 2Ho x 2Wo image: a deconv phase
        ld, coff = Cout, 0
        st, ext = (4 * Ho * Wo * ld, 2 * 2 * Wo * ld, 2 * ld), N * 4 * Ho * Wo * ld
        off = (2 * Wo + 1) * ld
    return lead * ld + ext + trail * ld, lead * ld + off, coff, st


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_pingpong_matches_cooperative(case):
    c = case
    g = torch.Generator().manual_seed(zlib.crc32(c.id.encode()))
    dev = "cuda"
    N, H, W, Cin, Cout, k = c.N, c.H, c.W, c.Cin, c.Cout, c.k
    x = torch.randn(N, H, W, Cin, generator=g).half().to(dev)
    w = (torch.randn(Cout, k, k, Cin, generator=g) / (k * Cin ** 0.5)).half().to(dev)
    up = torch.randn(N, c.up[0], c.up[1], Cout, generator=g).to(dev) if c.up else None
    scale = None if up is not None else (torch.rand(Cout, generator=g) + 0.5).to(dev)
    shift = torch.randn(Cout, generator=g).to(dev)
    S, base, coff, st = layout_of(c.layout, N, H, W, Cout)
    want32, want16 = c.outs in ("both", "f32"), c.outs in ("both", "f16")
    buf32 = torch.empty(S, dtype=torch.int32, device=dev)
    buf16 = torch.empty(S, dtype=torch.int16, device=dev)
    idx = (base + coff + torch.arange(N, device=dev).view(-1, 1, 1, 1) * st[0] +
           torch.arange(H, device=dev).view(1, -1, 1, 1) * st[1] + torch.arange(W, device=dev).view(1, 1, -1, 1) * st[2] +
           torch.arange(Cout, device=dev).view(1, 1, 1, -1)).reshape(-1)

    bn = block_n(Cout)
    patch = c.entry == "tc" and (k == 3 or up is not None)
    m_tiles = N * -(-H // TH) * -(-W // TW) if patch else -(-(N * H * W) // BM)
    tiles = m_tiles * -(-Cout // bn)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert 4 <= tiles <= sms, (c.id, tiles)
    # CTAs with one tile each (cooperative); two each (an odd count leaves the last CTA one); three each; all but
    # one CTA with a single tile
    grids = [tiles, -(-tiles // 2), -(-tiles // 3), tiles - 1]
    kb = k * k * Cin // 64
    assert kb in (1, 3, 5, 8, 9, 10, 18)

    def launch(max_ctas):
        buf32.fill_(SENT32)
        buf16.fill_(SENT16)
        o32 = buf32.view(torch.float32)[base:] if want32 else None
        o16 = buf16.view(torch.float16)[base:] if want16 else None
        d = G.conv_desc(x, w, o32, Cin, Cout, k, k, 1, k // 2, H, W, scale=scale, shift=shift, up_src=up, relu=c.relu,
                        out_coff=coff, out_strides=st, out16=o16, max_ctas=max_ctas)
        if c.entry == "rows":
            G.conv2d_rows(d)
        else:
            assert G.conv2d(d, "tc") == "tc"
        torch.cuda.synchronize()
        return buf32.clone(), buf16.clone()

    lib = L.load()
    tbuf = torch.zeros(lib.sb_conv_trace_bytes(len(grids)) // 8, dtype=torch.int64, device=dev)
    assert lib.sb_conv_trace(ctypes.c_void_p(tbuf.data_ptr()), len(grids)) == 0
    try:
        outs = [launch(mc) for mc in grids]
        infos = []
        for i in range(lib.sb_conv_trace_count()):
            v = (ctypes.c_int * 12)()
            assert lib.sb_conv_trace_info(i, v) == 0
            infos.append(list(v))
    finally:
        lib.sb_conv_trace(None, 0)
    assert [(v[4], v[5], v[6], v[10]) for v in infos] == [(bn, tiles, kb, mc) for mc in grids]

    # ---- which schedule each launch ran: one tile per CTA is cooperative, more is ping-pong where the width allows
    tr = tbuf.view(len(grids), TRACE_CTAS, TRACE_WORDS).cpu()
    for i, mc in enumerate(grids):
        t = tr[i, :mc]
        pp = mc < tiles and pingpong_ok(bn, up is not None)
        assert bool((t[:, W_SCHED] == int(pp)).all()), (c.id, mc, t[:, W_SCHED].tolist())
        assert bool((tr[i, mc:, 0] == 0).all()), "trace words of CTAs past the grid"
        per_cta = torch.tensor([len(range(b, tiles, mc)) for b in range(mc)])
        if pp:      # warpgroup g computes the CTA's tiles j = g, g + 2, ...
            assert torch.equal(t[:, W_TILES], (per_cta + 1) // 2) and torch.equal(t[:, W_TILES + 1], per_cta // 2)
        else:       # both warpgroups take part in every tile
            assert torch.equal(t[:, W_TILES], per_cta) and torch.equal(t[:, W_TILES + 1], per_cta)

    # ---- the reference launch wrote every logical element and nothing else
    b32, b16 = outs[0]
    written = torch.zeros(S, dtype=torch.bool, device=dev)
    written[idx] = True
    if want32:
        assert bool((b32[~written] == SENT32).all()) and bool(torch.isfinite(b32.view(torch.float32)[idx]).all())
    else:
        assert bool((b32 == SENT32).all())
    if want16:
        assert bool((b16[~written] == SENT16).all()) and bool(torch.isfinite(b16.view(torch.float16)[idx]).all())
    else:
        assert bool((b16 == SENT16).all())

    # ---- bit-identical outputs, guard bands included
    for mc, (o32, o16) in zip(grids[1:], outs[1:]):
        assert torch.equal(o32, b32), "%s: fp32 output with max_ctas=%d differs from one tile per CTA" % (c.id, mc)
        assert torch.equal(o16, b16), "%s: fp16 output with max_ctas=%d differs from one tile per CTA" % (c.id, mc)
