"""GPU: every instantiation of the tensor-core conv kernel (conv_tc.cu) at its tile tails, against float64.

Instantiations: fp16 and TF32 operands x tile widths 32 / 64 / 128 / 256 x {plain, upsample-add, residual} (the
residual at widths <= 128; its fp16 form is the TMA epilogue), and the data-gradient entry (mask, residual).  Each
runs at M tails (last m-tile of 1, 64, 65, 127, 128, 129 rows and a large odd M; 3x3 / upsample patches of 1x1,
8x16, 9x17, 7x33 pixels), Cout tails (Cout % 32 != 0) and K of one and of many K-steps.

Per element, with A = |s| conv(|x~|, |w~|) + |shift| + |res| + up(|u|) in float64 (x~, w~: the operands as the
tensor core reads them):
  fp32 output  |got - ref| <= 2^-12 A
  fp16 twin    |got - ref| <= 2^-11 |ref| + 2^-12 A
A missing, misplaced or double-counted element, row, box or MMA is off by O(A).

Every output lives in a larger buffer filled with a NaN sentinel (rows before and after, a channel slice of wider
rows, scattered pixels); every element of the logical output must be written and every other byte left alone.

Invariants (torch.equal): the grid size (max_ctas 1 and 3), the TMA residual epilogue against the register one
(sb_conv2d_tc_dgrad without a mask on the same descriptor), and the tile width (128 against 256)."""
import collections
import ctypes
import math
import zlib

import pytest
import torch
import torch.nn.functional as F

from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import ops as G

pytestmark = pytest.mark.gpu

SENT32 = 0x7FA5A5A5            # NaN bit patterns the kernels never produce
SENT16 = 0x7E5A
BM = 128                       # rows of an m-tile
TW, TH = 16, 8                 # pixels of a 3x3 / upsample patch tile
ERR32 = 2.0 ** -12
Case = collections.namedtuple("Case", "id mode epi N H W Cin Cout k bn env layout outs relu up mask")


def num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def pick_bn(cout, m_tiles, env, res):
    """conv_tc.cu pick_block_n + SB_TC_BLOCK_N + the residual cap"""
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
    if env in (128, 256) and cout >= 256:
        bn = env
    return 128 if res and bn == 256 else bn


def patch_mode(c):
    return c.k == 3 or c.up is not None


def m_tiles(c):
    if patch_mode(c):
        return c.N * -(-c.H // TH) * -(-c.W // TW)
    return -(-(c.N * c.H * c.W) // BM)


def m_cell(c):
    """does the last m-tile leave the second consumer warpgroup (rows 64..127) without a valid row?"""
    if patch_mode(c):
        return "le64" if c.H - (-(-c.H // TH) - 1) * TH <= TH // 2 else "gt64"
    M = c.N * c.H * c.W
    return "le64" if M - (m_tiles(c) - 1) * BM <= 64 else "gt64"


def cout_cell(c, bn):
    return "full" if c.Cout % bn == 0 else ("tail32" if c.Cout % 32 else "tailBN")


def inst(c, bn):
    return "%s/%s/%d" % (c.mode, c.epi, bn)


# ---------------------------------------------------------------------------------------------------- cases
FLAT = {1: (1, 1, 1), 64: (1, 8, 8), 65: (1, 5, 13), 127: (1, 1, 127), 128: (2, 8, 8), 129: (3, 1, 43),
        1157: (1, 13, 89), 1221: (3, 11, 37)}
FLAT_LE, FLAT_GT = (1, 64, 129, 1157), (65, 127, 128, 1221)
PATCH_LE, PATCH_GT = ((1, 1, 1), (1, 9, 17)), ((3, 8, 16), (3, 7, 33))
TAIL = {32: (24, 4), 64: (36, 40), 128: (100, 132, 200), 256: (260, 516)}
FULL = {32: 32, 64: 64, 128: 256, 256: 512}
CIN = {"f16": (64, 1024), "tf32": (32, 512), "dgrad": (64, 1024)}       # one K-step, 16 K-steps (1x1)


def _cases():
    out = []

    def add(mode, epi, geo, cin, cout, k, bn, j, up=None, mask=False, layout=None):
        N, H, W = geo
        res = epi == "res"
        env = 256 if bn == 256 else None
        tma = mode == "f16" and res
        if layout is None:
            layout = ("slice", "dense", "slice", "slice" if tma or res and mode != "dgrad" else "scatter")[j % 4]
            if mode == "dgrad" and res and j % 4 == 3:
                layout = "scatter0"          # stride-2 data gradient: even positions
        outs = {"f16": ("both", "both", "f16", "f32"), "tf32": ("f32", "both", "f32", "f32"),
                "dgrad": ("both", "f32", "both", "f16")}[mode][j % 4]
        if tma and cout % 8 and outs != "f32":
            outs = "f32"                     # the TMA path takes a twin only with Cout % 8 == 0 (16-byte rows)
        relu = mode != "dgrad" and j % 2 == 1
        cid = "%s-%s-bn%d-%dx%dx%d-c%d-co%d-k%d-%s-%s%s%s%s" % (
            mode, epi, bn, N, H, W, cin, cout, k, layout, outs, "-relu" if relu else "",
            "" if up is None else "-up%dx%d" % up, "-mask" if mask else "")
        out.append(Case(cid, mode, epi, N, H, W, cin, cout, k, bn, env, layout, outs, relu, up, mask))

    for mi, mode in enumerate(("f16", "tf32", "dgrad")):
        few, many = CIN[mode]
        epis = ("plain", "up", "res") if mode != "dgrad" else ("mask", "res")
        for ei, epi in enumerate(epis):
            for bi, bn in enumerate((32, 64, 128, 256)):
                if epi == "res" and bn == 256:
                    continue                 # residual layers use tiles of at most 128 columns
                i = mi + ei + bi
                t = TAIL[bn]
                mask = lambda j: epi == "mask" or (epi == "res" and j % 2 == 0)
                if epi == "up":
                    for j, geo in enumerate((PATCH_LE[i % 2], PATCH_GT[i % 2], PATCH_LE[(i + 1) % 2],
                                             PATCH_GT[(i + 1) % 2])):
                        N, H, W = geo
                        up = ((H + 1) // 2, (W + 1) // 2)
                        add(mode, epi, geo, many if j == 1 else few, (t[0], t[-1], FULL[bn], t[0])[j], 1, bn, j,
                            up=up)
                    continue
                flat = ((FLAT_LE[i % 4], t[0], few), (FLAT_GT[i % 4], t[-1], many if i % 4 < 3 else few),
                        (FLAT_LE[(i + 2) % 4], FULL[bn], many if (i + 2) % 4 < 3 else few),
                        (FLAT_GT[(i + 2) % 4], t[0], few))
                for j, (M, cout, cin) in enumerate(flat):
                    add(mode, epi, FLAT[M], cin, cout, 1, bn, j, mask=mode == "dgrad" and mask(j))
                if epi != "res":             # 3x3 patches (the residual epilogue is for 1x1 convs)
                    for j, geo in enumerate((PATCH_LE[i % 2], PATCH_GT[i % 2])):
                        add(mode, epi, geo, 2 * few if j == 1 else few, t[j % len(t)], 3, bn, j + 4 * (bi % 2),
                            mask=mode == "dgrad")
    # upsample edges: Ho / Wo = 1 (ratio 0), UH / UW = 1, Ho = 2 UH - 1 (exact ratio), Ho = 2 UH, UH = Ho
    for mode in ("f16", "tf32"):
        few = CIN[mode][0]
        for j, (N, Ho, Wo, UH, UW) in enumerate(((1, 1, 17, 1, 9), (2, 9, 1, 5, 1), (1, 1, 1, 1, 1),
                                                  (1, 9, 17, 5, 9), (2, 8, 16, 4, 8), (1, 7, 33, 7, 33),
                                                  (1, 9, 17, 1, 9))):
            bn, cout = ((64, 40), (128, 100))[j % 2]
            add(mode, "up", (N, Ho, Wo), few, cout, 1, bn, j, up=(UH, UW))
    return out


CASES = _cases()
SEEN = {}              # case id -> (instantiation, m cell, cout cell, worst err / A)


# ---------------------------------------------------------------------------------------------------- helpers
def tf32_trunc(t):
    return (t.contiguous().view(torch.int32) & ~0x1FFF).view(torch.float32)


def tf32_round(t):
    return G.round_tf32_(t.clone().contiguous())


def nchw64(t):
    return t.double().permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


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
    else:                             # every other pixel of a 2Ho x 2Wo image: 2x2 deconv (1, 1), stride-2 dgrad (0, 0)
        ld, coff = Cout, 0
        st, ext = (4 * Ho * Wo * ld, 2 * 2 * Wo * ld, 2 * ld), N * 4 * Ho * Wo * ld
        off = 0 if kind == "scatter0" else (2 * Wo + 1) * ld
    return lead * ld + ext + trail * ld, lead * ld + off, coff, st


def run_case(c, monkeypatch):
    g = torch.Generator().manual_seed(zlib.crc32(c.id.encode()))
    dev = "cuda"
    N, H, W, Cin, Cout, k = c.N, c.H, c.W, c.Cin, c.Cout, c.k
    Ho, Wo, M = H, W, N * H * W
    res = c.epi == "res"
    f16 = c.mode != "tf32"
    dgrad = c.mode == "dgrad"
    x = torch.randn(N, H, W, Cin, generator=g)
    w = torch.randn(Cout, k, k, Cin, generator=g) / math.sqrt(Cin * k * k)
    if f16:
        xk, wk = x.half(), w.half()
        xo, wo_ = xk.float(), wk.float()
    else:
        xk, wk = x, w
        xo, wo_ = tf32_trunc(x), tf32_trunc(w)
    scale = None if dgrad or c.up is not None else torch.rand(Cout, generator=g) + 0.5
    shift = None if dgrad else torch.randn(Cout, generator=g)
    rld, rcoff = (Cout, 0) if c.layout == "dense" else (Cout + 12, 4)
    resbig = torch.randn(N, Ho, Wo, rld, generator=g) if res else None
    up = torch.randn(N, c.up[0], c.up[1], Cout, generator=g) if c.up is not None else None

    S, base, coff, st = layout_of(c.layout, N, Ho, Wo, Cout)
    want32, want16 = c.outs in ("both", "f32"), c.outs in ("both", "f16")
    buf32 = torch.empty(S, dtype=torch.int32, device=dev)
    buf16 = torch.empty(S, dtype=torch.int16, device=dev)
    n_i = torch.arange(N, device=dev).view(-1, 1, 1, 1) * st[0]
    h_i = torch.arange(Ho, device=dev).view(1, -1, 1, 1) * st[1]
    w_i = torch.arange(Wo, device=dev).view(1, 1, -1, 1) * st[2]
    idx = base + coff + n_i + h_i + w_i + torch.arange(Cout, device=dev).view(1, 1, 1, -1)
    maskbuf = torch.randn(S, generator=g).half().to(dev) if c.mask else None

    xg, wg = xk.to(dev), wk.to(dev)
    sg = scale.to(dev) if scale is not None else None
    shg = shift.to(dev) if shift is not None else None
    resg = resbig.to(dev)[..., rcoff:rcoff + Cout] if res else None
    upg = up.to(dev) if up is not None else None

    def launch(env=None, max_ctas=0, entry=None):
        buf32.fill_(SENT32)
        buf16.fill_(SENT16)
        if env is None:
            monkeypatch.delenv("SB_TC_BLOCK_N", raising=False)
        else:
            monkeypatch.setenv("SB_TC_BLOCK_N", str(env))
        o32 = buf32.view(torch.float32)[base:] if want32 else None
        o16 = buf16.view(torch.float16)[base:] if want16 else None
        d = G.conv_desc(xg, wg, o32, Cin, Cout, k, k, 1, k // 2, Ho, Wo, scale=sg, shift=shg, residual=resg,
                        up_src=upg, relu=c.relu, out_coff=coff, out_strides=st, out16=o16, max_ctas=max_ctas)
        if (entry or ("dgrad" if dgrad else "tc")) == "dgrad":
            G.conv2d_dgrad(d, maskbuf[base:] if maskbuf is not None else None)
        else:
            assert G.conv2d(d, "tc") == "tc"
        torch.cuda.synchronize()
        return buf32.clone(), buf16.clone()

    tbuf = torch.zeros(L.load().sb_conv_trace_bytes(16), dtype=torch.uint8, device=dev)
    lib = L.load()
    assert lib.sb_conv_trace(ctypes.c_void_p(tbuf.data_ptr()), 16) == 0
    variant = int(f16) | (2 if dgrad else 0) | (4 if c.mask else 0)      # sb_conv_trace_info word 9
    launches = []                    # expected (BLOCK_N, max_ctas, variant) of every launch
    try:
        b32, b16 = launch(env=c.env)
        launches.append((c.bn, 0, variant))
        tiles = m_tiles(c) * -(-Cout // c.bn)
        invariants = []
        if tiles <= 400:
            for mc in (1, 3):
                invariants.append(("max_ctas=%d" % mc, launch(env=c.env, max_ctas=mc)))
                launches.append((c.bn, mc, variant))
        if res and c.mode == "f16" and not c.relu:
            invariants.append(("register epilogue", launch(env=c.env, entry="dgrad")))
            launches.append((c.bn, 0, 1 | 2))
        if not res and Cout >= 256:
            other = 128 if c.bn == 256 else 256
            invariants.append(("BLOCK_N=%d" % other, launch(env=other)))
            launches.append((other, 0, variant))
        count = lib.sb_conv_trace_count()
        infos = []
        for i in range(count):
            v = (ctypes.c_int * 12)()
            assert lib.sb_conv_trace_info(i, v) == 0
            infos.append(list(v))
    finally:
        lib.sb_conv_trace(None, 0)
        monkeypatch.delenv("SB_TC_BLOCK_N", raising=False)

    # ---- the launches hit the instantiation and the tile geometry the case claims
    assert pick_bn(Cout, m_tiles(c), c.env, res) == c.bn, "case list out of date: %s" % c.id
    assert count == len(launches), (count, launches)
    kb = k * k * Cin // (64 if f16 else 32)
    for v, (bn, mc, var) in zip(infos, launches):
        want = [Cin, Cout, k, M, bn, m_tiles(c) * -(-Cout // bn), kb, int(res), int(c.up is not None), var, mc, N]
        assert v == want, (c.id, v, want)

    # ---- guard bands: every logical element written, every other byte untouched
    flat_idx = idx.reshape(-1)
    written = torch.zeros(S, dtype=torch.bool, device=dev)
    written[flat_idx] = True
    if want32:
        assert bool((b32[~written] == SENT32).all()), "fp32 output: bytes outside the output were written"
        got32 = b32.view(torch.float32)[idx].cpu().double()
        assert bool(torch.isfinite(got32).all()), "fp32 output: elements not written"
    else:
        assert bool((b32 == SENT32).all())
    if want16:
        assert bool((b16[~written] == SENT16).all()), "fp16 twin: bytes outside the output were written"
        got16 = b16.view(torch.float16)[idx].cpu().double()
        assert bool(torch.isfinite(got16).all()), "fp16 twin: elements not written"
    else:
        assert bool((b16 == SENT16).all())

    # ---- float64 reference on the operands as the kernel sees them
    wr = wo_.permute(0, 3, 1, 2)                 # [Cout, Cin, k, k]
    conv = nhwc(F.conv2d(nchw64(xo), wr.double(), padding=k // 2))
    aconv = nhwc(F.conv2d(nchw64(xo).abs(), wr.double().abs(), padding=k // 2))
    s64 = scale.double() if scale is not None else torch.ones(Cout, dtype=torch.float64)
    sh64 = shift.double() if shift is not None else torch.zeros(Cout, dtype=torch.float64)

    def epilogue(cv):
        y = cv * s64 + sh64
        if res:
            y = y + resbig[..., rcoff:rcoff + Cout].double()
        if up is not None:
            y = y + nhwc(F.interpolate(nchw64(up), size=(Ho, Wo), mode="bilinear", align_corners=True))
        if c.mask:
            m = maskbuf.cpu()[idx.cpu()].float()
            y = torch.where(m > 0, y, torch.zeros_like(y))
        if c.relu:
            y = y.clamp_min(0)
        return y

    ref = epilogue(conv)
    A = aconv * s64.abs() + sh64.abs()
    if res:
        A = A + resbig[..., rcoff:rcoff + Cout].double().abs()
    if up is not None:
        A = A + nhwc(F.interpolate(nchw64(up).abs(), size=(Ho, Wo), mode="bilinear", align_corners=True))
    A = A.clamp_min(1e-30)
    line = "%-78s" % c.id
    worst = 0.0
    if want32:
        e = ((got32 - ref).abs() / A).max().item()
        worst = max(worst, e)
        line += " fp32 err/A %.2e" % e
        assert e <= ERR32, (c.id, "fp32", e)
        if f16:
            assert rel_err(got32, ref) < 5e-5, (c.id, rel_err(got32, ref))
        else:
            # against full-precision operands, the 1e-3 max-norm bound of the TF32 tests: a statistical bound (a
            # truncated product is up to 2^-9 smaller), so only where the output has thousands of elements
            if ref.numel() >= 4096:
                full = epilogue(nhwc(F.conv2d(nchw64(x), w.permute(0, 3, 1, 2).double(), padding=k // 2)))
                assert rel_err(got32, full) < 1e-3, (c.id, rel_err(got32, full))
            # tf32 round-to-nearest operand model, printed only: the kernel comment says the MMA truncates
            rn = epilogue(nhwc(F.conv2d(nchw64(tf32_round(x)), tf32_round(w).permute(0, 3, 1, 2).double(),
                                        padding=k // 2)))
            line += " (tf32 rn model %.2e)" % ((got32 - rn).abs() / A).max().item()
    if want16:
        bound = 2.0 ** -11 * ref.abs() + ERR32 * A
        e = ((got16 - ref).abs() / A).max().item()
        worst = max(worst, e)
        line += " twin err/A %.2e" % e
        assert bool(((got16 - ref).abs() <= bound).all()), (c.id, "twin", e)

    # ---- invariants: bit for bit, guard bands included
    for name, (i32, i16) in invariants:
        assert torch.equal(i32, b32), (c.id, name, "fp32")
        assert torch.equal(i16, b16), (c.id, name, "twin")
    line += " | " + ", ".join(n for n, _ in invariants)
    print(line)
    SEEN[c.id] = (inst(c, c.bn), m_cell(c), cout_cell(c, c.bn), worst)


def rel_err(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_conv_tc_sweep(case, monkeypatch, capsys):
    with capsys.disabled():
        run_case(case, monkeypatch)


def required_cells():
    insts = ["%s/%s/%d" % (m, e, bn) for m in ("f16", "tf32") for e in ("plain", "up", "res")
             for bn in (32, 64, 128, 256) if not (e == "res" and bn == 256)]
    insts += ["dgrad/%s/%d" % (e, bn) for e in ("mask", "res") for bn in (32, 64, 128, 256)
              if not (e == "res" and bn == 256)]
    return [(i, mc) for i in insts for mc in ("le64", "gt64")]


def test_case_list_covers_every_cell():
    """statically: each (instantiation x last m-tile <= / > 64 rows) cell has a case with Cout % 32 != 0 (so a
    partial column box or tile), and the 1x1 M tails, the patch shapes and the K extremes all occur"""
    have = collections.defaultdict(list)
    for c in CASES:
        have[(inst(c, c.bn), m_cell(c))].append(c)
    missing = [cell for cell in required_cells() if not any(c.Cout % 32 for c in have[cell])]
    assert not missing, missing
    flat_m = {c.N * c.H * c.W for c in CASES if not patch_mode(c)}
    assert {1, 64, 65, 127, 128, 129} <= flat_m and max(flat_m) > 1000
    assert {(c.H, c.W) for c in CASES if c.k == 3} >= {(1, 1), (8, 16), (9, 17), (7, 33)}
    for mode, (few, many) in CIN.items():
        assert any(c.mode == mode and c.k == 1 and c.Cin == few for c in CASES)
        assert any(c.mode == mode and c.k * c.k * c.Cin >= 16 * few for c in CASES)
    assert {c.layout for c in CASES} == {"dense", "slice", "scatter", "scatter0"}
    assert any(c.outs == "f16" and c.mode == "f16" and c.epi == "res" for c in CASES)
    assert any(c.outs == "f32" and c.mode == "f16" and c.epi == "res" for c in CASES)


def test_sweep_coverage_table(capsys):
    """at runtime: the launches traced by the sweep fill every cell (printed with the shape that filled it)"""
    if len(SEEN) < len(CASES):
        pytest.skip("the sweep did not run in full in this session")
    table = collections.defaultdict(list)
    for cid, (i, mc, cc, worst) in SEEN.items():
        table[(i, mc, cc)].append((worst, cid))
    with capsys.disabled():
        print("\ncoverage: instantiation x last m-tile x Cout tail -> launches (worst err/A, first shape)")
        for key in sorted(table):
            v = table[key]
            print("  %-18s %-5s %-7s %3d  %.2e  %s" % (key + (len(v), max(w for w, _ in v), v[0][1])))
    missing = [(i, mc) for i, mc in required_cells() if (i, mc, "tail32") not in table]
    assert not missing, missing
