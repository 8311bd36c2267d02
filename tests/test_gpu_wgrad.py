"""GPU: the weight gradient (conv_wgrad.cu: sb_conv_wgrad, sb_conv_wgrad_acc) and the FPN level gradient
(sb_fpn_grad_combine, ops.upsample_transpose) element by element against float64.

Weight gradient.  dW[co, ci, r, s] = s[co] / gs * sum_p dY[p, co] X[p + (r - 1, s - 1), ci] is a wgmma GEMM over
64-pixel K-blocks.  K is split into `splits` pixel ranges of `kb_per_split` K-blocks each (plan() in conv_wgrad.cu,
restated below for the device's SM count), and a second pass sums the fp32 partial tiles in split order.  The bias
gradient db[co] = sum_p dy32[p, co] / gs is summed in up to 256 row chunks, then over the chunks.

  Integer operands.  dY, X and dy32 hold integers in [-3, 3].  Every product and every partial sum is then an integer
  below 2^24, exact in fp32 in any order of k-steps, K-splits and bias chunks.  So dW and db must equal the float64
  sums as fp32 values.  With `scale`, the reduce pass's two fp32 multiplies (acc * s[co], then * 1/gs) are mirrored
  in fp32; with `accumulate`, so is the add to the integer-preloaded destination.  A dropped, doubled or misplaced
  pixel, tap, channel, tile, split or bias chunk changes an integer.

  Random-normal operands, per element.  The reference is float64 on the fp16-rounded operands.  Let
  A = |s[co]| / gs * sum_p |dy| |x| (+ |dst| when accumulating).  Inside one split a K-block is 4 k16 MMAs; each adds
  16 exact fp16 products to the fp32 accumulator.  The tensor core aligns the addends to the largest exponent and
  truncates, so an MMA step is charged c = 2 units of 2^-23 of the magnitudes summed so far.  The reduce pass adds
  `splits` partials (one rounding each), then multiplies by s[co] and by 1/gs and adds the destination (three more):
      |got - ref| <= c (4 kb_per_split + splits + 3) 2^-23 A
  db is a sequential fp32 sum of `rows` values per chunk, then of the chunks, then * 1/gs and + dst:
      |got - ref| <= (rows + chunks + 2) 2^-24 (sum_p |dy32| / gs + |dst|)
  A missing pixel or tap is off by O(A).

  Every dW / db destination (dw, dw_hi, db, db_hi) sits in a NaN-sentinel buffer with lead and tail regions: every
  logical element must be written and every other byte left alone, rows past `rows` and the destination not chosen
  by `split` included.  Channels of a strided dY / X / dy32 row outside the logical slice hold Inf or NaN: the result
  must stay finite and exact, so they are never read.

FPN level gradient.  dP = scale * dP_in + up^T(dT) + scatter2(scale * dP6).  up^T is the transpose of the
align_corners bilinear upsample whose taps the forward's epilogue computes in fp32: r = (n - 1) / (T - 1)
(__fdiv_rn, 0 when T = 1), s = r * o (__fmul_rn), i1 = (int)s, l1 = s - i1, weights (1 - l1) on i1 and l1 on i1 + 1,
or on i1 itself when i1 = n - 1 (the fold; there the fp32 sum (1 - l1) + l1 is the weight).  The mirror builds that
interpolation matrix M [T, n] in float64 from the fp32 taps; a CPU test pins it to F.interpolate.

  Impulse response, exact.  dT = one-hot rows (channel c holds fine row c) make every output element a single weight
  times 1: the device must reproduce M^T bit for bit at every swept size ratio.
  Random dT, per element.  Each addend passes through a product and the fine-column sum (nnz_w terms), a product and
  the fine-row sum (nnz_h terms), and the scale * dP and P6 terms:
      |got - ref| <= (nnz_h + nnz_w + 4) 2^-24 A,   A = |scale dP| + M_h^T |dT| M_w + |scale dP6|
  where nnz is the largest number of fine rows (columns) with a non-zero weight on one coarse row (column).
  out16 must equal out.half() bit for bit, and both outputs sit in sentinel guard bands.
"""
import collections
import time
import zlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from stereo_rcnn_b200 import ops as G

SENT32 = 0x7FA5A5A5            # NaN bit patterns the kernels never produce
SENT16 = 0x7E5A
H100_SMS = 132                 # H100 SXM: the SM count the CPU census assumes
GS14 = 2.0 ** 14
C_MMA = 2.0                    # units of 2^-23 charged per k16 MMA step (see the module docstring)


def device_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---------------------------------------------------------------------------------------------------- plan()
Plan = collections.namedtuple("Plan", "wchunks num_kb kb_per_split splits m_tiles n_tiles tiles")


def plan(N, H, W, Cin, Cout, k, sms):
    """conv_wgrad.cu plan(): about two CTAs per SM, every split at least 8 K-blocks long"""
    wchunks = -(-W // 64)
    num_kb = N * H * wchunks if k == 3 else -(-(N * H * W) // 64)
    m_tiles, n_tiles = -(-Cout // 128), -(-Cin // 128)
    tiles = m_tiles * k * k * n_tiles
    splits = max(1, min(-(-2 * sms // tiles), num_kb // 8))
    kbs = -(-num_kb // splits)
    return Plan(wchunks, num_kb, kbs, -(-num_kb // kbs), m_tiles, n_tiles, tiles)


def bias_chunks(M):
    """conv_wgrad.cu bias_chunks() -> (chunks, rows per chunk)"""
    chunks = min(256, M)
    return chunks, -(-M // chunks)


# ---------------------------------------------------------------------------------------------------- cases
# entry "wgrad": sb_conv_wgrad (dense operands, rows = split = Cout, no accumulate); "acc": sb_conv_wgrad_acc.
# dy / x / y32: (row pitch, channel offset) of the operand inside wider rows, None = dense.
Case = collections.namedtuple("Case", "id entry N H W Cin Cout k dy x y32 scale gs acc rows split bias")


def _case(cid, entry, N, H, W, Cin, Cout, k, dy=None, x=None, y32=None, scale=False, gs=1.0, acc=False, rows=None,
          split=None, bias=True):
    rows = Cout if rows is None else rows
    split = rows if split is None else split
    if entry == "wgrad":
        assert dy is None and x is None and y32 is None and not acc and rows == split == Cout
    return Case(cid, entry, N, H, W, Cin, Cout, k, dy, x, y32, scale, gs, acc, rows, split, bias)


CASES = [
    # 1x1: flat [C, M] maps
    _case("flat-m45", "wgrad", 1, 5, 9, 64, 64, 1, scale=True),
    _case("flat-m1-strided", "acc", 1, 1, 1, 128, 64, 1, dy=(72, 0), y32=(67, 0), gs=GS14),
    _case("flat-m256", "wgrad", 2, 8, 16, 256, 128, 1, gs=GS14),
    _case("flat-m65-coff", "acc", 1, 1, 65, 192, 320, 1, dy=(336, 8), x=(200, 0), scale=True),
    _case("flat-m127-rows100-acc", "acc", 1, 1, 127, 64, 128, 1, x=(80, 8), y32=(131, 2), rows=100, acc=True),
    _case("flat-split3-equal-acc", "acc", 1, 24, 64, 128, 128, 1, scale=True, gs=GS14, acc=True),
    _case("flat-split3-short", "wgrad", 1, 19, 83, 128, 128, 1),
    _case("flat-many-splits", "acc", 2, 100, 700, 64, 64, 1, y32=(65, 1), scale=True, gs=GS14),
    _case("flat-m300-split64of150-acc", "acc", 1, 3, 100, 128, 192, 1, dy=(200, 8), rows=150, split=64, acc=True),
    _case("flat-m640-nobias", "acc", 1, 10, 64, 64, 128, 1, scale=True, bias=False),
    # the fused RPN head: 24 of 64 rows, rows 0..5 -> RPN_cls_score, 6..23 -> RPN_bbox_pred_left_right
    _case("rpn-head", "acc", 1, 11, 37, 1024, 64, 1, rows=24, split=6),
    _case("rpn-head-acc", "acc", 2, 5, 8, 1024, 64, 1, rows=24, split=6, gs=GS14, acc=True),
    # FPN laterals at the small golden size (P4 from C4, P5 from C5; both sides)
    _case("lateral-1024", "wgrad", 2, 10, 16, 1024, 256, 1, gs=GS14),
    _case("lateral-2048", "wgrad", 2, 5, 8, 2048, 256, 1, gs=GS14),
    # 3x3: [C, W, H, N] maps
    _case("patch-1px", "acc", 1, 1, 1, 128, 64, 3, y32=(70, 3)),
    _case("patch-w9-n2", "wgrad", 2, 6, 9, 64, 64, 3, scale=True),
    _case("patch-w64-acc", "acc", 1, 3, 64, 64, 128, 3, x=(72, 0), gs=GS14, acc=True),
    _case("patch-w65-coff", "acc", 1, 3, 65, 128, 64, 3, dy=(80, 16), scale=True),
    _case("patch-w100-n2-rows200-acc", "acc", 2, 4, 100, 256, 256, 3, scale=True, rows=200, acc=True),
    _case("patch-h1-w130-split50-acc", "acc", 1, 1, 130, 64, 192, 3, rows=192, split=50, acc=True, gs=GS14),
    _case("patch-split3-short", "acc", 1, 25, 50, 128, 64, 3, x=(136, 8)),
    _case("patch-split3-equal", "wgrad", 1, 24, 40, 64, 128, 3),
    # RPN_Conv 256 -> 512 at the small golden size: one channel half of the [.., 1024] cat gradient (left, right)
    _case("rpn-conv-p2-left", "acc", 1, 40, 64, 256, 512, 3, dy=(1024, 0), y32=(1024, 0), gs=GS14),
    _case("rpn-conv-p3-right-acc", "acc", 1, 20, 32, 256, 512, 3, dy=(1024, 512), y32=(1024, 512), gs=GS14,
          acc=True),
    # layer-4 3x3 at 512 (frozen-BN scale, no bias), small golden size
    _case("layer4-3x3", "wgrad", 2, 5, 8, 512, 512, 3, scale=True, bias=False),
]
REAL_SHAPES = ("rpn-conv-p2-left", "rpn-conv-p3-right-acc", "lateral-1024", "lateral-2048", "layer4-3x3",
               "rpn-head", "rpn-head-acc")


def cells(c, sms):
    """the matrix cells one case reaches"""
    p = plan(c.N, c.H, c.W, c.Cin, c.Cout, c.k, sms)
    M = c.N * c.H * c.W
    out = {("k", "flat 1x1" if c.k == 1 else "patch 3x3"), ("entry", c.entry),
           ("Cout % 128", c.Cout % 128), ("Cin % 128", c.Cin % 128),
           ("m-tiles", "one" if p.m_tiles == 1 else "several"), ("n-tiles", "one" if p.n_tiles == 1 else "several")}
    if c.k == 1:
        out.add(("1x1 K tail", "M < 64" if M < 64 else "M %% 64 = %s" % (
            M % 64 if M % 64 in (0, 1, 63) else "other")))
    else:
        out.add(("3x3 K tail", "W < 64" if c.W < 64 else "W = 64" if c.W == 64 else
                 "W % 64 = 1" if c.W % 64 == 1 else "other"))
        if c.H == 1:
            out.add(("3x3 K tail", "H = 1"))
        if c.N > 1:
            out.add(("3x3 K tail", "N > 1"))
    if p.splits == 1:
        out.add(("splits", "1, num_kb < 8" if p.num_kb < 8 else "1, num_kb >= 8"))
    else:
        out.add(("splits", "several, equal" if p.num_kb % p.kb_per_split == 0 else "several, short last"))
    if c.bias:
        out.add(("bias chunks", "M < 256" if M < 256 else "M % 256 = 0" if M % 256 == 0 else "M % 256 != 0"))
    if c.dy is not None and M > 1:          # (a single pixel has no row pitch)
        out.add(("strides", "dy_ld > Cout, coff 0" if c.dy[1] == 0 else "dy_ld > Cout, coff > 0"))
    if c.x is not None and M > 1:
        out.add(("strides", "x_ld > Cin"))
    if c.y32 is not None and M > 1:
        out.add(("strides", "dy32_ld > Cout"))
    out |= {("scale", "given" if c.scale else "null"), ("grad_scale", c.gs), ("accumulate", c.acc)}
    if c.split < c.rows:
        out.add(("rows", "split < rows"))
        if c.acc:
            out.add(("rows", "split < rows, accumulate"))
    else:
        out.add(("rows", "rows = split = Cout" if c.rows == c.Cout else "rows < Cout"))
    return out


REQUIRED = ({("k", "flat 1x1"), ("k", "patch 3x3"), ("entry", "wgrad"), ("entry", "acc"),
             ("Cout % 128", 0), ("Cout % 128", 64), ("Cin % 128", 0), ("Cin % 128", 64),
             ("m-tiles", "one"), ("m-tiles", "several"), ("n-tiles", "one"), ("n-tiles", "several")}
            | {("1x1 K tail", v) for v in ("M < 64", "M % 64 = 0", "M % 64 = 1", "M % 64 = 63", "M % 64 = other")}
            | {("3x3 K tail", v) for v in ("W < 64", "W = 64", "W % 64 = 1", "other", "H = 1", "N > 1")}
            | {("splits", v) for v in ("1, num_kb < 8", "1, num_kb >= 8", "several, equal", "several, short last")}
            | {("bias chunks", v) for v in ("M < 256", "M % 256 != 0", "M % 256 = 0")}
            | {("strides", v) for v in ("dy_ld > Cout, coff 0", "dy_ld > Cout, coff > 0", "x_ld > Cin",
                                        "dy32_ld > Cout")}
            | {("scale", "null"), ("scale", "given"), ("grad_scale", 1.0), ("grad_scale", GS14),
               ("accumulate", False), ("accumulate", True)}
            | {("rows", v) for v in ("rows = split = Cout", "rows < Cout", "split < rows", "split < rows, accumulate")})


def census(sms):
    have = collections.defaultdict(list)
    for c in CASES:
        for cell in cells(c, sms):
            have[cell].append(c.id)
    return have


def _census_check(sms, show):
    have = census(sms)
    if show:
        print("\nweight-gradient case matrix at %d SMs: cell -> cases" % sms)
        for cell in sorted(have, key=str):
            print("  %-40s %2d  %s" % ("%s: %s" % cell, len(have[cell]), ", ".join(have[cell][:3])))
    missing = sorted(REQUIRED - set(have), key=str)
    assert not missing, missing
    assert len({c.id for c in CASES}) == len(CASES)
    assert set(REAL_SHAPES) <= {c.id for c in CASES}


def test_wgrad_census_at_h100_sm_count():
    """statically, at the H100 SXM's 132 SMs: the case matrix reaches every cell"""
    _census_check(H100_SMS, show=False)
    # the plan arithmetic at fixed points (conv_wgrad.cu plan())
    assert plan(2, 100, 700, 64, 64, 1, H100_SMS) == Plan(11, 2188, 9, 244, 1, 1, 1)
    assert plan(1, 40, 64, 256, 512, 3, H100_SMS) == Plan(1, 40, 10, 4, 4, 2, 72)
    assert plan(2, 5, 8, 512, 512, 3, H100_SMS) == Plan(1, 10, 10, 1, 4, 4, 144)


@pytest.mark.gpu
def test_wgrad_census_on_device(capsys):
    """at this device's SM count (the split geometry depends on it): every cell reached, the matrix printed"""
    with capsys.disabled():
        _census_check(device_sms(), show=True)


# ---------------------------------------------------------------------------------------------------- helpers
def guarded(n, lead, tail, dev="cuda"):
    """-> (int32 sentinel buffer, fp32 view of its n logical elements)"""
    buf = torch.full((lead + n + tail,), SENT32, dtype=torch.int32, device=dev)
    return buf, buf[lead:lead + n].view(torch.float32)


def check_guard(buf, lead, n, what):
    assert bool((buf[:lead] == SENT32).all()) and bool((buf[lead + n:] == SENT32).all()), \
        "%s: bytes outside the destination were written" % what
    assert bool(torch.isfinite(buf[lead:lead + n].view(torch.float32)).all()), "%s: elements not written" % what


def embed(t, spec, dtype, poison):
    """t [N,H,W,C] -> a [N,H,W,C] CUDA view of rows `ld` wide at channel offset `coff` (spec = (ld, coff), None =
    dense); the other channels of every row hold `poison`"""
    if spec is None:
        return t.to(dtype).cuda()
    ld, coff = spec
    N, H, W, C = t.shape
    wide = torch.full((N, H, W, ld), poison, dtype=dtype)
    wide[..., coff:coff + C] = t.to(dtype)
    return wide.cuda()[..., coff:coff + C]


def ref_wgrad(dy, x, k):
    """float64 sum_p dy[p, co] x[p + tap, ci] -> [Cout, Cin, k, k] (pad k // 2), dy / x NHWC float64"""
    Cout, Cin = dy.shape[3], x.shape[3]
    d = dy.reshape(-1, Cout).t()
    if k == 1:
        return (d @ x.reshape(-1, Cin)).view(Cout, Cin, 1, 1)
    N, H, W = dy.shape[:3]
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    out = torch.empty(Cout, Cin, 3, 3, dtype=torch.float64, device=dy.device)
    for r in range(3):
        for s in range(3):
            out[:, :, r, s] = d @ xp[:, r:r + H, s:s + W].reshape(-1, Cin)
    return out


def call_wgrad(c, dy16, x16, dy32, scale, dw, db, dw_hi, db_hi, flag):
    if c.entry == "wgrad":
        G.conv_wgrad(dy16, x16, c.k, dw.view(c.Cout, c.Cin, c.k, c.k), scale=scale, grad_scale=c.gs, dy32=dy32,
                     db=db, nonfinite=flag)
    else:
        G.conv_wgrad_acc(dy16, x16, c.k, dw, db=db, dy32=dy32, scale=scale, grad_scale=c.gs, accumulate=c.acc,
                         rows=c.rows, split=c.split, dw_hi=dw_hi, db_hi=db_hi, nonfinite=flag)


def run_wgrad(c, kind):
    """one case with integer ("int") or random-normal ("randn") operands -> (worst err / bound, plan)"""
    g = torch.Generator().manual_seed(zlib.crc32((c.id + kind).encode()))
    N, H, W, Cin, Cout, k = c.N, c.H, c.W, c.Cin, c.Cout, c.k
    if kind == "int":
        dy = torch.randint(-3, 4, (N, H, W, Cout), generator=g).float()
        x = torch.randint(-3, 4, (N, H, W, Cin), generator=g).float()
    else:
        dy = torch.randn(N, H, W, Cout, generator=g)
        x = torch.randn(N, H, W, Cin, generator=g)
    scale = torch.rand(Cout, generator=g) + 0.5 if c.scale else None
    dy16 = embed(dy, c.dy, torch.float16, float("inf"))
    x16 = embed(x, c.x, torch.float16, float("nan"))
    dy32 = embed(dy, c.y32, torch.float32, float("-inf")) if c.bias else None
    kk = Cin * k * k
    rows_lo, rows_hi = c.split, c.rows - c.split
    # destinations: (name, rows, elements per row); lead / tail of two rows and a few elements
    dests = [("dw", rows_lo, kk)] + ([("dw_hi", rows_hi, kk)] if rows_hi else [])
    if c.bias:
        dests += [("db", rows_lo, 1)] + ([("db_hi", rows_hi, 1)] if rows_hi else [])
    bufs, views, pre = {}, {}, {}           # name -> (sentinel buffer, lead, elements), fp32 view, preloaded values
    for name, nr, per in dests:
        lead, tail = 2 * per + 5, 2 * per + 7
        buf, views[name] = guarded(nr * per, lead, tail)
        bufs[name] = (buf, lead, nr * per)
        if c.acc:
            p = (torch.randint(-50, 51, (nr * per,), generator=g).float() if kind == "int"
                 else torch.randn(nr * per, generator=g))
            views[name].copy_(p)
            pre[name] = p.cuda()
    flag = torch.zeros(1, dtype=torch.int32, device="cuda")
    sg = scale.cuda() if scale is not None else None
    call_wgrad(c, dy16, x16, dy32, sg, views["dw"], views.get("db"), views.get("dw_hi"), views.get("db_hi"), flag)
    torch.cuda.synchronize()
    for name, (buf, lead, n) in bufs.items():
        check_guard(buf, lead, n, "%s %s" % (c.id, name))
    assert int(flag.item()) == 0, "nonfinite flag set on a finite result"

    # float64 references on the operands as the kernel reads them
    dyd, xd = dy.half().double().cuda(), x.half().double().cuda()
    sw = ref_wgrad(dyd, xd, k).reshape(Cout, kk)[:c.rows]          # rows past `rows` are dropped
    sb = dy.double().cuda().sum((0, 1, 2))[:c.rows]
    inv = 1.0 / c.gs
    s64 = scale.double().cuda()[:c.rows].view(-1, 1) if scale is not None else None
    p = plan(N, H, W, Cin, Cout, k, device_sms())
    worst = 0.0
    for base, ref, is_w in (("dw", sw, True), ("db", sb, False)):
        if not is_w and not c.bias:
            continue
        got = torch.cat([views[base].view(rows_lo, -1)] +
                        ([views[base + "_hi"].view(rows_hi, -1)] if rows_hi else [])).double()
        dst = None
        if c.acc:
            dst = torch.cat([pre[base].view(rows_lo, -1)] + ([pre[base + "_hi"].view(rows_hi, -1)] if rows_hi else []))
        ref = ref.view(c.rows, -1)
        if kind == "int":
            # exact: fp32 of the integer sums, then the reduce pass's fp32 operations in its order
            v = ref.float()
            if is_w and s64 is not None:
                v = v * scale.cuda()[:c.rows].view(-1, 1)
            v = v * inv                                              # a power of two: exact
            if dst is not None:
                v = dst + v
            bad = (got != v.double())
            assert not bool(bad.any()), "%s %s: %d of %d elements differ, first at %s: got %r want %r" % (
                c.id, base, int(bad.sum()), bad.numel(), bad.nonzero()[0].tolist(),
                float(got[bad][0]), float(v.double()[bad][0]))
        else:
            if is_w:
                a = ref_wgrad(dyd.abs(), xd.abs(), k).reshape(Cout, kk)[:c.rows]
                want, A = ref * inv, a * inv
                if s64 is not None:
                    want, A = want * s64, A * s64
                bound = C_MMA * (4 * p.kb_per_split + p.splits + 3) * 2.0 ** -23
            else:
                chunks, per = bias_chunks(N * H * W)
                want, A = ref.view(-1, 1) * inv, dy.double().abs().cuda().sum((0, 1, 2))[:c.rows].view(-1, 1) * inv
                bound = (per + chunks + 2) * 2.0 ** -24
            if dst is not None:
                want, A = want + dst.double(), A + dst.double().abs()
            err = (got - want).abs()
            ratio = float((err / (bound * A).clamp_min(1e-300)).max())
            worst = max(worst, ratio)
            assert ratio <= 1.0, "%s %s: err / bound %.3g at %s" % (c.id, base, ratio,
                                                                   (err - bound * A).argmax().item())
    if kind == "randn" and not c.acc:
        # repeatability: a second call into the same destinations is bit-identical
        first = {n: b.clone() for n, (b, _, _) in bufs.items()}
        call_wgrad(c, dy16, x16, dy32, sg, views["dw"], views.get("db"), views.get("dw_hi"), views.get("db_hi"),
                   flag)
        torch.cuda.synchronize()
        for n, (b, _, _) in bufs.items():
            assert torch.equal(b, first[n]), "%s %s: a second call differs" % (c.id, n)
    return worst, p


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["int", "randn"])
@pytest.mark.parametrize("case", CASES, ids=[c.id for c in CASES])
def test_wgrad_case(case, kind, capsys):
    t0 = time.time()
    worst, p = run_wgrad(case, kind)
    with capsys.disabled():
        print("\n%-30s %-5s %4d K-blocks, %3d per split, %3d splits  %s  %.2f s" % (
            case.id, kind, p.num_kb, p.kb_per_split, p.splits,
            "exact" if kind == "int" else "worst err/bound %.2e" % worst, time.time() - t0), end="")


# ---------------------------------------------------------------------------------------------------- nonfinite flag
@pytest.mark.gpu
@pytest.mark.parametrize("entry", ["wgrad", "acc"])
def test_wgrad_nonfinite_flag(entry):
    """the flag stays 0 on finite results, becomes 1 on an Inf in one dY pixel, on an Inf in dy32 alone (the bias
    path) and on a finite dW that overflows after the scale, and a flag already at 1 is never cleared"""
    c = _case("flag", entry, 1, 7, 70, 64, 128, 3, scale=True)
    g = torch.Generator().manual_seed(7)
    dy = torch.randint(-3, 4, (c.N, c.H, c.W, c.Cout), generator=g).float()
    x = torch.randint(1, 4, (c.N, c.H, c.W, c.Cin), generator=g).float()
    scale = torch.rand(c.Cout, generator=g) + 0.5

    def run(dy16, dy32, s, flag0=0):
        dw = torch.empty(c.Cout * c.Cin * 9, device="cuda")
        db = torch.empty(c.Cout, device="cuda")
        flag = torch.full((1,), flag0, dtype=torch.int32, device="cuda")
        call_wgrad(c, dy16.cuda(), x.half().cuda(), dy32.cuda(), s.cuda(), dw, db, None, None, flag)
        torch.cuda.synchronize()
        return int(flag.item()), dw.view(c.Cout, -1), db

    f0, dw0, db0 = run(dy.half(), dy, scale)
    assert f0 == 0
    d16 = dy.half().clone()
    d16[0, 3, 5, 7] = float("inf")
    assert run(d16, dy, scale)[0] == 1, "Inf in one dY pixel"
    d32 = dy.clone()
    d32[0, 2, 2, 9] = float("inf")
    f, dw, db = run(dy.half(), d32, scale)
    assert f == 1, "Inf in dy32 alone"
    assert torch.equal(dw, dw0) and bool(torch.isinf(db[9])), "the bias path alone carries the Inf"
    row = int((dw0.abs().sum(1) > 0).nonzero()[0])
    s = scale.clone()
    s[row] = 3e38
    f, dw, _ = run(dy.half(), dy, s)
    assert f == 1 and not bool(torch.isfinite(dw[row]).all()), "finite dW overflowing after the scale"
    assert torch.equal(dw[row + 1:], dw0[row + 1:])
    assert run(dy.half(), dy, scale, flag0=1)[0] == 1, "a flag already at 1 was cleared"


# ---------------------------------------------------------------------------------------------------- FPN mirror
def up_taps(n, T):
    """the forward epilogue's fp32 taps of fine rows 0..T-1 on a coarse axis of n rows: (i1, l1, b) per row"""
    r = np.float32(n - 1) / np.float32(T - 1) if T > 1 else np.float32(0.0)
    taps = []
    for o in range(T):
        s = np.float32(r * np.float32(o))
        i1 = int(s)
        assert 0 <= i1 <= n - 1
        taps.append((i1, np.float32(s - np.float32(i1)), i1 < n - 1))
    return taps


def up_matrix(n, T):
    """float64 [T, n] interpolation matrix of the fp32 taps (each entry an fp32 value)"""
    M = np.zeros((T, n))
    for o, (i1, l1, b) in enumerate(up_taps(n, T)):
        w0 = np.float32(1.0) - l1
        if b:
            M[o, i1], M[o, i1 + 1] = w0, l1
        else:
            M[o, i1] = np.float32(w0 + l1)        # the fold: both taps on the last row
    return M


def folds(n, T):
    """does some fine row fold onto the last coarse row with a non-zero l1 (where the b flag changes a weight)?"""
    return any(not b and l1 > 0 for _, l1, b in up_taps(n, T))


# coarse 1..64 against fine 2n-1, 2n, 2n+1, plus fine = 1 (ratio 0), fine = coarse, fine < coarse and ratios where
# fp32 rounding makes the last fine row fold with l1 > 0
SWEEP = sorted({(n, T) for n in range(1, 65) for T in (2 * n - 1, 2 * n, 2 * n + 1)} |
               {(1, 1), (1, 9), (7, 1), (64, 1), (9, 9), (64, 64), (9, 5), (64, 33), (40, 7), (64, 2),
                (4, 22), (4, 43), (6, 40), (7, 46), (6, 79)})
LEVELS = {"small": ((40, 64), (20, 32), (10, 16), (5, 8)), "bench": ((150, 497), (75, 249), (38, 125), (19, 63))}


def test_up_matrix_vs_interpolate():
    """CPU: the mirror's matrix applied to random rows agrees with F.interpolate(align_corners=True) at every swept
    size pair and every level pair of the engine, within what the fp32 taps allow, and the sweep reaches every edge.

    The fp32 coordinate s = fl(fl(r) o) is off the exact o (n - 1) / (T - 1) by at most 2^-23 (n - 1) (two roundings
    of 2^-24 relative, s <= n - 1), which moves an interpolated value by that times the largest step between
    neighbouring source rows, D; the fp32 weight 1 - l1 adds 2^-24 of the largest |src|.  The worst relative error
    this allows is printed (1e-6 and below for coarse sizes up to about 8)."""
    g = torch.Generator().manual_seed(9)
    pairs = set(SWEEP)
    for lv in LEVELS.values():
        for (fh, fw), (ch, cw) in zip(lv[:-1], lv[1:]):
            pairs |= {(ch, fh), (cw, fw)}
    worst = 0.0
    for n, T in sorted(pairs):
        src = torch.randn(1, 3, n, generator=g, dtype=torch.float64)
        ref = F.interpolate(src, size=T, mode="linear", align_corners=True)[0]
        got = (torch.from_numpy(up_matrix(n, T)) @ src[0].t()).t()
        D = float(src.diff(dim=2).abs().max()) if n > 1 else 0.0
        bound = 2.0 ** -23 * (n - 1) * D + 2.0 ** -24 * float(src.abs().max())
        err = float((got - ref).abs().max())
        assert err <= bound, (n, T, err, bound)
        worst = max(worst, err / float(ref.abs().max()))
        if n <= 8:
            assert err <= 1e-6 * float(ref.abs().max()), (n, T, err)
    print("mirror vs F.interpolate: %d size pairs, worst relative error %.2e" % (len(pairs), worst))
    assert {(1, 1), (1, 9)} <= set(SWEEP)                          # coarse = 1
    assert any(T == 1 and n > 1 for n, T in SWEEP)                 # fine = 1: ratio 0
    assert any(T == n > 1 for n, T in SWEEP)                       # fine = coarse
    assert any(T < n for n, T in SWEEP)                            # fine < coarse
    assert any(folds(n, T) for n, T in SWEEP)                      # the b flag changes a weight
    assert {n for n, _ in SWEEP} >= set(range(1, 65))


# ---------------------------------------------------------------------------------------------------- FPN on device
@pytest.mark.gpu
@pytest.mark.parametrize("axis", ["h", "w"])
def test_upsample_transpose_impulse_exact(axis):
    """dT with one fine row per channel (a one-hot): every output element is one weight, so the device must give the
    mirror's M^T bit for bit -- every tap, the ratio-0, fold and fine < coarse edges included"""
    for n, T in SWEEP:
        eye = torch.eye(T, device="cuda")
        if axis == "h":
            got = G.upsample_transpose(eye.view(1, T, 1, T), n, 1)[0, :, 0, :]
        else:
            got = G.upsample_transpose(eye.view(1, 1, T, T), 1, n)[0, 0, :, :]
        want = torch.from_numpy(up_matrix(n, T)).t().float().cuda()       # [n, T]: coarse row x fine row
        bad = got != want
        assert not bool(bad.any()), "axis %s, coarse %d, fine %d: weight at (coarse, fine) %s is %r, want %r" % (
            axis, n, T, bad.nonzero()[0].tolist(), float(got[bad][0]), float(want[bad][0]))


def run_combine(N, H, W, TH, TW, C, dp=True, dt=True, dp6=False, outs="both", scale=1.0, seed=0):
    """one sb_fpn_grad_combine launch with outputs in sentinel guard bands against float64 -> worst err / bound"""
    g = torch.Generator().manual_seed(seed)
    H6, W6 = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    dpt = torch.randn(N, H, W, C, generator=g).cuda() if dp else None
    dtt = torch.randn(N, TH, TW, C, generator=g).cuda() if dt else None
    d6 = torch.randn(N, H6, W6, C, generator=g).cuda() if dp6 else None
    n, lead, tail = N * H * W * C, 3 * C + 5, 4 * C + 7
    b32, o32 = guarded(n, lead, tail)
    b16 = torch.full((lead + n + tail,), SENT16, dtype=torch.int16, device="cuda")
    o16 = b16[lead:lead + n].view(torch.float16)
    want32, want16 = outs in ("both", "f32"), outs in ("both", "f16")
    G.fpn_grad_combine(dpt, dt=dtt, dp6=d6, scale=scale, shape=(N, H, W, C),
                       out=o32.view(N, H, W, C) if want32 else None, out16=o16.view(N, H, W, C) if want16 else None,
                       f32=want32, f16=want16)
    torch.cuda.synchronize()
    tag = "%dx%dx%d <- %dx%d C=%d dp=%d dt=%d dp6=%d %s" % (N, H, W, TH, TW, C, dp, dt, dp6, outs)
    if want32:
        check_guard(b32, lead, n, tag + " fp32")
        got = o32.view(N, H, W, C)
    else:
        assert bool((b32 == SENT32).all())
        got = G.fpn_grad_combine(dpt, dt=dtt, dp6=d6, scale=scale, shape=(N, H, W, C), f16=False)[0]
    if want16:
        assert bool((b16[:lead] == SENT16).all()) and bool((b16[lead + n:] == SENT16).all()), tag + ": fp16 guard"
        assert torch.equal(o16.view(N, H, W, C), got.half()), tag + ": out16 is not out.half()"
    else:
        assert bool((b16 == SENT16).all())
    ref = torch.zeros(N, H, W, C, dtype=torch.float64, device="cuda")
    A = torch.zeros_like(ref)
    nnz = 0
    if dp:
        ref += scale * dpt.double()
        A += abs(scale) * dpt.double().abs()
    if dt:
        Mh, Mw = up_matrix(H, TH), up_matrix(W, TW)
        nnz = int((Mh != 0).sum(0).max()) + int((Mw != 0).sum(0).max())
        Mh, Mw = torch.from_numpy(Mh).cuda(), torch.from_numpy(Mw).cuda()
        ref += torch.einsum("oy,nopc,px->nyxc", Mh, dtt.double(), Mw)
        A += torch.einsum("oy,nopc,px->nyxc", Mh, dtt.double().abs(), Mw)
    if dp6:
        ref[:, ::2, ::2] += scale * d6.double()
        A[:, ::2, ::2] += abs(scale) * d6.double().abs()
    bound = (nnz + 4) * 2.0 ** -24 * A
    err = (got.double() - ref).abs()
    assert bool((err <= bound).all()), "%s: err / bound %.3g" % (tag, float((err / bound.clamp_min(1e-300)).max()))
    return float((err / bound.clamp_min(1e-300)).max())


@pytest.mark.gpu
@pytest.mark.parametrize("axis", ["h", "w"])
def test_upsample_transpose_sweep_random(axis, capsys):
    """random dT at every swept size pair on one axis (the other axis 3 <- 6), two images, three channels"""
    worst = 0.0
    for i, (n, T) in enumerate(SWEEP):
        geo = (n, 3, T, 6) if axis == "h" else (3, n, 6, T)
        worst = max(worst, run_combine(2, geo[0], geo[1], geo[2], geo[3], 3, dp=False, outs="f32", seed=i))
    with capsys.disabled():
        print("\nupsample^T sweep along %s: %d size pairs, worst err/bound %.3f" % (axis, len(SWEEP), worst), end="")


@pytest.mark.gpu
@pytest.mark.parametrize("size", ["small", "bench"])
def test_fpn_grad_combine_engine_levels(size, capsys):
    """the engine's level pairs (P3 <- P2 ... P5 <- P4) at the small golden size and 600x1987: dP + up^T(dT), P6
    on the P5 level, 256 channels, scale = 2^14"""
    lv = LEVELS[size]
    worst = 0.0
    for i, ((fh, fw), (ch, cw)) in enumerate(zip(lv[:-1], lv[1:])):
        worst = max(worst, run_combine(2, ch, cw, fh, fw, 256, dp6=i == 2, scale=GS14, seed=20 + i))
    with capsys.disabled():
        print("\nfpn_grad_combine %s levels: worst err/bound %.3f" % (size, worst), end="")


@pytest.mark.gpu
@pytest.mark.parametrize("C", [1, 3, 256, 257, 512])
def test_fpn_grad_combine_channels(C):
    """channel counts below, at and past the 256-thread block (the c += blockDim loop)"""
    run_combine(2, 5, 7, 9, 13, C, dp6=True, scale=3.0, seed=C)


@pytest.mark.gpu
@pytest.mark.parametrize("hw", [(5, 7), (6, 8), (5, 8), (6, 7), (1, 1), (2, 1)])
def test_fpn_grad_combine_p6_scatter(hw):
    """scatter2 of dP6 at odd and even H and W, alone and with dP"""
    H, W = hw
    run_combine(1, H, W, 0, 0, 64, dt=False, dp=False, dp6=True, scale=8.0, seed=H * 10 + W)
    run_combine(2, H, W, 0, 0, 64, dt=False, dp6=True, scale=8.0, seed=H * 10 + W + 1)


OPERANDS = [dict(dp=True, dt=False, dp6=False), dict(dp=False, dt=True, dp6=False), dict(dp=False, dt=False, dp6=True),
            dict(dp=False, dt=True, dp6=True), dict(dp=True, dt=True, dp6=True)]


@pytest.mark.gpu
@pytest.mark.parametrize("outs", ["f32", "f16", "both"])
@pytest.mark.parametrize("ops_i", range(len(OPERANDS)), ids=["dp", "dt", "dp6", "dt+dp6", "all"])
def test_fpn_grad_combine_operands(ops_i, outs):
    """each of dP, dT and dP6 alone, dT and dP6 without dP, all three; fp32 only, fp16 only and both outputs"""
    run_combine(2, 7, 10, 13, 19, 96, outs=outs, scale=2.0, seed=100 + ops_i, **OPERANDS[ops_i])
