"""GPU: engine.trunk_fpn_backward replayed layer by layer against float64, on the engine's own fp16 operands and
ReLU masks.

Recorders wrap the engine's _dgrad and _wgrad and ops.fpn_grad_combine: each calls the original and keeps the key,
the shapes and clones of the outputs (taken on the stream, so later launches cannot overwrite them).  Every data
gradient output is then named by its role in the model (test_trunk_backward_replay.py lists them), and
trunk_fpn_backward_ref runs teacher-forced: each layer reads the engine's own recorded fp16 or fp32 gradient for the
role the model gives its input, with the weights restated from the state_dict as the engine packs them (h16(s w) for
the data gradient, s[co] sum dy16 x16 / gs for the weight gradient, the FPN biases from the fp32 twin).  A wrong
operand, mask, shortcut, scatter or scale then shows up at the first layer that reads it, not diluted by a hundred
layers of fp16 noise as in the end-to-end comparison against the fp32 oracle (test_gpu_backward.py).

Bars: fp32 data gradients relative L2 < 2e-5, and their fp16 twins the fp32 values rounded to nearest, bit for bit.
An fp16 output cannot be held to h16(ref) itself: where the fp32 value and the reference straddle a rounding
boundary the two roundings differ by a whole ulp (2^-11 to 2^-10 relative), which alone puts the relative L2 near
5e-5 (measured 4e-5 .. 6e-5), and where cancellation leaves an element small against its terms the fp32
accumulation error exceeds that element's ulp.  The output is the rounding of an fp32 value r, so
|got16 - ref| <= |h16(ref) - ref| + 2 |r - ref|: in L2 the excess over the reference's own rounding error must stay
below 2 x 2e-5, and element by element got16 must be within one fp16 ulp of h16(ref) or within the excess allowed
by the MMA bound c (K / 16 + 3) 2^-23 A of its K-term sum.  Weight and bias gradients are held element by element
to the bound of test_gpu_wgrad.py, c (4 kb_per_split + splits + 3) 2^-23 A, with plan() for this device's SM count.
A, the sum of |terms| of each element, is the same replay on absolute values.  The structure is checked too:
exactly one data gradient per conv whose input gradient the model needs (none for a frozen layer, none into a
frozen layer's output), exactly one weight gradient per trainable conv, four level combines, found_inf clear, and
with dP at one level only the parameters with no path from it exactly 0."""
import time

import pytest
import torch

from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200 import ops as G
from stereo_rcnn_b200.synth import make_state_dict
from test_gpu_backward import GRAD_SCALE, KERNEL_TOL, _small_hw
from test_gpu_rpn_backward import _pairs
from test_gpu_wgrad import C_MMA, bias_chunks, device_sms, plan
from test_trunk_backward_replay import (FPN, LATERAL_OF, LEVELS, block, bn_key, last_block, trunk_convs,
                                        trunk_fpn_backward_ref, zero_params)

pytestmark = pytest.mark.gpu

SMOOTH_DT = {smooth: "dt%d" % lvl for lvl, smooth, _ in FPN}
LATERAL_INPUT = {lat: L for L, lat in LATERAL_OF.items()}


def l2_err(a, b):
    return float((a.double() - b).norm() / max(float(b.norm()), 1e-300))


def h16(t):
    return t.half().double()


def ulp16(x):
    """one fp16 ulp at |x| (2^-24 in the subnormal range)"""
    e = torch.frexp(x.abs().clamp_min(2.0 ** -14).float())[1]        # |x| = m 2^e, m in [0.5, 1)
    return torch.pow(2.0, (e - 11).double())


# ---------------------------------------------------------------------------------------------------- the model
def trainable(L, fixed_blocks):
    return L > fixed_blocks


def expected_dgrads(fixed_blocks):
    """the convs whose input gradient the model needs: every FPN smooth conv and the top layer; the lateral reading
    c_L when layer L - 1 trains; in a trainable layer conv3 and conv2 of every block, conv1 of every block but the
    first, and conv1 and the downsample of the first when the layer below trains"""
    out = set(SMOOTH_DT) | {"RCNN_toplayer"}
    for L in range(1, 5):
        if not trainable(L, fixed_blocks):
            continue
        below = L > 1 and trainable(L - 1, fixed_blocks)
        if below:
            out.add(LATERAL_OF[L])
        for b in range(E.LAYERS[L - 1]):
            p = block(L, b)
            out |= {p + ".conv3", p + ".conv2"}
            if b > 0 or below:
                out.add(p + ".conv1")
            if b == 0 and below:
                out.add(p + ".downsample.0")
    return out


def dgrad_role(key):
    """the role of conv `key`'s input gradient (None: the first block's conv1, whose scatter the lateral reads)"""
    if key in SMOOTH_DT:
        return SMOOTH_DT[key]
    if key == "RCNN_toplayer":
        return last_block(4) + ".dy"
    if key in LATERAL_INPUT:
        return last_block(LATERAL_INPUT[key] - 1) + ".dy"
    if key.endswith(".downsample.0"):
        return key[:-len(".downsample.0")] + ".ds"
    p, conv = key.rsplit(".", 1)
    if conv == "conv3":
        return p + ".d2"
    if conv == "conv2":
        return p + ".d1"
    L, b = int(p.split(".")[0][len("RCNN_layer"):]), int(p.split(".")[2])
    return block(L, b - 1) + ".dy" if b > 0 else None


def weights_as_packed(sd, dev):
    """{conv key: (w, s)} as the engine applies them: w = h16(s w) in fp32 (the data-gradient copy; the plain fp16
    weight for the FPN convs), s the fp32 BN fold (engine.bn_fold) the weight gradient multiplies by"""
    out = {}
    for k in trunk_convs():
        w = sd[k + ".weight"].float()
        if k.startswith("RCNN_layer"):
            bk = bn_key(k)
            s = sd[bk + ".weight"].float() / torch.sqrt(sd[bk + ".running_var"].float() + E.EPS)
            out[k] = (h16(w * s.view(-1, 1, 1, 1)).to(dev), s.double().to(dev))
        else:
            out[k] = (h16(w).to(dev), None)
    return out


# ---------------------------------------------------------------------------------------------------- recording
class Recorder(object):
    """monkeypatched onto eng._dgrad, eng._wgrad and ops.fpn_grad_combine for one backward"""

    def __init__(self, eng, monkeypatch):
        self.dgrad, self.wgrad, self.combine = {}, {}, []
        dgrad0, wgrad0, combine0 = eng._dgrad, eng._wgrad, G.fpn_grad_combine
        clone = lambda t: t.clone() if t is not None else None

        def dgrad(dy16, key, **kw):
            assert key not in self.dgrad, "data gradient of %s taken twice" % key
            o32, o16 = dgrad0(dy16, key, **kw)
            self.dgrad[key] = dict(out=clone(o32), out16=clone(o16), residual=clone(kw.get("residual")))
            return o32, o16

        def wgrad(grads, key, dy16, x16, gs, dy32=None):
            assert key not in self.wgrad, "weight gradient of %s taken twice" % key
            wgrad0(grads, key, dy16, x16, gs, dy32=dy32)
            self.wgrad[key] = tuple(dy16.shape) + (x16.shape[3], eng.p[key].kh)

        def combine(*a, **kw):
            o32, o16 = combine0(*a, **kw)
            self.combine.append((clone(o32), clone(o16)))
            return o32, o16
        monkeypatch.setattr(eng, "_dgrad", dgrad)
        monkeypatch.setattr(eng, "_wgrad", wgrad)
        monkeypatch.setattr(G, "fpn_grad_combine", combine)

    def given(self):
        """{role: fp32 gradient, role + "_16": fp16 gradient} of every recorded output"""
        out = {}

        def put(role, o32, o16):
            if o32 is not None:
                out[role] = o32
            if o16 is not None:
                out[role + "_16"] = o16
        for i, (o32, o16) in enumerate(self.combine):
            put("dp%d" % (i + 2), o32, o16)
        for key, r in self.dgrad.items():
            role = dgrad_role(key)
            if role is not None:
                put(role, r["out"], r["out16"])
            if key in LATERAL_INPUT:       # the stride-2 scatter (conv1 + downsample), as the lateral reads it
                put(block(LATERAL_INPUT[key], 0) + ".dx", r["residual"], None)
        return out


def _abs(x):
    if isinstance(x, dict):
        return {k: _abs(v) for k, v in x.items()}
    if isinstance(x, tuple):
        return tuple(_abs(v) for v in x)
    return x.abs() if x is not None else None


# ---------------------------------------------------------------------------------------------------- the replay
def replay(monkeypatch, eng, sd, saved, d, fixed_blocks, label):
    """one trunk_fpn_backward under the recorders, checked layer by layer; returns the engine's gradients"""
    t0 = time.time()
    dc = {k: v.cuda() for k, v in d.items()}
    rec = Recorder(eng, monkeypatch)
    got = eng.trunk_fpn_backward(saved, dc, fixed_blocks=fixed_blocks, grad_scale=GRAD_SCALE)
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert int(eng.found_inf.item()) == 0
    names = [n for n, _ in E.trainable_trunk_fpn_params(fixed_blocks)]
    assert sorted(got) == sorted(names)
    # structure: one data gradient per conv whose input gradient is needed, one weight gradient per trainable conv,
    # the four level combines
    assert set(rec.dgrad) == expected_dgrads(fixed_blocks), sorted(set(rec.dgrad) ^ expected_dgrads(fixed_blocks))
    assert set(rec.wgrad) == {n[:-len(".weight")] for n in names if n.endswith(".weight")}
    assert len(rec.combine) == 4

    given = rec.given()
    weights = weights_as_packed(sd, "cuda")
    d64 = {k: v.double() for k, v in dc.items()}
    with torch.no_grad():
        ref, roles = trunk_fpn_backward_ref(weights, saved, d64, fixed_blocks, GRAD_SCALE, given=given)
        assert sorted(ref) == sorted(names)
        recorded = {k[:-len("_16")] if k.endswith("_16") else k for k in given}
        assert set(roles) == recorded, sorted(set(roles) ^ recorded)
        # the same replay on absolute values gives A, the sum of |terms|, of every element of every gradient
        A, A_roles = trunk_fpn_backward_ref(_abs(weights), _abs(saved), _abs(d64), fixed_blocks, GRAD_SCALE,
                                            given=_abs(given))
        err32, err16, errw, bad = {}, {}, {}, []
        conv_of = {dgrad_role(k): k for k in rec.dgrad}
        for role, want in roles.items():
            if role in given:
                e = err32[role] = l2_err(given[role], want)
                if not e < KERNEL_TOL:
                    bad.append((role, "fp32 relative L2 %.2e" % e))
                if role + "_16" in given and not torch.equal(given[role + "_16"], given[role].half()):
                    bad.append((role, "the fp16 twin is not the fp32 output rounded to nearest"))
            if role + "_16" in given:
                # an fp16 output is the rounding of an fp32 value r with |r - ref| < the fp32 bar, so
                # |got16 - ref| <= |h16(ref) - ref| + 2 |r - ref|: in L2, and element by element with the MMA bound
                # c (K / 16 + 3) 2^-23 A of a K-term data gradient where one fp16 ulp of h16(ref) does not cover it
                g16, w16 = given[role + "_16"].double(), h16(want)
                rnd = float((w16 - want).norm())
                e = err16[role + "_16"] = (float((g16 - want).norm()) - rnd) / max(float(want.norm()), 1e-300)
                w = weights[conv_of[role]][0] if role in conv_of else None
                over = 0
                if w is not None:
                    K = w.shape[0] * w.shape[2] * w.shape[3]
                    e32 = C_MMA * (K / 16 + 3) * 2.0 ** -23 * A_roles[role]
                    ok = (g16 - w16).abs() <= ulp16(torch.maximum(g16.abs(), w16.abs()))
                    ok |= (g16 - want).abs() <= (w16 - want).abs() + 2 * e32
                    over = int((~ok).sum())
                if not e < 2 * KERNEL_TOL or over:
                    bad.append((role + "_16", "L2 beyond fp16 rounding %.2e, %d elements out of bounds" % (e, over)))
        # weight and bias gradients, element by element within test_gpu_wgrad.py's bound
        sms = device_sms()
        for n in names:
            key = n.rsplit(".", 1)[0]
            N, Hh, Ww, Cout, Cin, k = rec.wgrad[key]
            if n.endswith(".weight"):
                p = plan(N, Hh, Ww, Cin, Cout, k, sms)
                bound = C_MMA * (4 * p.kb_per_split + p.splits + 3) * 2.0 ** -23
            else:
                chunks, per = bias_chunks(N * Hh * Ww)
                bound = (per + chunks + 2) * 2.0 ** -24
            err = (got[n].double() - ref[n]).abs()
            r = errw[n] = float((err / (bound * A[n]).clamp_min(1e-300)).max())
            if not r <= 1.0:
                bad.append((n, "err / bound %.3g" % r))
    show = lambda errs: ", ".join("%s %.2e" % (n, e) for e, n in sorted(((e, n) for n, e in errs.items()),
                                                                         reverse=True))
    print("%s (%.1f s)\n  fp32 data gradients, relative L2: %s\n  fp16 data gradients, relative L2 beyond the "
          "rounding of the reference: %s\n  weight and bias gradients, worst err / bound: %s" % (
              label, time.time() - t0, show(err32), show(err16), show(errw)))
    assert not bad, bad
    return got


def _engine_run(H, W, B, seed=5):
    sd = make_state_dict(3)
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    with torch.no_grad():
        feats, saved = eng.trunk_fpn(_pairs(H, W, B, seed).cuda(), save_for_backward=True)
    g = torch.Generator().manual_seed(seed + 6)
    d = {k: torch.randn(feats[k].shape, generator=g) * 1e-3 for k in LEVELS}
    return sd, eng, saved, d


@pytest.fixture(scope="module")
def small():
    H, W = _small_hw()
    return _engine_run(H, W, 1)


@pytest.mark.parametrize("fixed_blocks", [0, 1, 2, 3])
def test_replay_small(small, monkeypatch, fixed_blocks):
    sd, eng, saved, d = small
    replay(monkeypatch, eng, sd, saved, d, fixed_blocks, "160x256 B=1 fixed_blocks=%d" % fixed_blocks)


@pytest.mark.parametrize("level", LEVELS)
def test_replay_single_level(small, monkeypatch, level):
    """dP at one level only: the gradients with no path from it are exactly 0, the others not"""
    sd, eng, saved, d = small
    d1 = {k: v if k == level else torch.zeros_like(v) for k, v in d.items()}
    got = replay(monkeypatch, eng, sd, saved, d1, 1, "160x256 dP at %s only" % level)
    zero = set(zero_params(level))
    for n, g in got.items():
        assert (n in zero) == (not bool(g.any())), n


@pytest.mark.parametrize("fixed_blocks", [0, 1])
def test_replay_odd_maps(monkeypatch, fixed_blocks):
    """200x330: c2 50x82, c3 25x41, c4 13x21, c5 7x11, so the stride-2 blocks of layers 3 and 4 read odd maps"""
    sd, eng, saved, d = _engine_run(200, 330, 1, seed=7)
    assert [tuple(saved["c%d" % k].shape[1:3]) for k in range(2, 6)] == [(50, 82), (25, 41), (13, 21), (7, 11)]
    replay(monkeypatch, eng, sd, saved, d, fixed_blocks, "200x330 B=1 fixed_blocks=%d" % fixed_blocks)


def test_replay_batched(monkeypatch):
    """B = 2 pairs, N = 4 images: the batched training step"""
    H, W = _small_hw()
    sd, eng, saved, d = _engine_run(H, W, 2, seed=9)
    replay(monkeypatch, eng, sd, saved, d, 1, "160x256 B=2 fixed_blocks=1")


def test_replay_benchmark_size(monkeypatch):
    """the benchmarked 600x1987 pair, where a weight gradient sums ~150 000 pixels"""
    sd, eng, saved, d = _engine_run(600, 1987, 1, seed=3)
    replay(monkeypatch, eng, sd, saved, d, 1, "600x1987 B=1 fixed_blocks=1")
