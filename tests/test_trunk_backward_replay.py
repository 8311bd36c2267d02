"""CPU: a float64 reference of the trunk + FPN backward (engine.trunk_fpn_backward), written from the model, checked
against float64 autograd through oracle.model.trunk_fpn.

trunk_fpn_backward_ref restates the backward of ResNet-101 layers 1-4 and the FPN (resnet.py:66-102, stereo_rcnn.py:
155-168 of the reference): the bottleneck's stride sits on conv1 and on the downsample, every BN is frozen and folded
as y = s conv(x, w) + b, P_k = smooth(lat(c_k) + up(P_k+1)) with the align_corners bilinear upsample, and
P6 = P5[::2, ::2].  It reads the forward's saved tensors in the engine's layout (per block xin, o1, o2; c2..c5 and
t2..t4; NHWC) and takes each ReLU mask as `saved > 0`, so the same function replays the engine's fp16 operands in
test_gpu_trunk_backward_replay.py.

Every gradient it computes has a role, named after the model:
  dp2..dp5        the gradient at P_k (dP_k times gs, plus up^T of the level above's dT, plus P6's scatter at P5)
  dt2..dt4        the gradient at t_k = lat(c_k) + up(P_k+1), the input of the smooth conv
  <block>.dy      the gradient at the block's pre-ReLU output (conv3 + shortcut)
  <block>.d2      ... at conv2's pre-ReLU output (conv3's masked input gradient)
  <block>.d1      ... at conv1's pre-ReLU output
  <block>.ds      the downsample's input gradient at the block's (strided) input pixels
  <block>.dx      the first block's input gradient through conv1 and the downsample, scattered to the full-size
                  input (zero at the pixels a stride-2 block skips), before the lateral's part and the mask
With `given`, an incoming gradient is read from given[role] where the model reads it in fp32 (the shortcut, the
upsample, bias gradients) and from given[role + "_16"] where a conv reads it as its fp16 operand, instead of the
reference's own value: teacher forcing, so that each layer is computed from the bits the engine fed it."""
import pytest
import torch
import torch.nn.functional as F

from oracle import model as OM
from stereo_rcnn_b200 import engine as E

pytestmark = pytest.mark.slow     # about 30 s on a CPU: ResNet-101 at 200x330 in float64, nine backward passes

LEVELS = ("p2", "p3", "p4", "p5", "p6")
# FPN level k (finest first): (k, smooth conv reading t_k, lateral conv reading c_k)
FPN = ((2, "RCNN_smooth3", "RCNN_latlayer3"), (3, "RCNN_smooth2", "RCNN_latlayer2"),
       (4, "RCNN_smooth1", "RCNN_latlayer1"))
# the lateral conv that reads c_L, the output of layer L - 1 and the input of layer L (L = 2, 3, 4)
LATERAL_OF = {2: "RCNN_latlayer3", 3: "RCNN_latlayer2", 4: "RCNN_latlayer1"}
DT_OF = {2: "dt2", 3: "dt3", 4: "dt4"}


def block(L, b):
    return "RCNN_layer%d.0.%d" % (L, b)


def last_block(L):
    return block(L, E.LAYERS[L - 1] - 1)


def bn_key(conv):
    return conv.replace("conv", "bn").replace("downsample.0", "downsample.1")


def trunk_convs():
    """every conv of layers 1-4 and the FPN, by state_dict key (without .weight)"""
    return [n[:-len(".weight")] for n, _ in E.trainable_trunk_fpn_params(0) if n.endswith(".weight")]


def weights_float64(sd):
    """{conv key: (w, s)} in float64 from a state_dict: w the weight the input gradient is taken through (s w, the
    frozen BN's scale folded in; the plain weight for the FPN convs) and s the per-output-channel factor of the
    weight gradient (None for the FPN convs)"""
    out = {}
    for k in trunk_convs():
        w = sd[k + ".weight"].double()
        if k.startswith("RCNN_layer"):
            bk = bn_key(k)
            s = sd[bk + ".weight"].double() / torch.sqrt(sd[bk + ".running_var"].double() + E.EPS)
            out[k] = (w * s.view(-1, 1, 1, 1), s)
        else:
            out[k] = (w, None)
    return out


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def ref_wgrad(dy, x, k):
    """sum over pixels of dy[p, co] x[p + tap, ci] -> [Cout, Cin, k, k] (pad k // 2), dy / x NHWC"""
    Cout, Cin = dy.shape[3], x.shape[3]
    d = dy.reshape(-1, Cout).t()
    if k == 1:
        return (d @ x.reshape(-1, Cin)).view(Cout, Cin, 1, 1)
    N, H, W = dy.shape[:3]
    xp = F.pad(x, (0, 0, 1, 1, 1, 1))
    out = torch.empty(Cout, Cin, 3, 3, dtype=dy.dtype, device=dy.device)
    for r in range(3):
        for s in range(3):
            out[:, :, r, s] = d @ xp[:, r:r + H, s:s + W].reshape(-1, Cin)
    return out


def dgrad(dy, w):
    """input gradient of the stride-1 conv with weight w [Cout, Cin, k, k] (pad k // 2): dy NHWC -> NHWC"""
    return nhwc(F.conv_transpose2d(nchw(dy), w, padding=w.shape[2] // 2))


def up_transpose(dt, H, W):
    """the adjoint of F.interpolate(size=dt's, bilinear, align_corners=True) from an H x W map, applied to dt (NHWC)"""
    src = torch.zeros(dt.shape[0], dt.shape[3], H, W, dtype=dt.dtype, device=dt.device, requires_grad=True)
    with torch.enable_grad():
        up = F.interpolate(src, size=dt.shape[1:3], mode="bilinear", align_corners=True)
        g, = torch.autograd.grad(up, src, nchw(dt))
    return nhwc(g)


def relu_mask(t):
    return (t > 0).to(torch.float64)


def trunk_fpn_backward_ref(weights, saved, d_feats, fixed_blocks, gs, given=None):
    """float64 backward of layers 1-4 and the FPN for the gradients d_feats["p2".."p6"] (NHWC) of the P levels.
    weights: {conv key: (w, s)} (see weights_float64); saved: the forward's tensors in the engine's layout.  The
    input gradients are multiplied by gs and every parameter gradient is divided by it, as the engine does.
    Returns (grads, roles): {state_dict name: float64 gradient} of exactly trainable_trunk_fpn_params(fixed_blocks)
    and {role: float64 gradient} of every intermediate gradient computed (see the module docstring)."""
    given = given or {}
    dev = d_feats["p2"].device
    roles, grads = {}, {}

    def f64(t):
        return t.to(dev, torch.float64)

    def g32(role):
        return f64(given[role]) if role in given else roles[role]

    def g16(role):
        return f64(given[role + "_16"]) if role + "_16" in given else roles[role]

    def wgrad(key, dy16, x, dy32=None):
        w, s = weights[key]
        dw = ref_wgrad(dy16, f64(x), w.shape[2]) / gs
        grads[key + ".weight"] = dw * s.view(-1, 1, 1, 1) if s is not None else dw
        if dy32 is not None:
            grads[key + ".bias"] = dy32.sum((0, 1, 2)) / gs

    dp = {k: f64(d_feats[k]) * gs for k in LEVELS}
    # ---- FPN, finest level first: P_k = smooth(t_k), t_k = lat(c_k) + up(P_k+1)
    roles["dp2"] = dp["p2"]
    for lvl, smooth, lat in FPN:
        pk, tk = "dp%d" % lvl, "dt%d" % lvl
        wgrad(smooth, g16(pk), saved["t%d" % lvl], g32(pk))
        roles[tk] = dgrad(g16(pk), weights[smooth][0])
        wgrad(lat, g16(tk), saved["c%d" % lvl], g32(tk))
        up = dp["p%d" % (lvl + 1)]
        roles["dp%d" % (lvl + 1)] = up + up_transpose(g32(tk), up.shape[1], up.shape[2])
    d5 = roles["dp5"].clone()
    d5[:, ::2, ::2] += dp["p6"]                         # P6 = P5[::2, ::2]
    roles["dp5"] = d5
    wgrad("RCNN_toplayer", g16("dp5"), saved["c5"], g32("dp5"))
    # c5 = relu(layer 4's last block): the toplayer's input gradient through c5's mask
    roles[last_block(4) + ".dy"] = dgrad(g16("dp5"), weights["RCNN_toplayer"][0]) * relu_mask(saved["c5"])
    # ---- trunk, top layer first
    for L in range(4, fixed_blocks, -1):
        for b in range(E.LAYERS[L - 1] - 1, -1, -1):
            p = block(L, b)
            r = saved[p]
            dy = g16(p + ".dy")
            wgrad(p + ".conv3", dy, r["o2"])
            roles[p + ".d2"] = dgrad(dy, weights[p + ".conv3"][0]) * relu_mask(r["o2"])
            wgrad(p + ".conv2", g16(p + ".d2"), r["o1"])
            roles[p + ".d1"] = dgrad(g16(p + ".d2"), weights[p + ".conv2"][0]) * relu_mask(r["o1"])
            wgrad(p + ".conv1", g16(p + ".d1"), r["xin"])
            if b > 0:
                # identity shortcut: the block's input is the previous block's ReLU'd output
                roles[block(L, b - 1) + ".dy"] = ((dgrad(g16(p + ".d1"), weights[p + ".conv1"][0]) + g32(p + ".dy"))
                                                  * relu_mask(r["xin"]))
                continue
            wgrad(p + ".downsample.0", dy, r["xin"])
            if L - 1 <= fixed_blocks:        # layer L - 1 is frozen (layer 0 always): no gradient into its output
                continue
            stride = E.STRIDES[L - 1]
            roles[p + ".ds"] = dgrad(dy, weights[p + ".downsample.0"][0])
            x = saved["c%d" % L]
            dx = torch.zeros(x.shape, dtype=torch.float64, device=dev)
            dx[:, ::stride, ::stride] = dgrad(g16(p + ".d1"), weights[p + ".conv1"][0]) + g32(p + ".ds")
            roles[p + ".dx"] = dx
            lat = dgrad(g16(DT_OF[L]), weights[LATERAL_OF[L]][0])
            roles[last_block(L - 1) + ".dy"] = (lat + g32(p + ".dx")) * relu_mask(x)
    return grads, roles


# ---------------------------------------------------------------------------------------------------- CPU checks
def forward_saved(im, sd):
    """float64 forward of oracle.model.trunk_fpn with the same operations in the same order (so the same bits),
    keeping what the backward reads in the engine's layout: per block xin (the strided input), o1, o2 (ReLU'd);
    c2..c5; t2..t4 (the smooth convs' inputs).  Returns (feats NCHW, saved NHWC)."""
    saved = {}
    x = OM.layer0(im, sd)
    feats = {}
    for L in range(1, 5):
        for b in range(E.LAYERS[L - 1]):
            p = block(L, b)
            stride = E.STRIDES[L - 1] if b == 0 else 1
            o1 = F.relu(OM._bn(OM._conv(x, sd, p + ".conv1", stride=stride), sd, p + ".bn1"))
            o2 = F.relu(OM._bn(OM._conv(o1, sd, p + ".conv2", pad=1), sd, p + ".bn2"))
            out = OM._bn(OM._conv(o2, sd, p + ".conv3"), sd, p + ".bn3")
            res = x
            if b == 0:
                res = OM._bn(OM._conv(x, sd, p + ".downsample.0", stride=stride), sd, p + ".downsample.1")
            saved[p] = dict(xin=nhwc(x[:, :, ::stride, ::stride]), o1=nhwc(o1), o2=nhwc(o2))
            x = F.relu(out + res)
        feats["c%d" % (L + 1)] = x
        saved["c%d" % (L + 1)] = nhwc(x)
    p5 = OM._conv(feats["c5"], sd, "RCNN_toplayer")
    up = p5
    for lvl, smooth, lat in reversed(FPN):
        t = OM.upsample_add(up, OM._conv(feats["c%d" % lvl], sd, lat))
        saved["t%d" % lvl] = nhwc(t)
        up = feats["p%d" % lvl] = OM._conv(t, sd, smooth, pad=1)
    feats.update(p5=p5, p6=p5[:, :, ::2, ::2])
    return feats, saved


def autograd_grads(sd, im, d_feats, names):
    """float64 autograd through oracle.model.trunk_fpn -> {name: grad}"""
    sdd = dict(sd)
    for n in names:
        sdd[n] = sd[n].clone().requires_grad_(True)
    with torch.enable_grad():
        f = OM.trunk_fpn(im, sdd)
        loss = sum((f[k] * nchw(d_feats[k])).sum() for k in LEVELS)
        gr = torch.autograd.grad(loss, [sdd[n] for n in names])
    return dict(zip(names, gr))


def zero_params(level):
    """the parameters with no path from dP at `level` alone: the smooth and lateral convs of the finer levels"""
    fine = {"p2": 0, "p3": 1, "p4": 2, "p5": 3, "p6": 3}[level]
    out = []
    for lvl, smooth, lat in FPN[:fine]:
        out += [smooth + ".weight", smooth + ".bias", lat + ".weight", lat + ".bias"]
    return out


def rel_err(a, b):
    return float((a - b).norm() / max(float(b.norm()), 1e-300))


H, W = 200, 330
GS = 2.0 ** 14


def map_sizes(h, w):
    """c2..c5 sizes of an h x w input: the stem conv (7x7 / 2, pad 3), the ceil-mode 3x3 / 2 max pool, then the
    stride-2 first blocks of layers 2-4"""
    h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    h, w = -(-(h - 3) // 2) + 1, -(-(w - 3) // 2) + 1
    out = [(h, w)]
    for _ in range(3):
        h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        out.append((h, w))
    return out


@pytest.fixture(scope="module")
def pair():
    sd = {k: v.double() for k, v in OM.make_state_dict(3).items()}
    g = torch.Generator().manual_seed(31)
    im = torch.randn(2, 3, H, W, generator=g, dtype=torch.float64) * 50.0
    with torch.no_grad():
        feats, saved = forward_saved(im, sd)
    d = {k: nhwc(torch.randn(feats[k].shape, generator=g, dtype=torch.float64)) * 1e-3 for k in LEVELS}
    return sd, im, feats, saved, d


def test_pair_size_has_odd_maps_before_stride2_blocks(pair):
    sd, im, feats, saved, d = pair
    sizes = map_sizes(H, W)
    assert sizes == [tuple(feats["c%d" % k].shape[2:]) for k in range(2, 6)]
    # the input of some stride-2 block (layers 2-4 read c2, c3, c4) is odd in both dimensions
    assert any(h % 2 and w % 2 for h, w in sizes[:3]), sizes


def test_reference_vs_float64_autograd(pair):
    """the free-running reference equals autograd for every trainable parameter at fixed_blocks 0..3; autograd runs
    once with every layer trainable, since freezing a layer does not change the other parameters' gradients"""
    sd, im, feats, saved, d = pair
    names = [n for n, _ in E.trainable_trunk_fpn_params(0)]
    ref = autograd_grads(sd, im, d, names)
    weights = weights_float64(sd)
    for fb in range(4):
        got, roles = trunk_fpn_backward_ref(weights, saved, d, fb, GS)
        want = [n for n, _ in E.trainable_trunk_fpn_params(fb)]
        assert sorted(got) == sorted(want)
        errs = {n: rel_err(got[n], ref[n]) for n in want}
        worst = max(errs, key=errs.get)
        print("fixed_blocks=%d: worst relative L2 %.2e (%s)" % (fb, errs[worst], worst))
        assert errs[worst] < 1e-10, errs[worst]
        # the roles of the stride-2 scatter exist exactly for the trainable layers above a trainable one
        assert sorted(k for k in roles if k.endswith(".dx")) == sorted(block(L, 0) + ".dx" for L in range(2, 5)
                                                                       if L - 1 > fb)


@pytest.mark.parametrize("level", LEVELS)
def test_reference_single_level_zero_pattern(pair, level):
    """dP at one level only: the parameters with no path from it come out exactly 0, every other one non-zero and
    equal to autograd's"""
    sd, im, feats, saved, d = pair
    d1 = {k: d[k] if k == level else torch.zeros_like(d[k]) for k in LEVELS}
    got, _ = trunk_fpn_backward_ref(weights_float64(sd), saved, d1, 1, GS)
    zero = set(zero_params(level))
    for n, _ in E.trainable_trunk_fpn_params(1):
        if n in zero:
            assert not bool(got[n].any()), n
        else:
            assert bool((got[n] != 0).any()), n
    if level in ("p3", "p6"):
        names = [n for n, _ in E.trainable_trunk_fpn_params(1)]
        ref = autograd_grads(sd, im, d1, names)
        for n in names:
            assert (n in zero) == (not bool(ref[n].any())), n
            if n not in zero:
                assert rel_err(got[n], ref[n]) < 1e-10, n
