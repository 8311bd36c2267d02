"""CPU: a float64 reference of the fp16 forward (engine.trunk_fpn, rpn, heads), written from the model, checked
against oracle.model in float64, and the per-role checker the GPU replay (test_gpu_forward_replay.py) applies to the
engine's recorded tensors.

ForwardRef restates the test-mode forward layer by layer (resnet.py:66-163,236-286, stereo_rcnn.py:91-108,155-271,
stereo_rpn.py:52-95 of the reference): the stem (7x7 / 2 conv, frozen BN, ReLU), the ceil-mode 3x3 / 2 max pool,
ResNet-101 layers 1-4 (the stride on conv1 and on the downsample), the FPN t_k = lat(c_k) + up(P_k+1) with the
align_corners bilinear upsample, the smooth convs and P6 = P5[::2, ::2], RPN_Conv on the left and the right image of
every level into the L | R concatenation, the 1x1 class and box heads, the softmax over the (c, c + 3) score pairs,
RCNN_top.0 as the 7x7 / 7 conv of the NCHW pooled tile, RCNN_top.3, the keypoint convs RCNN_kpts.0..10 and the 2x2 / 2
transposed conv.  Every conv is y = s conv(x, w) + b (+ residual) (+ upsample), then the ReLU: s, b the folded BN
(s = None, b the bias for the convs that have one).

Every tensor it computes has a role, named after the model:
  image, pooled_box, pooled_kpts   the inputs (NCHW image; NHWC pooled tiles, right image in channels 256..511)
  stem, c1                         the stem conv's output and the max pool's
  <block>.xin                      the strided input of a stride-2 first block (layers 2-4)
  <block>.o1 / .o2 / .ds / .out    conv1, conv2 (ReLU'd), the downsample, the block output; the last block of
                                   layer L writes c<L+1> instead of .out
  t2..t4, p2..p6                   the FPN: the smooth convs' inputs and the P levels
  rpn_cat.<level>                  [B,h,w,1024] ReLU(RPN_Conv) of the left images | of the right images
  rpn_head                         [B,P,32] the fused head: 0..5 class scores, 6..23 box deltas, 24..31 zero
  rpn_cls_prob, rpn_bbox_pred      [B,3P,2], [B,3P,6]
  top0, fc7, kpts0..kpts10, up     the R-CNN heads (NHWC, R rows)
With `given`, a layer reads its input from given[role + "_16"] where the engine's conv reads an fp16 operand and from
given[role] where the epilogue reads fp32 (the residual, the upsample source, the RPN head), instead of the
reference's own value: teacher forcing, so that a wrong operand shows up at the first layer that reads it.
emulate=True feeds the reference its own outputs rounded as the engine stores them (stores()), which gives
self-consistent "engine records" for testing the checker; `faults` then perturbs chosen roles before the ReLU."""
import pytest
import torch
import torch.nn.functional as F

from oracle import model as OM
from stereo_rcnn_b200 import engine as E
from test_trunk_backward_replay import FPN, block, bn_key, forward_saved, nchw, nhwc, trunk_convs

pytestmark = pytest.mark.slow     # ResNet-101 in float64 a dozen times

LEVELS = ("p2", "p3", "p4", "p5", "p6")
KPTS = tuple("RCNN_kpts.%d" % i for i in range(0, 12, 2))
C_MMA = 2.0                     # units of 2^-23 per k16 MMA step, as test_gpu_wgrad.py
EPI = 8 * 2.0 ** -24            # the epilogue's fp32 operations (fma, residual / upsample adds), times A
KERNEL_TOL = 2e-5               # relative L2 of an fp32 output
SOFTMAX_TOL = 2.0 ** -20        # absolute, on a probability


def stores(role):
    """(fp32, fp16): which copies of a role the fp16 engine keeps.  Block outputs, the downsample, the P levels, the
    RPN head and its epilogue's outputs and fc7 are fp32 (the residual stream, the upsample source, RoIAlign's and
    the tails' inputs), with an fp16 twin where a conv reads them; everything else only a conv reads, in fp16."""
    if role.endswith(".ds") or role in ("rpn_head", "rpn_cls_prob", "rpn_bbox_pred", "fc7"):
        return True, False
    if role.endswith(".out") or role in ("c2", "c3", "c4", "c5") or role in LEVELS:
        return True, True
    return False, True


def last_role(L, b):
    """the role of block (L, b)'s output"""
    return "c%d" % (L + 1) if b == E.LAYERS[L - 1] - 1 else block(L, b) + ".out"


def h16(t):
    return t.half().double()


def ulp16(x):
    """one fp16 ulp at |x| (2^-24 in the subnormal range)"""
    e = torch.frexp(x.abs().clamp_min(2.0 ** -14).float())[1]        # |x| = m 2^e, m in [0.5, 1)
    return torch.pow(2.0, (e - 11).double())


# ---------------------------------------------------------------------------------------------------- weights
def _heads_w(sd, bias, weight):
    """the RPN and R-CNN head convs {key: (w, None, b)}, w and b through `weight` and `bias` (their precision)"""
    out = {"RCNN_rpn.RPN_Conv": None, "RCNN_rpn.RPN_cls_score": None, "RCNN_rpn.RPN_bbox_pred_left_right": None,
           "RCNN_top.0": None, "RCNN_top.3": None, "RCNN_kpts.12": None}
    for k in list(out) + list(KPTS):
        out[k] = (weight(sd[k + ".weight"]), None, bias(sd[k + ".bias"]))
    return out


def weights_exact(sd):
    """{conv key: (w, s, b)} in float64: s = gamma / sqrt(var + eps), b = beta - mean s for a conv with a frozen BN"""
    d = lambda t: t.double()
    out = {}
    for k in ["RCNN_layer0.0"] + trunk_convs():
        w = d(sd[k + ".weight"])
        if k.startswith("RCNN_layer"):
            bk = "RCNN_layer0.1" if k == "RCNN_layer0.0" else bn_key(k)
            s = d(sd[bk + ".weight"]) / torch.sqrt(d(sd[bk + ".running_var"]) + E.EPS)
            out[k] = (w, s, d(sd[bk + ".bias"]) - d(sd[bk + ".running_mean"]) * s)
        else:
            out[k] = (w, None, d(sd[k + ".bias"]))
    out.update(_heads_w(sd, d, d))
    return out


def weights_as_packed(sd, dev="cpu"):
    """{conv key: (w, s, b)} as the fp16 engine applies them: w = h16(w) unscaled, s and b the fp32 BN fold of
    engine.bn_fold (float32 arithmetic on the host), the biases in fp32; all as float64 on `dev`"""
    f = lambda t: t.float()
    out = {}
    for k in ["RCNN_layer0.0"] + trunk_convs():
        w = h16(f(sd[k + ".weight"]))
        if k.startswith("RCNN_layer"):
            bk = "RCNN_layer0.1" if k == "RCNN_layer0.0" else bn_key(k)
            s = f(sd[bk + ".weight"]) / torch.sqrt(f(sd[bk + ".running_var"]) + E.EPS)
            b = f(sd[bk + ".bias"]) - f(sd[bk + ".running_mean"]) * s
            out[k] = (w, s.double(), b.double())
        else:
            out[k] = (w, None, f(sd[k + ".bias"]).double())
    out.update(_heads_w(sd, lambda t: f(t).double(), lambda t: h16(f(t))))
    return {k: tuple(v.to(dev) if v is not None else None for v in t) for k, t in out.items()}


def abs_weights(W):
    return {k: tuple(v.abs() if v is not None else None for v in t) for k, t in W.items()}


# ---------------------------------------------------------------------------------------------------- the reference
class ForwardRef(object):
    """the float64 forward (module docstring).  After run(): roles {role: float64 tensor}, K {role: the number of
    MMA terms of a conv role, 0 for an exact copy (max pool, subsample, P6), "softmax", or None for an input},
    slack {role: extra absolute bound} (the upsample's coordinate rounding), reads {conv role: {"x": role of the fp16
    operand, "res" / "up": role of the fp32 residual / upsample source}}, uses {conv key: launches}; with
    emulate=True also rec, the engine-like records."""

    def __init__(self, W, given=None, emulate=False, faults=None):
        self.W, self.faults = W, faults or {}
        self.roles, self.K, self.slack, self.reads, self.uses = {}, {}, {}, {}, {}
        self.rec = {} if emulate else None
        self.given = self.rec if emulate else (given or {})

    # ---- reads and writes
    def g16(self, role):
        t = self.given.get(role + "_16")
        return t.to(self.dev, torch.float64) if t is not None else self.roles[role]

    def g32(self, role):
        t = self.given.get(role)
        return t.to(self.dev, torch.float64) if t is not None else self.roles[role]

    def put(self, role, v, K):
        assert role not in self.roles, "role %s produced twice" % role
        self.roles[role], self.K[role] = v, K
        if self.rec is not None and K is not None:
            f32, f16 = stores(role)
            if f32:
                self.rec[role] = v.float()
            if f16:
                self.rec[role + "_16"] = v.half()
        return v

    def use(self, key):
        self.uses[key] = self.uses.get(key, 0) + 1
        return self.W[key]

    # ---- the layers
    def up(self, src, Ho, Wo, slack=False):
        """F.interpolate(src, (Ho, Wo), bilinear, align_corners=True) on NHWC; slack=True: instead, per output pixel
        the sum of |src| over the 3 x 3 source pixels around its top-left tap times 2^-22 (sy + sx + 2), a bound on
        what fp32 coordinates (sy = ho (UH - 1) / (Ho - 1), one rounding each) move the result by, a tap row or
        column crossing included"""
        N, UH, UW, C = src.shape
        sy = torch.arange(Ho, dtype=torch.float64, device=src.device) * ((UH - 1) / (Ho - 1) if Ho > 1 else 0.0)
        sx = torch.arange(Wo, dtype=torch.float64, device=src.device) * ((UW - 1) / (Wo - 1) if Wo > 1 else 0.0)
        y1, x1 = sy.floor().long().clamp(max=UH - 1), sx.floor().long().clamp(max=UW - 1)
        if slack:
            box = nhwc(F.avg_pool2d(nchw(src.abs()), 3, 1, 1, count_include_pad=True) * 9)
            return box[:, y1][:, :, x1] * (2.0 ** -22 * (sy.view(-1, 1) + sx.view(1, -1) + 2)).view(1, Ho, Wo, 1)
        y2, x2 = (y1 + 1).clamp(max=UH - 1), (x1 + 1).clamp(max=UW - 1)
        ly, lx = (sy - y1).view(1, Ho, 1, 1), (sx - x1).view(1, 1, Wo, 1)
        r1, r2 = src[:, y1], src[:, y2]
        return ((1 - ly) * ((1 - lx) * r1[:, :, x1] + lx * r1[:, :, x2]) +
                ly * ((1 - lx) * r2[:, :, x1] + lx * r2[:, :, x2]))

    def lin(self, key, x, stride=1, pad=0):
        """s conv(x, w) + b, NHWC"""
        w, s, b = self.use(key)
        y = nhwc(F.conv2d(nchw(x), w, stride=stride, padding=pad))
        return (y * s if s is not None else y) + b

    def conv(self, role, key, x_role, stride=1, pad=0, relu=True, res=None, up=None):
        """role = [ReLU](s conv(g16(x_role), w) + b [+ g32(res)] [+ up(g32(up))]), NHWC"""
        y = self.lin(key, self.g16(x_role), stride, pad)
        w = self.W[key][0]
        self.reads[role] = dict(x=x_role)
        if res is not None:
            y = y + self.g32(res)
            self.reads[role]["res"] = res
        if up is not None:
            u = self.g32(up)
            y = y + self.up(u, y.shape[1], y.shape[2])
            self.slack[role] = self.up(u, y.shape[1], y.shape[2], slack=True)
            self.reads[role]["up"] = up
        if role in self.faults:
            y = self.faults[role](y, self)
        return self.put(role, F.relu(y) if relu else y, w.shape[1] * w.shape[2] * w.shape[3])

    def trunk(self):
        im = self.g16("image")
        w, s, b = self.use("RCNN_layer0.0")
        y = nhwc(F.conv2d(im, w, stride=2, padding=3)) * s + b
        if "stem" in self.faults:
            y = self.faults["stem"](y, self)
        self.reads["stem"] = dict(x="image")
        self.put("stem", F.relu(y), 192)          # the 147 taps, zero padded to three 64-wide K-steps
        self.reads["c1"] = dict(x="stem")
        self.put("c1", nhwc(F.max_pool2d(nchw(self.g16("stem")), 3, 2, ceil_mode=True)), 0)
        x = "c1"
        for L in range(1, 5):
            for bi in range(E.LAYERS[L - 1]):
                p = block(L, bi)
                xin = x
                if bi == 0 and E.STRIDES[L - 1] == 2:
                    xin = p + ".xin"
                    self.reads[xin] = dict(x=x)
                    self.put(xin, self.g16(x)[:, ::2, ::2], 0)
                self.conv(p + ".o1", p + ".conv1", xin)
                self.conv(p + ".o2", p + ".conv2", p + ".o1", pad=1)
                res = x
                if bi == 0:
                    res = p + ".ds"
                    self.conv(res, p + ".downsample.0", xin, relu=False)
                x = last_role(L, bi)
                self.conv(x, p + ".conv3", p + ".o2", res=res)

    def fpn(self):
        self.conv("p5", "RCNN_toplayer", "c5", relu=False)
        for lvl, smooth, lat in reversed(FPN):
            self.conv("t%d" % lvl, lat, "c%d" % lvl, relu=False, up="p%d" % (lvl + 1))
            self.conv("p%d" % lvl, smooth, "t%d" % lvl, pad=1, relu=False)
        self.reads["p6"] = dict(x="p5")
        self.put("p6", self.g32("p5")[:, ::2, ::2], 0)

    def rpn(self, B):
        heads = []
        for lvl in LEVELS:
            f = self.g16(lvl)
            cat = "rpn_cat." + lvl
            # the shared RPN_Conv on the left images, then on the right ones, concatenated along the channels
            y = torch.cat([self.lin("RCNN_rpn.RPN_Conv", f[side * B:(side + 1) * B], pad=1) for side in range(2)], 3)
            if cat in self.faults:
                y = self.faults[cat](y, self)
            self.reads[cat] = dict(x=lvl)
            self.put(cat, F.relu(y), 9 * 256)
            x = self.g16(cat)
            h = [self.lin(k, x) for k in ("RCNN_rpn.RPN_cls_score", "RCNN_rpn.RPN_bbox_pred_left_right")]
            h.append(torch.zeros(h[0].shape[:3] + (8,), dtype=h[0].dtype, device=h[0].device))
            heads.append(torch.cat(h, 3).reshape(B, -1, 32))
        y = torch.cat(heads, 1)
        if "rpn_head" in self.faults:
            y = self.faults["rpn_head"](y, self)
        self.reads["rpn_head"] = dict(x="rpn_cat")
        self.put("rpn_head", y, 1024)
        head = self.g32("rpn_head")
        s = head[..., :6]
        e = torch.exp(s - torch.maximum(s[..., :3], s[..., 3:]).repeat(1, 1, 2))
        prob = e / (e[..., :3] + e[..., 3:]).repeat(1, 1, 2)       # softmax over the pairs (c, c + 3)
        for role, v, K in (("rpn_cls_prob", prob.reshape(B, -1, 2), "softmax"),
                           ("rpn_bbox_pred", head[..., 6:24].reshape(B, -1, 6), 0)):
            self.reads[role] = dict(x="rpn_head")
            self.put(role, v, K)

    def heads(self):
        R = self.g16("pooled_box").shape[0]
        # Conv2d(512, 2048, 7, stride 7) of the pooled 7x7 tile: the NHWC tile viewed NCHW
        self.conv("top0", "RCNN_top.0", "pooled_box", stride=7)
        self.conv("fc7", "RCNN_top.3", "top0")
        x = "pooled_kpts"
        for i, k in enumerate(KPTS):
            self.conv("kpts%d" % (2 * i), k, x, pad=1)
            x = "kpts%d" % (2 * i)
        w, _, b = self.use("RCNN_kpts.12")
        y = nhwc(F.conv_transpose2d(nchw(self.g16(x)), w, b, stride=2))
        if "up" in self.faults:
            y = self.faults["up"](y, self)
        self.reads["up"] = dict(x=x)
        self.put("up", F.relu(y), 256)
        assert R == y.shape[0]

    def run(self, inputs, B, rpn=True, heads=True):
        """inputs: {"image": [2B,3,H,W], "pooled_box": [R,7,7,512], "pooled_kpts": [R,14,14,256]} (float64, or
        None where `given` has the fp16 copy)"""
        self.dev = next(iter(self.W.values()))[0].device
        for k in ("image",) + (("pooled_box", "pooled_kpts") if heads else ()):
            v = inputs.get(k)
            self.put(k, v.to(self.dev, torch.float64) if v is not None else self.g16(k), None)
            if self.rec is not None:
                self.rec[k + "_16"] = self.roles[k].half()
        self.trunk()
        self.fpn()
        if rpn:
            self.rpn(B)
        if heads:
            self.heads()
        return self


def run_ref(W, inputs, B, given=None, rpn=True, heads=True, emulate=False, faults=None):
    return ForwardRef(W, given, emulate, faults).run(inputs, B, rpn, heads)


def expected_uses(rpn=True, heads=True):
    """conv launches of one forward, per key: every trunk and FPN conv once (on the whole batch of images),
    RPN_Conv on both images of each level, the two RPN heads once per level, the R-CNN head convs once"""
    out = {k: 1 for k in ["RCNN_layer0.0"] + trunk_convs()}
    if rpn:
        out.update({"RCNN_rpn.RPN_Conv": 10, "RCNN_rpn.RPN_cls_score": 5, "RCNN_rpn.RPN_bbox_pred_left_right": 5})
    if heads:
        out.update({k: 1 for k in ("RCNN_top.0", "RCNN_top.3", "RCNN_kpts.12") + KPTS})
    return out


# ---------------------------------------------------------------------------------------------------- the checker
def bound(ref, A, role):
    """e: C_MMA (K / 16 + 3) 2^-23 A for the MMA sum, EPI A for the epilogue, plus the upsample's slack"""
    K = ref.K[role]
    e = (C_MMA * (K / 16 + 3) * 2.0 ** -23 + EPI) * A.roles[role]
    return e + ref.slack[role] if role in ref.slack else e


def check(recorded, ref, A):
    """Hold every recorded role to the teacher-forced reference `ref` (a ForwardRef run on `recorded`) with A the same
    run on absolute values.  Returns ({role: reason} of the roles out of bounds, {role: worst err / bound}).
      exact roles (K == 0): every stored copy is the reference in its type, bit for bit;
      fp32 outputs: relative L2 < KERNEL_TOL and |got - ref| <= e element by element;
      fp16 twins of an fp32 output: the fp32 output rounded to nearest, bit for bit;
      fp16-only outputs: within one fp16 ulp of h16(ref), or |got - ref| <= |h16(ref) - ref| + 2 e (the rounding of
      an fp32 value within e of the reference);
      the class probabilities: within SOFTMAX_TOL."""
    bad, ratio = {}, {}

    def fail(role, why):
        bad.setdefault(role, why)
    for role, want in ref.roles.items():
        K = ref.K[role]
        if K is None:
            continue
        f32, f16 = recorded.get(role), recorded.get(role + "_16")
        if f32 is None and f16 is None:
            fail(role, "not recorded")
            continue
        if K == 0:
            for t in (f32, f16):
                if t is not None and not torch.equal(t, want.to(t.dtype)):
                    fail(role, "not bit-identical (%d elements differ)" % int((t != want.to(t.dtype)).sum()))
            continue
        if K == "softmax":
            err = float((f32.double() - want).abs().max())
            ratio[role] = err / SOFTMAX_TOL
            if not err <= SOFTMAX_TOL:
                fail(role, "max |err| %.3g" % err)
            continue
        e = bound(ref, A, role)
        if f32 is not None:
            d = (f32.double() - want).abs()
            l2 = float(d.norm() / max(float(want.norm()), 1e-300))
            r = ratio[role] = float((d / e.clamp_min(1e-300)).max())
            if not l2 < KERNEL_TOL:
                fail(role, "fp32 relative L2 %.3g" % l2)
            if not r <= 1.0:
                fail(role, "fp32 err / bound %.3g at %d elements" % (r, int((d > e).sum())))
            if f16 is not None and not torch.equal(f16, f32.half()):
                fail(role, "the fp16 twin is not the fp32 output rounded to nearest (%d elements)"
                     % int((f16 != f32.half()).sum()))
        elif f16 is not None:
            g, w16 = f16.double(), h16(want)
            ok = (g - w16).abs() <= ulp16(torch.maximum(g.abs(), w16.abs()))
            slack = (w16 - want).abs() + 2 * e
            d = (g - want).abs()
            ok |= d <= slack
            over = d - (w16 - want).abs()
            ratio[role] = float(torch.where(ok, torch.zeros_like(over), over / (2 * e).clamp_min(1e-300)).max())
            if not bool(ok.all()):
                fail(role, "fp16 output out of bounds at %d elements" % int((~ok).sum()))
    return bad, ratio


def role_class(role):
    """stem, layer k, FPN, RPN, head: the classes the replay's report groups roles into"""
    if role in ("stem", "c1"):
        return "stem"
    if role.startswith("RCNN_layer"):
        return "layer" + role[len("RCNN_layer")]
    if role in ("c2", "c3", "c4", "c5"):
        return "layer%d" % (int(role[1]) - 1)
    if role[0] in "tp" and role[1:].isdigit():
        return "FPN"
    if role.startswith("rpn"):
        return "RPN"
    return "head"


# ---------------------------------------------------------------------------------------------------- CPU checks
H, W = 200, 330


def _inputs(N, h, w, R, seed):
    g = torch.Generator().manual_seed(seed)
    im = torch.randn(N, 3, h, w, generator=g, dtype=torch.float64) * 50.0
    pb = torch.randn(R, 7, 7, 512, generator=g, dtype=torch.float64).relu()
    pk = torch.randn(R, 14, 14, 256, generator=g, dtype=torch.float64).relu()
    return dict(image=im, pooled_box=pb, pooled_kpts=pk)


@pytest.fixture(scope="module")
def sd():
    return {k: v.double() for k, v in OM.make_state_dict(3).items()}


@pytest.fixture(scope="module")
def free(sd):
    inputs = _inputs(2, H, W, 3, 31)
    with torch.no_grad():
        return inputs, run_ref(weights_exact(sd), inputs, 1)


def rel_err(a, b):
    return float((a - b).norm() / max(float(b.norm()), 1e-300))


def test_reference_vs_oracle(sd, free):
    """the free-running reference equals oracle.model in float64 (trunk_fpn, rpn_head, box_head, kpts_head) at a
    size whose stride-2 blocks of layers 3 and 4 read odd maps"""
    inputs, ref = free
    r = ref.roles
    with torch.no_grad():
        want = OM.trunk_fpn(inputs["image"], sd)
        feats, saved = forward_saved(inputs["image"], sd)
        assert [tuple(want["c%d" % k].shape[2:]) for k in range(2, 6)] == [(50, 82), (25, 41), (13, 21), (7, 11)]
        errs = {k: rel_err(r[k], nhwc(want[k])) for k in ("c1", "c2", "c3", "c4", "c5") + LEVELS}
        errs.update({k: rel_err(r[k], saved[k]) for k in ("t2", "t3", "t4")})
        for L in range(1, 5):
            for b in range(E.LAYERS[L - 1]):
                p = block(L, b)
                errs[p + ".o1"] = rel_err(r[p + ".o1"], saved[p]["o1"])
                errs[p + ".o2"] = rel_err(r[p + ".o2"], saved[p]["o2"])
        lv = [want[k] for k in LEVELS]
        prob, bbox, shapes, scores = OM.rpn_head([t[:1] for t in lv], [t[1:] for t in lv], sd)
        errs["rpn_cls_prob"] = rel_err(r["rpn_cls_prob"], prob)
        errs["rpn_bbox_pred"] = rel_err(r["rpn_bbox_pred"], bbox)
        errs["rpn_head"] = rel_err(r["rpn_head"][..., :6].reshape(1, -1, 2), scores)
        assert not bool(r["rpn_head"][..., 24:].any())
        cls, _, _, fc7 = OM.box_head(nchw(inputs["pooled_box"]), sd)
        errs["fc7"] = rel_err(r["fc7"].flatten(1), fc7)
        _, _, _, ka = OM.kpts_head(nchw(inputs["pooled_kpts"]), sd)
        got = F.conv2d(nchw(r["up"]), sd["kpts_class.weight"], sd["kpts_class.bias"]).sum(2)
        errs["up"] = rel_err(got, ka)
    worst = max(errs, key=errs.get)
    print("worst relative L2 %.2e (%s)" % (errs[worst], worst))
    assert errs[worst] < 1e-12, (worst, errs[worst])


def test_role_census(free):
    """every role is produced once (ForwardRef.put asserts it), every conv key launched once per image group"""
    inputs, ref = free
    assert ref.uses == expected_uses()
    want = {"image", "pooled_box", "pooled_kpts", "stem", "c1", "t2", "t3", "t4", "rpn_head", "rpn_cls_prob",
            "rpn_bbox_pred", "top0", "fc7", "up"} | set(LEVELS) | {"rpn_cat." + k for k in LEVELS}
    want |= {"kpts%d" % i for i in range(0, 12, 2)}
    for L in range(1, 5):
        for b in range(E.LAYERS[L - 1]):
            p = block(L, b)
            want |= {p + ".o1", p + ".o2", last_role(L, b)}
            if b == 0:
                want.add(p + ".ds")
                if E.STRIDES[L - 1] == 2:
                    want.add(p + ".xin")
    assert set(ref.roles) == want, sorted(set(ref.roles) ^ want)
    # every role but the inputs says what it reads, and what it reads is a role
    assert set(ref.reads) == want - {"image", "pooled_box", "pooled_kpts"}
    for role, rd in ref.reads.items():
        assert all(v in ref.roles or v == "rpn_cat" for v in rd.values()), (role, rd)


# ---- the checker on engine-like records with one injected fault each
FH, FW, FR = 128, 200, 4     # B = 2, c4 8 x 13: the downsample of layer 3 has 416 rows, more than two 128-row tiles


def _shift_neighbour(role):
    key = role[:-len(".ds")] + ".downsample.0"

    def f(y, ref):
        b = ref.W[key][2]
        y = y.contiguous()
        rows = y.view(-1, y.shape[3])
        rows[128:256, :-1] += b[1:] - b[:-1]     # the second 128-row tile: channel c adds shift[c + 1]
        return y
    return f


def _residual_is_input(p):
    def f(y, ref):
        x = ref.g16(p + ".xin").repeat(1, 1, 1, 2)      # the block input, tiled to the output channels
        return y - ref.g32(p + ".ds") + x
    return f


def _swap_halves(y, ref):
    return torch.cat((y[..., 512:], y[..., :512]), 3)


def _padding(y, ref):
    y = y.clone()
    y[..., 24:] = 0.25
    return y


def _top0_k_order(y, ref):
    w, _, b = ref.W["RCNN_top.0"]
    R = y.shape[0]
    x = ref.g16("pooled_box").reshape(R, -1)                 # (ph, pw, c), the engine's operand
    wk = w.reshape(w.shape[0], -1)                            # (c, ph, pw), the state_dict's order
    return (x @ wk.t() + b).view(R, 1, 1, -1)


def _swap_phases(y, ref):
    y = y.clone()
    a, b = y[:, 0::2, 0::2].clone(), y[:, 0::2, 1::2].clone()
    y[:, 0::2, 0::2], y[:, 0::2, 1::2] = b, a
    return y


def _two_ulp(y, ref):
    y = y.contiguous().clone()
    i = int(y.flatten().argmax())
    y.view(-1)[i] += 2 * ulp16(y.view(-1)[i])
    return y


def _no_upsample(y, ref):
    return y - ref.up(ref.g32("p4"), y.shape[1], y.shape[2])


FAULTS = {
    "shift_of_neighbour_channel": ("RCNN_layer3.0.0.ds", _shift_neighbour("RCNN_layer3.0.0.ds")),
    "residual_is_block_input": ("RCNN_layer2.0.0.out", _residual_is_input("RCNN_layer2.0.0")),
    "rpn_cat_halves_swapped": ("rpn_cat.p4", _swap_halves),
    "rpn_head_padding_not_zero": ("rpn_head", _padding),
    "top0_k_order_c_ph_pw": ("top0", _top0_k_order),
    "deconv_phases_swapped": ("up", _swap_phases),
    "fp16_two_ulp": ("stem", _two_ulp),
    "t3_without_upsample": ("t3", _no_upsample),
}


@pytest.fixture(scope="module")
def packed(sd):
    return weights_as_packed({k: v.float() for k, v in sd.items()})


def _check_records(W, rec, B):
    with torch.no_grad():
        ref = run_ref(W, {}, B, given=rec)
        A = run_ref(abs_weights(W), {}, B, given={k: v.abs() for k, v in rec.items()})
    return check(rec, ref, A)


def test_checker_passes_clean_records(packed):
    inputs = _inputs(4, FH, FW, FR, 7)
    with torch.no_grad():
        rec = run_ref(packed, inputs, 2, emulate=True).rec
    bad, ratio = _check_records(packed, rec, 2)
    assert not bad, bad
    assert max(ratio.values()) <= 1.0


@pytest.mark.parametrize("fault", sorted(FAULTS))
def test_checker_names_the_faulty_role(packed, fault):
    role, f = FAULTS[fault]
    inputs = _inputs(4, FH, FW, FR, 7)
    with torch.no_grad():
        rec = run_ref(packed, inputs, 2, emulate=True, faults={role: f}).rec
    bad, _ = _check_records(packed, rec, 2)
    assert list(bad) == [role], bad
