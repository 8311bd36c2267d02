"""GPU: the fp16 forward (engine.trunk_fpn, rpn, heads) replayed layer by layer against float64, on the engine's own
fp16 operands, in both stream schedules, batched and at the benchmarked size.

Recorders wrap eng._conv and ops.stem_conv_tc, maxpool3x3s2_ceil, subsample2, roi_align_pyramid_nhwc and
rpn_head_epilogue: each calls the original, then clones its inputs and outputs on the current stream (the side stream
inside a fork), so later launches cannot overwrite them.  A conv is named by the identity of its PackedConv (eng.p,
eng.deconv), not by its tag; the launches of one role (the left and right chains of layers 3-4 under forks=True, the
two RPN_Conv launches of a level at B > 1) are put back together in the engine's image order.  ForwardRef
(test_forward_replay.py) then runs teacher-forced on the records, with the weights as the engine packs them, and
check() holds every role to it: fp32 outputs within the K-aware MMA bound C_MMA (K / 16 + 3) 2^-23 A plus the
epilogue's 8 2^-24 A element by element (RCNN_top.0 sums K = 25 088 terms, far past test_gpu_conv_tc.py's fixed
2^-12 A), fp16 twins the fp32 output rounded to nearest bit for bit, fp16-only outputs within one ulp of h16(ref) or
the rounding of a value within the bound, the max pool, subsample2, P6 and the box deltas bit for bit.

Besides the arithmetic the replay checks the wiring: each recorded conv's input, residual and upsample source are
bit-identical to the recorded output of the role the model feeds it from, the pooled tiles are a fresh RoIAlign of
the recorded P levels, and every conv launches the expected number of times on the tensor cores."""
import time

import pytest
import torch

from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200 import ops as G
from stereo_rcnn_b200.synth import make_state_dict
from test_forward_replay import (LEVELS, abs_weights, check, expected_uses, last_role, role_class, run_ref,
                                 weights_as_packed)
from test_gpu_rpn_backward import _pairs, _small_hw
from test_trunk_backward_replay import FPN, block

pytestmark = pytest.mark.gpu

FPN_ROLE = {"RCNN_toplayer": "p5"}
for _lvl, _smooth, _lat in FPN:
    FPN_ROLE.update({_smooth: "p%d" % _lvl, _lat: "t%d" % _lvl})


def conv_role(key):
    """the role of a conv's output, by state_dict key (RPN_Conv and the RPN heads by level, see Recorder.assemble)"""
    if key in FPN_ROLE:
        return FPN_ROLE[key]
    if key.startswith("RCNN_layer"):
        p, conv = key.rsplit(".", 1)
        if key.endswith(".downsample.0"):
            return key[:-len(".downsample.0")] + ".ds"
        if conv in ("conv1", "conv2"):
            return p + ".o" + conv[-1]
        L, b = int(p.split(".")[0][len("RCNN_layer"):]), int(p.split(".")[2])
        return last_role(L, b)
    if key.startswith("RCNN_kpts."):
        return "kpts" + key.split(".")[1]
    return {"RCNN_top.0": "top0", "RCNN_top.3": "fc7", "deconv": "up"}.get(key)


def _cl(t):
    return t.clone() if t is not None else None


class Recorder(object):
    """monkeypatched onto one engine's _conv and the ops the forward launches"""

    def __init__(self, eng, monkeypatch):
        self.convs, self.ops = [], []
        self.B = None
        ident = {id(pc): k for k, pc in eng.p.items()}
        for a in range(2):
            for b in range(2):
                ident[id(eng.deconv[a][b])] = "deconv"
        on_side = lambda: eng.side is not None and torch.cuda.current_stream() == eng.side
        conv0 = eng._conv

        def conv(x, pc, **kw):
            r = conv0(x, pc, **kw)
            o32, o16 = kw.get("out"), kw.get("out16")
            if isinstance(r, tuple):
                o32, o16 = r
            elif r.dtype == torch.float32:
                o32 = r
            else:
                o16 = r
            key = ident[id(pc)]
            if key == "deconv":           # the four phases write strided views of one tensor: keep all of it
                o16 = o16._base
            self.convs.append(dict(key=key, side=on_side(), x=x.clone(), out=_cl(o32), out16=_cl(o16),
                                   res=_cl(kw.get("residual")), up=_cl(kw.get("up_src")),
                                   coff=kw.get("out_coff", 0), stride=kw.get("stride", 1)))
            return r

        def wrap(name):
            f0 = getattr(G, name)

            def f(*a, **kw):
                r = f0(*a, **kw)
                ins = [t.clone() if torch.is_tensor(t) else t for t in a]
                outs = [t.clone() for t in (r if isinstance(r, tuple) else (r,))]
                self.ops.append(dict(name=name, side=on_side(), ins=ins, kw=dict(kw), outs=outs))
                return r
            monkeypatch.setattr(G, name, f)
        monkeypatch.setattr(eng, "_conv", conv)
        for name in ("stem_conv_tc", "maxpool3x3s2_ceil", "subsample2", "roi_align_pyramid_nhwc",
                     "rpn_head_epilogue"):
            wrap(name)

    def assemble(self, B):
        """({role: fp32 record, role + "_16": fp16 record}, {role: {"x", "res", "up": the operands it read}},
        {key: launches}, {level: the RPN heads' input}) with the launches of one role in the engine's image order"""
        rec, inputs, count, head_in = {}, {}, {}, {}
        ops = {}
        for o in self.ops:
            ops.setdefault(o["name"], []).append(o)
        stem, = ops["stem_conv_tc"]
        rec["image_16"], rec["stem_16"] = stem["ins"][0].half(), stem["outs"][0]
        mp, = ops["maxpool3x3s2_ceil"]
        rec["c1_16"] = mp["outs"][0]
        inputs["c1"] = dict(x=mp["ins"][0])
        inputs["stem"] = dict(x=stem["ins"][0])
        by_role = {}
        for c in self.convs:
            count[c["key"]] = count.get(c["key"], 0) + 1
            role = conv_role(c["key"])
            if role is not None:
                by_role.setdefault(role, []).append(c)
        for role, cs in by_role.items():
            order = sorted(cs, key=lambda c: c["side"])       # the right images' chain runs on the side stream
            cat = lambda k: (torch.cat([c[k] for c in order]) if len(order) > 1 else order[0][k]) \
                if order[0][k] is not None else None
            if role == "up":          # four phases, one launch each, on the same input
                assert all(torch.equal(c["x"], cs[0]["x"]) for c in cs)
                rec["up_16"] = cs[-1]["out16"]
                inputs[role] = dict(x=cs[0]["x"], res=None, up=None)
                continue
            else:
                if cs[0]["out"] is not None:
                    rec[role] = cat("out")
                if cs[0]["out16"] is not None:
                    rec[role + "_16"] = cat("out16")
            inputs[role] = dict(x=cat("x"), res=cat("res"), up=cat("up"))
        shape_of = {tuple(rec[k + "_16"].shape[1:3]): k for k in LEVELS if k != "p6"}
        # P6 and the strided inputs of layers 2-4, by the map subsample2 reads
        srcs = {tuple(rec["c%d_16" % L].shape[1:]): block(L, 0) + ".xin" for L in (2, 3, 4)}
        xin = {}
        for o in ops["subsample2"]:
            x = o["ins"][0]
            if tuple(x.shape[1:]) == tuple(rec["p5"].shape[1:]):
                rec["p6" if x.dtype == torch.float32 else "p6_16"] = o["outs"][0]
                inputs.setdefault("p6", {})["x" if x.dtype == torch.float32 else "x16"] = x
            else:
                xin.setdefault(srcs[tuple(x.shape[1:])], []).append(o)
        for role, os_ in xin.items():
            os_ = sorted(os_, key=lambda o: o["side"])
            rec[role + "_16"] = torch.cat([o["outs"][0] for o in os_])
            inputs[role] = dict(x=torch.cat([o["ins"][0] for o in os_]))
        shape_of.update({tuple(rec["p6_16"].shape[1:3]): "p6"})
        assert len(shape_of) == 5, "two P levels of one size"
        # RPN: RPN_Conv by level (the left launch, then the right one at B > 1, both into one buffer), the heads
        for c in self.convs:
            if c["key"] == "RCNN_rpn.RPN_Conv":
                lvl = shape_of[tuple(c["x"].shape[1:3])]
                rec["rpn_cat.%s_16" % lvl] = c["out16"]        # the last launch's copy holds both halves
                inputs.setdefault("rpn_cat." + lvl, dict(x=[]))["x"].append((c["coff"], c["x"], c["res"], c["up"]))
            elif c["key"] == "rpn_heads":
                head_in[shape_of[tuple(c["x"].shape[1:3])]] = c["x"]
        for lvl in LEVELS:
            parts = sorted(inputs["rpn_cat." + lvl]["x"], key=lambda p: p[0])
            assert [p[0] for p in parts] == ([0] if B == 1 else [0, 512]), parts
            assert all(p[2] is None and p[3] is None for p in parts)
            inputs["rpn_cat." + lvl] = dict(x=torch.cat([p[1] for p in parts]), res=None, up=None)
        ep, = ops["rpn_head_epilogue"]
        rec["rpn_head"], (rec["rpn_cls_prob"], rec["rpn_bbox_pred"]) = ep["ins"][0], ep["outs"]
        if "top0" in inputs:
            R = inputs["top0"]["x"].shape[0]
            rec["pooled_box_16"] = inputs["top0"]["x"].view(R, 7, 7, 512)
            rec["pooled_kpts_16"] = inputs["kpts0"]["x"]
        return rec, inputs, count, head_in


def expected_counts(forks, B, heads):
    """launches per key: the stem is not a _conv; layer 3-4 convs twice under forks (left chain, right chain)"""
    out = {}
    for k, n in expected_uses(rpn=True, heads=heads).items():
        if k in ("RCNN_layer0.0", "RCNN_rpn.RPN_cls_score", "RCNN_rpn.RPN_bbox_pred_left_right"):
            continue
        if k == "RCNN_rpn.RPN_Conv":
            n = 5 if B == 1 else 10
        elif k.startswith(("RCNN_layer3", "RCNN_layer4")) and forks:
            n = 2
        out["deconv" if k == "RCNN_kpts.12" else k] = 4 if k == "RCNN_kpts.12" else n
    out["rpn_heads"] = 5
    return out


def _abs(d):
    return {k: v.abs() for k, v in d.items()}


def replay(monkeypatch, sd, H, W, B, forks, heads, label, seed=5):
    """one recorded forward, checked role by role; returns (engine, images, records, trunk features)"""
    t0 = time.time()
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16", forks=forks)
    im = _pairs(H, W, B, seed).cuda()
    rec_ = Recorder(eng, monkeypatch)
    with torch.no_grad():
        feats = eng.trunk_fpn(im)
        cls_prob, bbox, shapes = eng.rpn(feats, B)
        if heads:
            info = torch.tensor([[float(H), float(W), 1.0]] * B, device="cuda")
            rl, rr = G.proposal_layer(cls_prob, bbox, info, "TEST", shapes)
            rois_l, rois_r = rl.view(-1, 5), rr.view(-1, 5)
            eng.heads(feats, B, rois_l, rois_r, float(H))
    torch.cuda.synchronize()
    monkeypatch.undo()
    rec, inputs, count, head_in = rec_.assemble(B)
    bad = []
    # ---- structure: every conv as often as the schedule launches it, all on the tensor cores
    want = expected_counts(forks, B, heads)
    assert count == want, sorted((k, count.get(k), want.get(k)) for k in set(count) | set(want)
                                 if count.get(k) != want.get(k))
    assert all(v.startswith("tc") for v in eng.impl_used.values()), eng.impl_used
    for c in rec_.convs:
        if forks and c["key"].startswith(("RCNN_layer3", "RCNN_layer4")):
            assert c["x"].shape[0] == B, c["key"]
    assert not bool(rec["rpn_head"][..., 24:].any()), "RPN head padding columns not zero"
    Wt = weights_as_packed(sd, "cuda")
    with torch.no_grad():
        ref = run_ref(Wt, {}, B, given=rec, heads=heads)
        A = run_ref(abs_weights(Wt), {}, B, given=_abs(rec), heads=heads)
        # ---- the wiring: every operand is the recorded output of the role the model feeds it from
        for role, rd in ref.reads.items():
            if role in ("rpn_head", "rpn_cls_prob", "rpn_bbox_pred"):
                continue
            got = inputs[role]
            if role == "p6":
                ok = torch.equal(got["x"], rec["p5"]) and torch.equal(got["x16"], rec["p5_16"])
            elif role == "stem":
                ok = torch.equal(got["x"], im)
            elif role in ("top0", "kpts0"):
                continue            # the pooled tiles: checked against a fresh RoIAlign below
            else:
                ok = torch.equal(got["x"], rec[rd["x"] + "_16"])
                for k in ("res", "up"):
                    if k in rd:
                        ok = ok and got[k] is not None and torch.equal(got[k], rec[rd[k]])
                    elif k in got:
                        ok = ok and got[k] is None
            if not ok:
                bad.append((role, "reads the wrong operand"))
        for lvl in LEVELS:
            if not torch.equal(head_in[lvl], rec["rpn_cat.%s_16" % lvl]):
                bad.append(("rpn_head", "level %s reads the wrong operand" % lvl))
        if heads:
            fl = [rec[k][:B] for k in ("p2", "p3", "p4", "p5")]
            fr = [rec[k][B:] for k in ("p2", "p3", "p4", "p5")]
            R = rois_l.shape[0]
            box = torch.empty(R, 7, 7, 512, dtype=torch.float16, device="cuda")
            G.roi_align_pyramid_nhwc(fl, float(H), rois_l, 7, out=box, out_coff=0, half=True)
            G.roi_align_pyramid_nhwc(fr, float(H), rois_r, 7, out=box, out_coff=256, half=True)
            if not torch.equal(box, rec["pooled_box_16"]):
                bad.append(("pooled_box", "not RoIAlign of the left P levels | the right ones"))
            if not torch.equal(G.roi_align_pyramid_nhwc(fl, float(H), rois_l, 14, half=True), rec["pooled_kpts_16"]):
                bad.append(("pooled_kpts", "not RoIAlign of the left P levels"))
        # ---- the arithmetic, role by role
        fails, ratio = check(rec, ref, A)
        bad += sorted(fails.items())
    worst = {}
    for role, r in ratio.items():
        c = role_class(role)
        if c not in worst or r > worst[c][0]:
            worst[c] = (r, role)
    print("%s (%.1f s): worst err / bound per class: %s" % (
        label, time.time() - t0, ", ".join("%s %.3f (%s)" % (c, r, n) for c, (r, n) in sorted(worst.items()))))
    assert not bad, bad[:20]
    return eng, im, rec, inputs, feats


@pytest.fixture(scope="module")
def sd():
    return make_state_dict(3)


@pytest.mark.parametrize("forks", [True, False])
def test_replay_small(monkeypatch, sd, forks):
    """160x256 B = 1: the latency schedule (forks=True) and the throughput schedule (forks=False)"""
    H, W = _small_hw()
    replay(monkeypatch, sd, H, W, 1, forks, True, "%dx%d B=1 forks=%s" % (H, W, forks))


def test_replay_odd_maps(monkeypatch, sd):
    """200x330: c2 50x82, c3 25x41, c4 13x21, c5 7x11: the stride-2 blocks of layers 3 and 4 read odd maps"""
    eng, im, rec, inputs, feats = replay(monkeypatch, sd, 200, 330, 1, True, True, "200x330 B=1 forks=True")
    assert [tuple(rec["c%d" % k].shape[1:3]) for k in range(2, 6)] == [(50, 82), (25, 41), (13, 21), (7, 11)]


@pytest.mark.parametrize("forks", [True, False])
def test_replay_batched(monkeypatch, sd, forks):
    """B = 2 pairs: the batched chains, the two-launch RPN_Conv path, 2 x 300 head rows"""
    H, W = _small_hw()
    replay(monkeypatch, sd, H, W, 2, forks, True, "%dx%d B=2 forks=%s" % (H, W, forks))


def test_replay_benchmark_size_latency(monkeypatch, sd):
    """the benchmarked 600x1987 pair in the latency schedule: trunk, FPN and RPN"""
    replay(monkeypatch, sd, 600, 1987, 1, True, False, "600x1987 B=1 forks=True", seed=3)


def test_replay_benchmark_size_throughput(monkeypatch, sd):
    """the benchmarked 600x1987 pair in the throughput schedule, the heads on its proposals included"""
    replay(monkeypatch, sd, 600, 1987, 1, False, True, "600x1987 B=1 forks=False", seed=3)


def test_training_forward_is_the_inference_forward(monkeypatch, sd):
    """trunk_fpn(save_for_backward=True), which never forks, gives the forked inference forward's features bit for
    bit, and every tensor it saves for the backward is the operand the recorded conv read"""
    H, W = _small_hw()
    eng, im, rec, inputs, feats = replay(monkeypatch, sd, H, W, 1, True, False, "%dx%d B=1 forks=True" % (H, W))
    with torch.no_grad():
        f2, saved = eng.trunk_fpn(im, save_for_backward=True)
    torch.cuda.synchronize()
    for k in ("c2", "c3", "c4", "c5") + LEVELS:
        for kk in (k, k + "_16"):
            assert torch.equal(f2[kk], feats[kk]), kk
    for L in range(1, 5):
        for b in range(E.LAYERS[L - 1]):
            p = block(L, b)
            assert torch.equal(saved[p]["xin"], inputs[p + ".o1"]["x"]), p
            assert torch.equal(saved[p]["o1"], rec[p + ".o1_16"]), p
            assert torch.equal(saved[p]["o2"], rec[p + ".o2_16"]), p
    for k in ("c2", "c3", "c4", "c5", "t2", "t3", "t4"):
        assert torch.equal(saved[k], rec[k + "_16"]), k


# ---------------------------------------------------------------------------------------------------- invariance
FEATS = tuple(k + s for k in ("c2", "c3", "c4", "c5") + LEVELS for s in ("", "_16"))


def _forward(eng, H, W, B, seed=5):
    im = _pairs(H, W, B, seed).cuda()
    info = torch.tensor([[float(H), float(W), 1.0]] * B, device="cuda")
    with torch.no_grad():
        out = eng.forward(im[:B], im[B:], info, keep_features=True)
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("B", [1, 2])
def test_schedules_bit_identical(sd, B):
    """forks=True and forks=False launch the same arithmetic: every output element is one K-ordered wgmma
    accumulation whatever the tile width or M, and the forward has no split-K, so every feature and every output
    is the same bits"""
    H, W = _small_hw()
    a, b = (_forward(E.StereoRCNNEngine(sd, "cuda", precision="fp16", forks=f), H, W, B) for f in (True, False))
    for k in FEATS:
        assert torch.equal(a["feats"][k], b["feats"][k]), k
    for k, v in a.items():
        if torch.is_tensor(v):
            assert torch.equal(v, b[k]), k


def test_pair_in_batch_bit_identical(sd):
    """pair j of a B = 2 batch gives the bits of pair j run alone: features, RPN outputs, proposals, head outputs"""
    H, W = _small_hw()
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    both = _forward(eng, H, W, 2)
    n = both["rois_left"].shape[1]
    for j in range(2):
        one = _forward(eng, H, W, 1, seed=5 + j)
        for k in FEATS:
            assert torch.equal(both["feats"][k][[j, 2 + j]], one["feats"][k]), (j, k)
        for k in ("rpn_cls_prob", "rpn_bbox_pred", "cls_prob", "bbox_pred", "dim_orien_pred"):
            assert torch.equal(both[k][j], one[k][0]), (j, k)
        for k in ("rois_left", "rois_right"):
            assert torch.equal(both[k][j, :, 1:], one[k][0, :, 1:]), (j, k)
        for k in ("pooled_box", "pooled_kpts", "fc7", "kpts_prob", "left_border_prob", "right_border_prob",
                  "kpts_pred_all"):
            assert torch.equal(both[k][j * n:(j + 1) * n], one[k]), (j, k)
