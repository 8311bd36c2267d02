"""GPU: every packed weight copy StereoRCNNEngine holds, against a torch restatement of its layout from the state_dict
(bit for bit, in the fp16, tf32 and exact-fp32 modes, data-gradient copies included); refresh_weights refuses the
frozen tensors, and an engine refreshed before its first backward packs its data-gradient copies from the refreshed
values."""
import pytest
import torch

from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200 import ops as G
from stereo_rcnn_b200.synth import make_state_dict
from test_gpu_train_step import bits, engine_tensors, perturbed

pytestmark = pytest.mark.gpu

MODES = {"fp16": dict(precision="fp16"), "tf32": dict(precision="tf32"), "simt": dict(conv_impl="simt")}
TRAINABLE = [n for n, _ in E.trainable_trunk_fpn_params(0) + E.trainable_rpn_params() + E.trainable_rcnn_head_params()]


def restated(sd, mode):
    """{engine_tensors name: CPU tensor} of an engine built in `mode` from sd, data-gradient copies included"""
    sd = {k: v.float() for k, v in sd.items()}
    out = {}

    def fwd(key, w, scale, shift):
        """[Cout,Cin,kh,kw] -> [Cout][kh][kw][Cin], TF32-rounded on the tensor-core paths, an fp16 twin in fp16"""
        k = w.permute(0, 2, 3, 1).contiguous()
        out["p.%s.w" % key] = k if mode == "simt" else G.round_tf32_(k.clone())
        if mode == "fp16":
            out["p.%s.w16" % key] = k.half()
        for f, t in (("scale", scale), ("shift", shift)):
            if t is not None:
                out["p.%s.%s" % (key, f)] = t

    def dgrad(key, w, scale=None):
        """[Cout,Cin,kh,kw] -> [Cin][kh][kw][Cout] fp16, taps flipped, the frozen-BN scale folded in"""
        if scale is not None:
            w = w * scale.view(-1, 1, 1, 1)
        out["bwd." + key] = w.flip(2, 3).permute(1, 2, 3, 0).contiguous().half()

    def bn(k):
        s = sd[k + ".weight"] / torch.sqrt(sd[k + ".running_var"] + E.EPS)
        return s, sd[k + ".bias"] - sd[k + ".running_mean"] * s

    # stem: [64][7][7][3] fp32; 64 rows of the 147 taps in (ci, r, s) order padded to 160 (GEMM) and 192 (fp16)
    w = sd["RCNN_layer0.0.weight"]
    s, b = bn("RCNN_layer0.1")
    out["stem0"], out["stem1"], out["stem2"] = w.permute(0, 2, 3, 1).contiguous(), s, b
    wg = torch.zeros(64, 160, 1, 1)
    wg[:, :147, 0, 0] = w.reshape(64, 147)
    fwd("stem_gemm", wg, s, b)
    w16 = torch.zeros(64, 192)
    w16[:, :147] = w.reshape(64, 147)
    out["stem_w16"] = w16.half()
    convs = [n[:-len(".weight")] for n, _ in E.trainable_trunk_fpn_params(0) if n.endswith(".weight")]
    for key in convs + ["RCNN_rpn.RPN_Conv", "RCNN_top.3"] + ["RCNN_kpts.%d" % i for i in range(0, 12, 2)]:
        w = sd[key + ".weight"]
        if key.startswith("RCNN_layer"):
            s, b = bn(key.replace("conv", "bn").replace("downsample.0", "downsample.1"))
            fwd(key, w, s, b)
            dgrad(key, w, s)
        else:
            fwd(key, w, None, sd[key + ".bias"])
            dgrad(key, w)
    # RPN heads fused: rows 0..5 cls, 6..23 box, zero to 32 rows (forward) and 64 (data gradient)
    wh, bh = torch.zeros(64, 1024, 1, 1), torch.zeros(32)
    wh[0:6], wh[6:24] = sd["RCNN_rpn.RPN_cls_score.weight"], sd["RCNN_rpn.RPN_bbox_pred_left_right.weight"]
    bh[0:6], bh[6:24] = sd["RCNN_rpn.RPN_cls_score.bias"], sd["RCNN_rpn.RPN_bbox_pred_left_right.bias"]
    fwd("rpn_heads", wh[:32], None, bh)
    dgrad("rpn_heads", wh)
    # RCNN_top.0 as a 1x1 conv over (ph, pw, c)
    w0 = sd["RCNN_top.0.weight"].permute(0, 2, 3, 1).reshape(2048, 7 * 7 * 512, 1, 1)
    fwd("RCNN_top.0", w0, None, sd["RCNN_top.0.bias"])
    dgrad("RCNN_top.0", w0)
    # deconv [Cin,Cout,2,2]: phase (a, b) = the 1x1 conv W[:, :, a, b]^T; data gradient channel (a, b, co)
    wd = sd["RCNN_kpts.12.weight"]
    for a in range(2):
        for b in range(2):
            fwd("deconv%d%d" % (a, b), wd[:, :, a, b].t().reshape(256, 256, 1, 1), None, sd["RCNN_kpts.12.bias"])
    dgrad("deconv", wd.permute(2, 3, 1, 0).reshape(1024, 256, 1, 1))
    for i, k in enumerate(("RCNN_cls_score.weight", "RCNN_cls_score.bias", "RCNN_bbox_pred.weight",
                           "RCNN_bbox_pred.bias", "RCNN_dim_orien_pred.weight", "RCNN_dim_orien_pred.bias")):
        out["fc%d" % i] = sd[k]
    out["kpts_class0"], out["kpts_class1"] = sd["kpts_class.weight"].reshape(6, 256), sd["kpts_class.bias"]
    return out


def assert_restated(eng, sd, mode):
    got, ref = engine_tensors(eng), restated(sd, mode)
    assert sorted(got) == sorted(ref)
    for k in ref:
        g = got[k].cpu()
        assert g.shape == ref[k].shape and g.dtype == ref[k].dtype, (k, g.shape, g.dtype, ref[k].shape, ref[k].dtype)
        assert torch.equal(bits(g), bits(ref[k])), k
    return len(ref)


@pytest.mark.parametrize("mode", sorted(MODES))
def test_packed_weights_equal_their_restatement(mode, capsys):
    sd = perturbed(make_state_dict(3), TRAINABLE + ["RCNN_layer0.0.weight"], 21)
    eng = E.StereoRCNNEngine(sd, "cuda", **MODES[mode])
    assert eng._bwd is None             # an inference engine holds no data-gradient copy
    eng._pack_heads_backward()
    torch.cuda.synchronize()
    n = assert_restated(eng, sd, mode)
    with capsys.disabled():
        print("%s engine: %d packed tensors bit-identical to their restatement" % (mode, n))


def test_refresh_refuses_frozen_tensors():
    sd = make_state_dict(3)
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    for n in ("RCNN_layer0.0.weight", "RCNN_layer0.1.weight", "RCNN_layer1.0.0.bn1.running_var"):
        with pytest.raises(KeyError):
            eng.refresh_weights({n: sd[n].cuda()})


@pytest.mark.parametrize("before", ["nothing", "trunk copies"])
def test_refresh_before_the_first_backward(before):
    """the refresh packs the data-gradient copies first, so none of them is later packed from the constructor's
    values: with none held yet, and with those of the trunk, FPN and RPN only (what rpn_backward allocates)"""
    sd = make_state_dict(3)
    sd2 = perturbed(sd, TRAINABLE, 22)
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    if before == "trunk copies":
        eng._pack_backward()
        assert "rpn_heads" in eng._bwd and "RCNN_top.0" not in eng._bwd
    eng.refresh_weights({n: sd2[n].cuda() for n in TRAINABLE})
    eng._pack_heads_backward()
    torch.cuda.synchronize()
    assert_restated(eng, sd2, "fp16")
