"""CPU: the RPN backward returns gradients for exactly the stereo RPN's parameters, in the reference's layout
(lib/model/rpn/stereo_rpn.py:32-39 of the reference, restated below), and the conv descriptor's explicit input pitch
that lets the RPN_Conv data gradient read one half of the 1024-channel `cat` gradient."""
import torch

from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200 import ops
from stereo_rcnn_b200.synth import param_shapes


def restated_rpn_module(din=256, n_ratios=3):
    """stereo_rpn.py:32-39: RPN_Conv = Conv2d(din, 512, 3, 1, 1, bias=True); RPN_cls_score = Conv2d(512*2,
    n_ratios*2, 1, 1, 0); RPN_bbox_pred_left_right = Conv2d(512*2, n_ratios*6, 1, 1, 0); din = 256 (the FPN width)"""
    nc_score, nc_bbox = n_ratios * 2, n_ratios * 6
    return {"RCNN_rpn.RPN_Conv.weight": (512, din, 3, 3), "RCNN_rpn.RPN_Conv.bias": (512,),
            "RCNN_rpn.RPN_cls_score.weight": (nc_score, 1024, 1, 1), "RCNN_rpn.RPN_cls_score.bias": (nc_score,),
            "RCNN_rpn.RPN_bbox_pred_left_right.weight": (nc_bbox, 1024, 1, 1),
            "RCNN_rpn.RPN_bbox_pred_left_right.bias": (nc_bbox,)}


def test_trainable_rpn_params_match_reference_module():
    got = E.trainable_rpn_params()
    names = [n for n, _ in got]
    assert len(names) == len(set(names))
    assert dict(got) == restated_rpn_module()
    shapes = param_shapes()
    assert {n for n in shapes if n.startswith("RCNN_rpn.")} == set(names)
    for n, s in got:
        assert tuple(shapes[n]) == tuple(s), n


def test_rpn_and_trunk_sets_are_disjoint():
    """rpn_gradients returns the union: no name may be produced by both backward passes"""
    rpn = {n for n, _ in E.trainable_rpn_params()}
    for fb in range(4):
        assert not rpn & {n for n, _ in E.trainable_trunk_fpn_params(fb)}


def test_conv_desc_input_pitch():
    """in_ld defaults to the input's channel count; a channel-half view of a [B,h,w,1024] tensor passes 1024"""
    cat = torch.zeros(1, 3, 5, 1024, dtype=torch.float16)
    w = torch.zeros(256, 3, 3, 512, dtype=torch.float16)
    out = torch.zeros(1, 3, 5, 256)
    half = cat[..., 512:]
    d = ops.conv_desc(half, w, out, 512, 256, 3, 3, 1, 1, 3, 5)
    assert d.in_ld == 512
    d = ops.conv_desc(half, w, out, 512, 256, 3, 3, 1, 1, 3, 5, in_ld=1024)
    assert d.in_ld == 1024 and d.in_ == half.data_ptr() == cat.data_ptr() + 1024
