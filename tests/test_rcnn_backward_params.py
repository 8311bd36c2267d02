"""CPU: the R-CNN heads' backward returns gradients for exactly the heads' parameters, in the reference's layout, and
the three gradient producers (trunk + FPN, RPN, heads) together with the frozen parameters cover the whole model."""
import pytest

from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200.synth import param_shapes

HEAD_PREFIXES = ("RCNN_top.", "RCNN_cls_score.", "RCNN_bbox_pred.", "RCNN_dim_orien_pred.", "RCNN_kpts.",
                 "kpts_class.")


@pytest.mark.parametrize("n_classes", [2, 3])
def test_trainable_rcnn_head_params_match_reference_module(n_classes):
    got = E.trainable_rcnn_head_params(n_classes)
    names = [n for n, _ in got]
    assert len(names) == len(set(names)) == 26
    shapes = param_shapes(n_classes)
    assert set(names) == {n for n in shapes if n.startswith(HEAD_PREFIXES)}
    for n, s in got:
        assert tuple(shapes[n]) == tuple(s), n


def _frozen(fixed_blocks):
    """layer0, every BatchNorm, and the convs of RCNN_layer1..fixed_blocks (resnet.py:289-309 of the reference)"""
    out = set()
    for n in param_shapes():
        if n.startswith("RCNN_layer0."):
            out.add(n)
        elif n.startswith("RCNN_layer"):
            li = int(n[len("RCNN_layer")])
            mod = n.rsplit(".", 1)[0]
            if li <= fixed_blocks or mod.endswith((".bn1", ".bn2", ".bn3", ".downsample.1")):
                out.add(n)
    return out


@pytest.mark.parametrize("fixed_blocks", [0, 1, 2, 3])
def test_gradient_producers_partition_the_model(fixed_blocks):
    heads = {n for n, _ in E.trainable_rcnn_head_params()}
    rpn = {n for n, _ in E.trainable_rpn_params()}
    trunk = {n for n, _ in E.trainable_trunk_fpn_params(fixed_blocks)}
    frozen = _frozen(fixed_blocks)
    assert not heads & rpn and not heads & trunk and not rpn & trunk
    assert not frozen & (heads | rpn | trunk)
    assert heads | rpn | trunk | frozen == set(param_shapes())
