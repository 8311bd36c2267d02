"""CPU: the trunk + FPN backward returns gradients for exactly the reference's trainable set
(lib/model/stereo_rcnn/resnet.py:289-309 of the reference): RCNN_layer0 frozen, cfg.RESNET.FIXED_BLOCKS = k freezes
RCNN_layer1..k, every BatchNorm frozen, the FPN top / lateral / smooth convs always trainable."""
import pytest

from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200.synth import param_shapes

FPN = ("RCNN_toplayer", "RCNN_latlayer1", "RCNN_latlayer2", "RCNN_latlayer3", "RCNN_smooth1", "RCNN_smooth2",
       "RCNN_smooth3")


def restated_trainable(fixed_blocks):
    """resnet.py:289-309 restated over the state-dict names of the trunk + FPN"""
    names = set()
    for name in param_shapes():
        if name.endswith(("running_mean", "running_var", "num_batches_tracked")):
            continue
        top = name.split(".")[0]
        if top.startswith("RCNN_layer"):
            layer = int(top[len("RCNN_layer"):])
            if layer == 0 or layer <= fixed_blocks:
                continue
            sub = name.split(".")[3]
            if sub.startswith("bn") or name.split(".")[3:5] == ["downsample", "1"]:
                continue
            names.add(name)
        elif top in FPN:
            names.add(name)
    return names


@pytest.mark.parametrize("fixed_blocks", [0, 1, 2, 3])
def test_trainable_set_matches_reference_rule(fixed_blocks):
    got = E.trainable_trunk_fpn_params(fixed_blocks)
    names = [n for n, _ in got]
    assert len(names) == len(set(names))
    assert set(names) == restated_trainable(fixed_blocks)
    shapes = param_shapes()
    for n, s in got:
        assert tuple(shapes[n]) == tuple(s), n


def test_fixed_blocks_out_of_range():
    with pytest.raises(AssertionError):
        E.trainable_trunk_fpn_params(4)
