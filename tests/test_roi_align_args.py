"""CPU: argument rules of the RoIAlign entry points.  Every call here carries fake device addresses and is refused
with SB_EINVAL (-22) before any launch, so no device is needed; the accepted neighbour of each rule runs on the GPU
(tests/test_gpu_roi_heads.py: slices with out_coff + C == out_ld, the 512-wide concat, C = 512 at P = 14, R = 0)."""
import ctypes

import pytest
import torch

from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import ops as G

EINVAL = -22
BASE = 0x7f0000000000          # fake device addresses, 16 MB apart
A_F = [BASE + i * (1 << 24) for i in range(4)]
A_ROIS, A_OUT = BASE + 4 * (1 << 24), BASE + 5 * (1 << 24)
SHAPES = ((150, 497), (75, 249), (38, 125), (19, 63))


@pytest.fixture(scope="module")
def lib():
    from stereo_rcnn_b200 import build
    build.build()
    return L.load()


def pyramid_call(lib, C=256, R=300, pooled=7, out_ld=512, out_coff=256, mode=2, shapes=SHAPES, feats=None,
                 rois=A_ROIS, out=A_OUT):
    fp = (ctypes.c_void_p * 4)(*(A_F if feats is None else feats))
    hs = (ctypes.c_int * 4)(*[s[0] for s in shapes])
    ws = (ctypes.c_int * 4)(*[s[1] for s in shapes])
    return lib.sb_roi_align_pyramid_nhwc(fp, hs, ws, C, 600.0, rois, R, pooled, out, out_ld, out_coff, mode, None)


def with_level(l, shape):
    s = list(SHAPES)
    s[l] = shape
    return tuple(s)


# (id, overrides): each is one rule's rejected call; the defaults are the engine's right-image box-head call
REJECT = [
    ("out_coff_negative", dict(out_coff=-4)),
    ("out_coff_not4", dict(out_coff=2)),
    ("slice_past_row", dict(out_ld=512, out_coff=260)),          # out_coff + C = 516 > 512
    ("slice_past_dense_row", dict(out_ld=256, out_coff=4)),
    ("out_ld_not4", dict(out_ld=514, out_coff=0)),
    ("C_zero", dict(C=0, out_coff=0)),
    ("C_negative", dict(C=-4, out_coff=0)),
    ("C_not4", dict(C=254, out_coff=0)),
    ("R_negative", dict(R=-1)),
    ("pooled_zero", dict(pooled=0)),
    ("mode_3", dict(mode=3)),
    ("mode_negative", dict(mode=-1)),
    ("level0_one_row", dict(shapes=with_level(0, (1, 497)))),
    ("level1_one_col", dict(shapes=with_level(1, (75, 1)))),
    ("level2_empty", dict(shapes=with_level(2, (0, 125)))),
    ("level3_one_row", dict(shapes=with_level(3, (1, 63)))),
    ("level3_null", dict(feats=A_F[:3] + [None])),
    ("level1_null", dict(feats=[A_F[0], None] + A_F[2:])),
    ("rois_null", dict(rois=None)),
    ("out_null", dict(out=None)),
    ("smem_over_200k", dict(C=2048, pooled=14, out_ld=2048, out_coff=0)),    # 245 760 + 4 800 bytes
    # a rejected argument is rejected also when there is nothing to pool
    ("R0_slice_past_row", dict(R=0, out_coff=260)),
    ("R0_level_one_row", dict(R=0, shapes=with_level(3, (1, 63)))),
]


@pytest.mark.parametrize("name,kw", REJECT, ids=[r[0] for r in REJECT])
def test_pyramid_rejects_before_launch(lib, name, kw):
    n0 = lib.sb_launch_count()
    assert pyramid_call(lib, **kw) == EINVAL, name
    assert lib.sb_launch_count() == n0


@pytest.mark.parametrize("H,W", [(1, 60), (40, 1), (1, 1), (0, 60)])
def test_roi_align_forward_backward_reject_maps_below_2x2(lib, H, W):
    """with H = 1 a tap in [0, 1) has hstart = min(0, H-2) = -1: the row before the map"""
    n0 = lib.sb_launch_count()
    args = (BASE, 1, 32, H, W, A_ROIS, 10, 8, 8, 0.25, A_OUT, None)
    assert lib.sb_roi_align_forward(*args) == EINVAL
    assert lib.sb_roi_align_backward(*args) == EINVAL
    assert lib.sb_launch_count() == n0


def test_pyramid_op_checks_the_levels():
    """ops.roi_align_pyramid_nhwc asserts on the tensors before it reaches the library"""
    rois = torch.zeros(3, 5)
    good = [torch.zeros(1, h, w, 8) for h, w in ((8, 12), (4, 6), (2, 3), (2, 2))]
    bad_sets = [
        good[:3],                                                         # three levels
        good[:1] + [torch.zeros(1, 4, 6, 12)] + good[2:],                 # C differs
        good[:2] + [good[2].double()] + good[3:],                         # fp64
        good[:2] + [good[2].half()] + good[3:],                           # fp16
        good[:3] + [torch.zeros(1, 8, 2, 2).permute(0, 2, 3, 1)],         # NCHW memory seen as NHWC
        good[:3] + [torch.zeros(1, 2, 4, 8)[:, :, :2]],                   # a column slice
        good[:3] + [torch.zeros(2, 2, 8)],                                # not 4-D
        good[:3] + [torch.zeros(1, 2, 2, 8, device="meta")],              # not on the RoIs' device
    ]
    for fs in bad_sets:
        with pytest.raises(AssertionError):
            G.roi_align_pyramid_nhwc(fs, 32.0, rois, 7)
