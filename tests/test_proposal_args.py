"""CPU: the selection entry points (sb_nms, sb_nms_mask, sb_proposal_layer, sb_generate_anchors, sb_class_nms) refuse
every invalid argument with SB_EINVAL before any CUDA call, and the oracle ranks scores as torch.sort(descending=True,
stable=True) does -- every NaN above +inf, -0.0 equal to +0.0, ties by ascending index -- which is the order the
proposal layer and the per-class NMS kernels implement."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from oracle import ops as O
from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import ops as G

SB_EINVAL = -22
FAKE = 1 << 20                                            # never dereferenced: every refusal precedes the first call
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
BIG = 1 << 40                                             # a workspace size no check can refuse
SHAPES = [[20, 32], [10, 16], [5, 8], [3, 4], [2, 2]]
A_SMALL = 3 * sum(h * w for h, w in SHAPES)


@pytest.fixture(scope="module")
def lib():
    from stereo_rcnn_b200 import build
    build.build()
    return L.load()


def cfg(shapes=SHAPES, **over):
    pc = G.make_proposal_cfg("TEST", shapes)
    for k, v in over.items():
        if k == "level":                                  # (level, field, value): shapes as "h" / "w"
            l, f, x = v
            if f in ("h", "w"):
                pc.shapes[l][f == "w"] = x
            else:
                getattr(pc, f)[l] = x
        elif k == "ratio":
            pc.ratios[v[0]] = v[1]
        else:
            setattr(pc, k, v)
    return pc


def without_device(check):
    """run check(lib) in a child process that sees no CUDA device.  The calls pass fake device pointers; if a refusal
    regressed, the call would go on to a launch, which then fails with a CUDA error (and the test with it) instead of
    reading or writing those addresses on a real GPU."""
    code = ("import sys; sys.path[:0] = %r; from stereo_rcnn_b200 import lib as L; import test_proposal_args as T; "
            "T.%s(L.load())" % ([ROOT, HERE], check))
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(args, env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr


def test_nms_rejections(lib):
    without_device("nms_rejections")


def test_proposal_layer_rejections(lib):
    without_device("proposal_layer_rejections")


def test_generate_anchors_rejections(lib):
    without_device("generate_anchors_rejections")


def test_class_nms_rejections(lib):
    without_device("class_nms_rejections")


def nms_rejections(lib):
    nb = lib.sb_nms_workspace_bytes(16384)
    assert nb >= 16384 * 256 * 8

    def nms(dets=FAKE, n=100, keep=FAKE, num=FAKE, ws=FAKE, nbytes=nb):
        return lib.sb_nms(dets, n, 0.7, keep, num, ws, nbytes, None)

    def mask(dets=FAKE, n=100, m=FAKE):
        return lib.sb_nms_mask(dets, n, 0.7, m, None)
    n0 = lib.sb_launch_count()
    bad = {"nms: n < 0": nms(n=-1), "nms: null dets": nms(dets=None), "nms: null keep": nms(keep=None),
           "nms: null num_out": nms(num=None), "nms: null workspace": nms(ws=None),
           "nms: short workspace": nms(nbytes=lib.sb_nms_workspace_bytes(100) - 1),
           "nms: n = 16385": nms(n=16385, nbytes=BIG), "nms: n = 0, null keep": nms(n=0, keep=None),
           "mask: n < 0": mask(n=-1), "mask: null dets": mask(dets=None), "mask: null mask": mask(m=None),
           "mask: n = 16385": mask(n=16385)}
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}
    assert mask(n=0, dets=None, m=None) == 0 and lib.sb_launch_count() == n0        # n = 0: nothing to do


def proposal_layer_rejections(lib):
    inf, nan = float("inf"), float("nan")
    nb = lib.sb_proposal_workspace_bytes(2, A_SMALL, 6000)

    def call(pc=None, B=2, A=A_SMALL, prob=FAKE, bbox=FAKE, info=FAKE, rl=FAKE, rr=FAKE, ws=FAKE, nbytes=nb):
        pc = cfg() if pc is None else pc
        return lib.sb_proposal_layer(prob, bbox, info, B, A, ctypes.byref(pc), rl, rr, ws, nbytes, None)

    big = [[4096, 2048]]                                  # one level, one ratio: A = 2048 * 4096, the limit
    n0 = lib.sb_launch_count()
    bad = {"null cls_prob": call(prob=None), "null bbox_pred_lr": call(bbox=None), "null im_info": call(info=None),
           "null rois_left": call(rl=None), "null rois_right": call(rr=None), "null workspace": call(ws=None),
           "short workspace": call(nbytes=nb - 1), "B < 0": call(B=-1), "A != pyramid": call(A=A_SMALL + 1),
           "A = 0": call(cfg([[0, 32]]), A=0),
           "null cfg": lib.sb_proposal_layer(FAKE, FAKE, FAKE, 2, A_SMALL, None, FAKE, FAKE, FAKE, nb, None),
           "n_levels 0": call(cfg(n_levels=0)), "n_levels 9": call(cfg(n_levels=9)),
           "n_ratios 0": call(cfg(n_ratios=0)), "n_ratios 5": call(cfg(n_ratios=5)),
           "h 0": call(cfg(level=(2, "h", 0)), A=A_SMALL - 3 * 5 * 8),
           "w 0": call(cfg(level=(2, "w", 0)), A=A_SMALL - 3 * 5 * 8),
           "h < 0": call(cfg(level=(0, "h", -20)), A=A_SMALL - 2 * 3 * 20 * 32),
           "h < 0 and w < 0": call(_both_negative()),
           "scale 0": call(cfg(level=(3, "anchor_scales", 0))), "scale < 0": call(cfg(level=(0, "anchor_scales", -32))),
           "stride 0": call(cfg(level=(4, "feat_strides", 0))), "stride < 0": call(cfg(level=(0, "feat_strides", -4))),
           "ratio 0": call(cfg(ratio=(1, 0.0))), "ratio < 0": call(cfg(ratio=(0, -0.5))),
           "ratio inf": call(cfg(ratio=(2, inf))), "ratio nan": call(cfg(ratio=(2, nan))),
           "nms_thresh nan": call(cfg(nms_thresh=nan)), "nms_thresh inf": call(cfg(nms_thresh=inf)),
           "nms_thresh -inf": call(cfg(nms_thresh=-inf)),
           "post_nms_top_n 0": call(cfg(post_nms_top_n=0)), "post_nms_top_n -1": call(cfg(post_nms_top_n=-1)),
           "K = 16385 (pre)": call(cfg([[128, 128]], pre_nms_top_n=16385), A=3 * 128 * 128, nbytes=BIG),
           "K = 16385 (pre 0)": call(cfg([[1, 16385]], n_ratios=1, pre_nms_top_n=0), A=16385, nbytes=BIG),
           "A = 2048*4096 + 1": call(cfg([[1, 2048 * 4096 + 1]], n_ratios=1, pre_nms_top_n=100), A=2048 * 4096 + 1,
                                     nbytes=BIG),
           "h*w overflows int": call(cfg([[65536, 65536]], n_ratios=1, pre_nms_top_n=100), A=0, nbytes=BIG),
           "A overflows int": call(cfg([[32768, 32768]], n_ratios=3, pre_nms_top_n=100), A=-(1 << 30), nbytes=BIG),
           "levels sum overflows int": call(cfg([[32768, 32768]] * 3, n_ratios=1, pre_nms_top_n=100),
                                            A=(3 << 30) - (1 << 32), nbytes=BIG)}
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}
    # the same configuration with B = 0 passes every check and launches nothing; so do the limits themselves
    assert call(B=0, prob=None, bbox=None, info=None, rl=None, rr=None) == 0
    assert call(cfg([[1, 16384]], n_ratios=1, pre_nms_top_n=0), B=0, A=16384, nbytes=BIG) == 0
    assert call(cfg(big, n_ratios=1, pre_nms_top_n=16384), B=0, A=2048 * 4096, nbytes=BIG) == 0
    assert lib.sb_launch_count() == n0


def _both_negative():
    pc = cfg()
    pc.shapes[1][0], pc.shapes[1][1] = -10, -16          # a positive product from two negative extents
    return pc


def generate_anchors_rejections(lib):
    inf, nan = float("inf"), float("nan")

    def call(pc=None, A=A_SMALL, out=FAKE):
        return lib.sb_generate_anchors(None if pc is None else ctypes.byref(pc), A, out, None)
    n0 = lib.sb_launch_count()
    bad = {"null cfg": call(None), "null anchors": call(cfg(), out=None), "misaligned anchors": call(cfg(), out=FAKE + 4),
           "A != pyramid": call(cfg(), A=A_SMALL - 1), "A = 0": call(cfg([[0, 32]]), A=0),
           "n_levels 0": call(cfg(n_levels=0)), "n_levels 9": call(cfg(n_levels=9)), "n_ratios 0": call(cfg(n_ratios=0)),
           "n_ratios 5": call(cfg(n_ratios=5)), "h 0": call(cfg(level=(0, "h", 0))), "w < 0": call(_both_negative()),
           "scale 0": call(cfg(level=(1, "anchor_scales", 0))), "stride < 0": call(cfg(level=(2, "feat_strides", -8))),
           "ratio 0": call(cfg(ratio=(0, 0.0))), "ratio nan": call(cfg(ratio=(1, nan))), "ratio inf": call(cfg(ratio=(1, inf))),
           "h*w overflows int": call(cfg([[65536, 65536]], n_ratios=1), A=0)}
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}


def class_nms_rejections(lib):
    def call(scores=FAKE, boxes=FAKE, R=300, nc=2, cls=1, keep=FAKE, num=FAKE):
        return lib.sb_class_nms(scores, boxes, R, nc, cls, 0.05, 0.3, keep, num, None)
    n0 = lib.sb_launch_count()
    bad = {"null scores": call(scores=None), "null boxes": call(boxes=None), "null keep": call(keep=None),
           "null num_out": call(num=None), "R < 0": call(R=-1), "R = 513": call(R=513), "cls < 0": call(cls=-1),
           "cls = n_classes": call(cls=2), "n_classes 0": call(nc=0, cls=0)}
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}


SPECIALS = np.array([np.nan, -np.nan, np.inf, -np.inf, 0.0, -0.0, 1.0, 0.5, np.finfo(np.float32).tiny / 8,
                     -np.finfo(np.float32).tiny / 8, np.float32(1) - np.finfo(np.float32).epsneg], np.float32)


@pytest.mark.parametrize("n, seed", [(7, 0), (64, 1), (1000, 2), (50000, 3)])
def test_oracle_order_is_torch_sort_descending_stable(n, seed):
    rs = np.random.RandomState(seed)
    x = SPECIALS[rs.randint(0, SPECIALS.size, n)]
    # NaNs with payloads, signalling and sign-bit NaNs: every NaN ranks as one value
    x[::5] = np.array([0x7fc00001, 0xffc00000, 0x7f800001, 0xffffffff], np.uint32).view(np.float32)[
        np.arange(x[::5].size) % 4]
    ref = torch.sort(torch.from_numpy(x), descending=True, stable=True).indices.numpy()
    np.testing.assert_array_equal(O.stable_order_desc(x), ref)


def test_oracle_order_small_examples():
    x = np.array([0.5, np.nan, np.inf, 0.5, -np.nan, 1, 0], np.float32)
    np.testing.assert_array_equal(O.stable_order_desc(x), [1, 4, 2, 5, 0, 3, 6])
    np.testing.assert_array_equal(O.stable_order_desc(np.array([-0.0, 0.0, -0.0], np.float32)), [0, 1, 2])
