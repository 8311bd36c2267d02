"""CPU: sb_kitti_eval and sb_kitti_overlaps refuse every argument the header rules out with SB_EINVAL before any
launch (null pointers, n_images < 1, negative or too large sizes, n_bars outside 1..4, bars outside [0, 1], a workspace
that is too small or misaligned), and sb_kitti_eval_workspace_bytes is 0 exactly for the sizes sb_kitti_eval refuses."""
import ctypes

import pytest

from stereo_rcnn_b200 import lib as L

SB_EINVAL = -22
FAKE = 1 << 20                                            # never dereferenced: every refusal precedes the first call
BIG = 1 << 40                                             # the first row or pair count refused
OUTPUTS = ("thresholds", "n_thresholds", "tp", "fp", "fn", "sim", "precision", "recall", "aos", "ap", "n_gt")


@pytest.fixture(scope="module")
def lib():
    from stereo_rcnn_b200 import build
    build.build()
    return L.load()


def _eval(lib, n_images=3, n_gt_rows=5, n_det_rows=7, n_pairs=11, bars=(0.7, 0.5), n_bars=None, ws=FAKE,
          ws_bytes=None, null=()):
    p = {k: (None if k in null else FAKE + 256 * i) for i, k in
         enumerate(("gt", "gt_code", "det", "det_code", "gt_off", "det_off", "pair_off") + OUTPUTS)}
    n_bars = len(bars) if n_bars is None else n_bars
    b = (ctypes.c_double * max(len(bars), 1))(*bars) if "bars" not in null else None
    if ws_bytes is None:
        ws_bytes = lib.sb_kitti_eval_workspace_bytes(max(n_images, 1), max(n_gt_rows, 0) % BIG, max(n_det_rows, 0) % BIG,
                                                     max(n_pairs, 0) % BIG, min(max(n_bars, 1), 4))
    return lib.sb_kitti_eval(p["gt"], p["gt_code"], p["det"], p["det_code"], p["gt_off"], p["det_off"], p["pair_off"],
                             n_images, n_gt_rows, n_det_rows, n_pairs, b, n_bars, None if "workspace" in null else ws,
                             ws_bytes, *[p[k] for k in OUTPUTS], None)


def test_kitti_eval_rejections(lib):
    n0 = lib.sb_launch_count()
    need = lib.sb_kitti_eval_workspace_bytes(3, 5, 7, 11, 2)
    assert need > 0 and need % 256 == 0
    nan, inf = float("nan"), float("inf")
    bad = {"null " + k: _eval(lib, null=(k,)) for k in ("gt_off", "det_off", "pair_off", "bars", "workspace") + OUTPUTS}
    bad.update({"null gt with gt rows": _eval(lib, null=("gt",)), "null gt_code": _eval(lib, null=("gt_code",)),
                "null det with det rows": _eval(lib, null=("det",)), "null det_code": _eval(lib, null=("det_code",)),
                "n_images 0": _eval(lib, n_images=0), "n_images -1": _eval(lib, n_images=-1),
                "n_gt_rows -1": _eval(lib, n_gt_rows=-1), "n_det_rows -1": _eval(lib, n_det_rows=-1),
                "n_pairs -1": _eval(lib, n_pairs=-1), "n_gt_rows 2^40": _eval(lib, n_gt_rows=BIG),
                "n_det_rows 2^40": _eval(lib, n_det_rows=BIG), "n_pairs 2^40": _eval(lib, n_pairs=BIG),
                "n_bars 0": _eval(lib, n_bars=0), "n_bars 5": _eval(lib, bars=(0.1, 0.2, 0.3, 0.4, 0.5)),
                "n_bars -1": _eval(lib, n_bars=-1), "bar < 0": _eval(lib, bars=(0.7, -1e-300)),
                "bar > 1": _eval(lib, bars=(float.fromhex("0x1.0000000000001p+0"),)),
                "bar nan": _eval(lib, bars=(0.5, nan)), "bar inf": _eval(lib, bars=(inf,)),
                "bar -inf": _eval(lib, bars=(-inf, 0.5)),
                "workspace one byte short": _eval(lib, ws_bytes=need - 1), "workspace empty": _eval(lib, ws_bytes=0),
                "workspace misaligned": _eval(lib, ws=FAKE + 128, ws_bytes=need + 256),
                "workspace off by 8": _eval(lib, ws=FAKE + 8, ws_bytes=need + 256)})
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}


def test_kitti_overlaps_rejections(lib):
    n0 = lib.sb_launch_count()

    def ov(n_images=2, n_pairs=6, null=()):
        p = [None if k in null else FAKE + 256 * i for i, k in
             enumerate(("gt", "gt_code", "det", "gt_off", "det_off", "pair_off", "ov_2d", "ov_bev", "ov_3d"))]
        return lib.sb_kitti_overlaps(*p[:6], n_images, n_pairs, *p[6:], None)
    bad = {"null " + k: ov(null=(k,)) for k in ("gt", "gt_code", "det", "gt_off", "det_off", "pair_off", "ov_2d",
                                                "ov_bev", "ov_3d")}
    bad.update({"n_images 0": ov(n_images=0), "n_images -3": ov(n_images=-3), "n_pairs -1": ov(n_pairs=-1),
                "n_pairs 2^40": ov(n_pairs=BIG), "no pairs, null offsets": ov(n_pairs=0, null=("pair_off",))})
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}
    # no pairs: nothing to launch, and the rows and outputs may be null
    assert ov(n_pairs=0, null=("gt", "gt_code", "det", "ov_2d", "ov_bev", "ov_3d")) == 0
    assert lib.sb_launch_count() == n0


def test_workspace_bytes_zero_exactly_where_refused(lib):
    w = lib.sb_kitti_eval_workspace_bytes
    refused = {"n_bars 0": w(3, 5, 7, 11, 0), "n_bars 5": w(3, 5, 7, 11, 5), "n_bars -1": w(3, 5, 7, 11, -1),
               "n_images 0": w(0, 5, 7, 11, 2), "n_images -1": w(-1, 5, 7, 11, 2),
               "n_gt_rows 2^40": w(3, BIG, 7, 11, 2), "n_det_rows 2^40": w(3, 5, BIG, 11, 2),
               "n_pairs 2^40": w(3, 5, 7, BIG, 2), "n_gt_rows -1": w(3, -1, 7, 11, 2),
               "n_det_rows -1": w(3, 5, -1, 11, 2), "n_pairs -1": w(3, 5, 7, -1, 2)}
    assert all(v == 0 for v in refused.values()), {k: v for k, v in refused.items() if v}
    accepted = [w(1, 0, 0, 0, 1), w(1, 0, 0, 0, 4), w(3769, 30171, 109357, 875335, 2), w(1, BIG - 1, 0, 0, 1),
                w(1, 0, BIG - 1, 0, 4), w(1, 0, 0, BIG - 1, 1), w(1 << 30, 0, 0, 0, 1)]
    assert all(v > 0 and v % 256 == 0 for v in accepted), accepted
    # it grows with every size it covers (by more than its 256-byte rounding)
    base = w(10, 20, 30, 40, 2)
    assert all(v > base for v in (w(74, 20, 30, 40, 2), w(10, 84, 30, 40, 2), w(10, 20, 94, 40, 2),
                                  w(10, 20, 30, 104, 2), w(10, 20, 30, 40, 3)))


def test_kitti_eval_wrapper_refuses_before_the_device(lib):
    """ops.kitti_eval turns a refused size into a ValueError before it allocates anything; KittiEval refuses bars"""
    import torch
    from stereo_rcnn_b200 import kitti_eval as K
    from stereo_rcnn_b200 import ops as G
    off = torch.zeros(2, dtype=torch.int64)
    rows, codes = torch.zeros(0, 16, dtype=torch.float64), torch.zeros(0, dtype=torch.int32)
    with pytest.raises(ValueError, match="refuses"):
        G.kitti_eval(rows, codes, rows, codes, off, off, off, 0, (0.1, 0.2, 0.3, 0.4, 0.5))
    with pytest.raises(ValueError, match="refuses"):
        G.kitti_eval(rows, codes, rows, codes, off[:1], off[:1], off[:1], 0, (0.5,))
    for bars in ((), (0.1, 0.2, 0.3, 0.4, 0.5), (-0.1,), (1.0 + 2 ** -52,), (float("nan"),)):
        with pytest.raises(ValueError):
            K.KittiEval("cpu", bars)
