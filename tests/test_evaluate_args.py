"""CPU: the test loop's host side and the argument checks of the device-calibrated entry points.

* ops.read_calibration gives P0-P3 and t_cam2_cam0_x bit for bit as the reference's read_obj_calibration
  (tests/golden/calibration.npz, minted by tests/golden/make_calibration_golden.py), from a path and from the text.
* sb_box_solve_devcalib, sb_box_rectify_devcalib and sb_dense_align_n_devcalib refuse, with SB_EINVAL and before any
  CUDA call, a null calibration and every argument their host-calibrated siblings refuse.
* pipeline.evaluate refuses a result directory that already holds result files before it reads any entry.
"""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import ops as G

SB_EINVAL = -22
FAKE = 1 << 20                                            # never dereferenced: every refusal precedes the first call
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(HERE, "golden", "calibration.npz")


@pytest.fixture(scope="module")
def lib():
    from stereo_rcnn_b200 import build
    build.build()
    return L.load()


def bits(a):
    return np.ascontiguousarray(a, np.float64).view(np.uint64)


@pytest.mark.parametrize("i", [0, 1, 2])
def test_read_calibration_matches_reference_reader(i, tmp_path):
    g = np.load(GOLD)
    text = str(g["texts"][i])
    path = tmp_path / ("%06d.txt" % i)
    path.write_text(text)
    for c in (G.read_calibration(text), G.read_calibration(str(path))):
        for k in ("p0", "p1", "p2", "p3"):
            got = getattr(c, k)
            assert got.shape == (3, 4) and got.dtype == np.float64
            np.testing.assert_array_equal(bits(got), bits(g[k][i]), err_msg=k)
        assert isinstance(c.t_cam2_cam0_x, float)
        assert bits(c.t_cam2_cam0_x) == bits(g["t_cam2_cam0_x"][i])


def test_read_calibration_goldens_differ_in_every_camera_constant():
    """the three calibrations the GPU tests use differ in f, cx, cy and baseline"""
    g = np.load(GOLD)
    p2, p3 = g["p2"], g["p3"]
    for v in (p2[:, 0, 0], p2[:, 0, 2], p2[:, 1, 2], p2[:, 0, 3] - p3[:, 0, 3]):
        assert len(set(v.tolist())) == 3


def test_read_calibration_rejects_malformed_text():
    g = np.load(GOLD)
    lines = str(g["texts"][0]).splitlines(True)
    with pytest.raises(ValueError):
        G.read_calibration("".join(lines[:3]))                       # no P3
    with pytest.raises(ValueError):
        G.read_calibration(lines[1] + lines[0] + "".join(lines[2:]))  # P1 before P0
    with pytest.raises(ValueError):
        G.read_calibration(lines[0].rsplit(" ", 1)[0] + "\n" + "".join(lines[1:]))   # 11 numbers


def test_device_calib_layout():
    """P2 then P3, row-major: what the _devcalib kernels index (calib4 = [0], [2], [6], [3] - [15])"""
    g = np.load(GOLD)
    c = np.concatenate([g["p2"][1].reshape(12), g["p3"][1].reshape(12)])
    np.testing.assert_array_equal(G.calib_vec(g["p2"][1], g["p3"][1]), [c[0], c[2], c[6], c[3] - c[15]])


def without_device(check):
    """run check(lib) in a child process that sees no CUDA device.  The calls pass fake device pointers; if a refusal
    regressed, the call would go on to a launch, which then fails with a CUDA error (and the test with it) instead of
    reading or writing those addresses on a real GPU."""
    code = ("import sys; sys.path[:0] = %r; from stereo_rcnn_b200 import lib as L; import test_evaluate_args as T; "
            "T.%s(L.load())" % ([ROOT, HERE], check))
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    args = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    r = subprocess.run(args, env=env, cwd=ROOT, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr


def test_box_solve_devcalib_rejections(lib):
    without_device("box_solve_rejections")


def test_box_rectify_devcalib_rejections(lib):
    without_device("box_rectify_rejections")


def test_dense_align_n_devcalib_rejections(lib):
    without_device("dense_align_rejections")


def _host_p():
    return (ctypes.c_double * 12)(*range(12))


def _refused_by_both(bad, sibling, devcalib, n0, lib):
    """every case refused by the sibling and by the _devcalib entry point, with no launch"""
    for k, args in bad.items():
        assert sibling(**args) == SB_EINVAL, ("host-calibrated sibling accepts", k)
        assert devcalib(**args) == SB_EINVAL, ("_devcalib accepts", k)
    assert lib.sb_launch_count() == n0


def box_solve_rejections(lib):
    names = ("scores", "boxes_left", "boxes_right", "dim_orien", "kpts", "keep", "num")
    outs = ("boxes_all", "kpts_all", "poses_all", "src_index", "n_out")

    def kw(nc=2, cls=1, cap=300, **null):
        a = {k: (None if k in null else FAKE) for k in names + ("inferred",) + outs}
        return dict(a, nc=nc, cls=cls, cap=cap)

    def sibling(nc, cls, cap, **p):
        return lib.sb_box_solve(*[p[k] for k in names], p["inferred"], nc, cls, 375, 1242, _host_p(), _host_p(), 0.05,
                                cap, *[p[k] for k in outs], None)

    def devcalib(nc, cls, cap, calib=FAKE, **p):
        return lib.sb_box_solve_devcalib(*[p[k] for k in names], p["inferred"], nc, cls, 375, 1242, calib, 0.05, cap,
                                         *[p[k] for k in outs], None)
    n0 = lib.sb_launch_count()
    bad = {"null " + k: kw(**{k: True}) for k in names + outs}
    bad.update({"cap 0": kw(cap=0), "cap < 0": kw(cap=-1), "cls < 0": kw(cls=-1), "cls = n_classes": kw(cls=2),
                "n_classes 0": kw(nc=0, cls=0)})
    _refused_by_both(bad, sibling, devcalib, n0, lib)
    assert devcalib(**kw(), calib=None) == SB_EINVAL
    assert lib.sb_box_solve(*[FAKE] * 8, 2, 1, 375, 1242, None, _host_p(), 0.05, 300, *[FAKE] * 5, None) == SB_EINVAL
    assert lib.sb_launch_count() == n0


def box_rectify_rejections(lib):
    names = ("boxes_all", "kpts_all", "poses_all", "succ", "best_dis", "n")

    def kw(cap=300, **null):
        a = {k: (None if k in null else FAKE) for k in names + ("final",)}
        return dict(a, cap=cap)

    def sibling(cap, final, **p):
        return lib.sb_box_rectify(*[p[k] for k in names], cap, 375, 1242, _host_p(), _host_p(), final, None)

    def devcalib(cap, final, calib=FAKE, **p):
        return lib.sb_box_rectify_devcalib(*[p[k] for k in names], cap, 375, 1242, calib, final, None)
    n0 = lib.sb_launch_count()
    bad = {"null " + k: kw(**{k: True}) for k in names + ("final",)}
    bad.update({"cap 0": kw(cap=0), "cap < 0": kw(cap=-5)})
    _refused_by_both(bad, sibling, devcalib, n0, lib)
    assert devcalib(**kw(), calib=None) == SB_EINVAL
    assert lib.sb_launch_count() == n0


def dense_align_rejections(lib):
    H, W = 375, 1242
    nb = lib.sb_dense_align_workspace_bytes(H, W, 40)

    def kw(H=H, W=W, box_ld=5, pose_ld=8, D=40, ws_bytes=nb, **null):
        a = {k: (None if k in null else FAKE) for k in ("iml", "imr", "ws", "n_dev")}
        return dict(a, H=H, W=W, box_ld=box_ld, pose_ld=pose_ld, D=D, ws_bytes=ws_bytes)

    def call(fn, c, iml, imr, ws, n_dev, H, W, box_ld, pose_ld, D, ws_bytes):
        return fn(iml, imr, H, W, c, 1.6, FAKE, box_ld, FAKE, FAKE, pose_ld, D, n_dev, FAKE, FAKE, ws, ws_bytes, None)

    def sibling(**a):
        return call(lib.sb_dense_align_n, (ctypes.c_double * 4)(721.5, 609.6, 172.9, 384.4), **a)

    def devcalib(calib=FAKE, **a):
        return call(lib.sb_dense_align_n_devcalib, calib, **a)
    n0 = lib.sb_launch_count()
    bad = {"null im_left": kw(iml=True), "null im_right": kw(imr=True), "null workspace": kw(ws=True),
           "null n_dev": kw(n_dev=True), "short workspace": kw(ws_bytes=nb - 1), "D_cap < 0": kw(D=-1),
           "H < 2": kw(H=1), "W < 2": kw(W=1), "box_ld < 4": kw(box_ld=3), "pose_ld < 7": kw(pose_ld=6),
           "short workspace, materialised": kw(D=49, ws_bytes=lib.sb_dense_align_workspace_bytes(H, W, 49) - 1)}
    _refused_by_both(bad, sibling, devcalib, n0, lib)
    assert devcalib(**kw(), calib=None) == SB_EINVAL
    assert devcalib(**kw(D=0), calib=None) == SB_EINVAL
    assert sibling(**kw(D=0)) == 0 and devcalib(**kw(D=0)) == 0           # D_cap 0: nothing to do, no launch
    assert lib.sb_dense_align_workspace_bytes(H, W, 40) == nb
    assert lib.sb_launch_count() == n0


def test_evaluate_refuses_a_directory_with_results(tmp_path):
    """no entry is read (the callbacks raise) and nothing is written when result_dir/data holds .txt files"""
    from stereo_rcnn_b200 import pipeline as PL
    data = tmp_path / "data"
    data.mkdir()
    (data / "000001.txt").write_text("Car -1 -1 0 0 0 0 0 0 0 0 0 0 0 0 1\n")

    def boom(entry):
        raise AssertionError("an entry was read")
    with pytest.raises(FileExistsError):
        PL.evaluate(None, [{"image_id": "000000"}], boom, boom, str(tmp_path))
    assert sorted(os.listdir(data)) == ["000001.txt"]
