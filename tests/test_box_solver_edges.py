"""CPU: the decisions of the box solver stage at their edges, against tests/golden/box_solver_edges.npz (minted from
the reference's own box_estimator.py / kitti_utils.py by tests/golden/make_box_solver_edges_golden.py).

* the status rules of box_estimator.py:187 at threshold - ulp, at the threshold and at threshold + ulp, and on pairs
  whose exact difference lies below the threshold while the float32 difference the reference computes equals it;
* the score test of test_net.py:285 at float32(0.05);
* infer_boundary on nested, column-sharing, tied, multiply painted, doubly occluded, edge, fractional and degenerate
  boxes, and on 1 to 300 detections at widths 1, 1242 and 4094.

The product's rules are checked in the host-compiled box_solver_core.h, the code the device kernel runs.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import box_solver as BS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "box_solver_edges.npz"))


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("boxhost") / "libboxhost.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests/tools/box_solver_host.cpp")])
    return ctypes.CDLL(so)


def rule_cases(g):
    """indices of the cases decided by the rules alone (every case but the far one)"""
    return [i for i, n in enumerate(g["st_name"]) if str(n) != "far"]


def test_golden_covers_every_rule_edge(gold):
    g = gold
    names = [str(n) for n in g["st_name"]]
    for rule in ("kp", "w", "h"):
        for edge, st in (("below", 0), ("at", 1), ("above", 1)):
            assert int(g["st_status"][names.index("%s_%s" % (rule, edge))]) == st
        f32_pairs = [i for i, n in enumerate(names) if n.startswith(rule + "_f32_")]
        assert len(f32_pairs) >= 3
        col = {"kp": (None, 3, 4), "w": (0, 0, 2), "h": (0, 1, 3)}[rule]
        for i in f32_pairs:
            a, b = (g["st_kpts"][i][3], g["st_kpts"][i][4]) if rule == "kp" else \
                (g["st_box_left"][i][col[1]], g["st_box_left"][i][col[2]])
            thresh = 3.0 if rule == "kp" else 10.0
            assert float(b) - float(a) < thresh and np.float32(b - a) == np.float32(thresh)
            assert int(g["st_status"][i]) == 1          # the reference solves it
    assert int(g["st_status"][names.index("far")]) == 0


def test_oracle_status_vs_reference(gold):
    """the oracle's rules and solve give the reference's status on every case, the far one (z > 100) included"""
    g = gold
    shape = tuple(int(v) for v in g["im_shape"])
    for i, name in enumerate(g["st_name"]):
        alpha = float(np.arctan2(np.float64(g["st_sincos"][i][0]), np.float64(g["st_sincos"][i][1])))
        st, _ = BS.solve_x_y_z_theta_from_kpt(shape, g["p2"], g["p3"], alpha, g["st_dim"][i], g["st_box_left"][i],
                                              g["st_box_right"][i], g["st_kpts"][i])
        assert st == int(g["st_status"][i]), str(name)
        if str(name) != "far":
            assert BS.rejected(g["st_box_left"][i], g["st_kpts"][i]) == (int(g["st_status"][i]) == 0), str(name)


def test_product_status_rules_in_float32(gold, host_lib):
    """sb_box_rejected (box_solver_core.h) decides as the reference does, including where the float32 difference
    rounds up to the threshold; evaluated in double it would drop those detections"""
    g = gold
    host_lib.box_rejected_host.restype = ctypes.c_int
    fp = ctypes.POINTER(ctypes.c_float)
    wrong = []
    for i in rule_cases(g):
        box = np.ascontiguousarray(g["st_box_left"][i], np.float32)
        kp = np.ascontiguousarray(g["st_kpts"][i], np.float32)
        got = host_lib.box_rejected_host(box.ctypes.data_as(fp), kp.ctypes.data_as(fp))
        if bool(got) != (int(g["st_status"][i]) == 0):
            wrong.append(str(g["st_name"][i]))
    assert not wrong, "status differs from the reference for %s" % wrong


def test_score_threshold_is_float32(gold):
    """test_net.py:285 compares a float32 element with 0.05 in float32: float32(0.05) itself is not solved, the next
    float up is.  The kernel compares the float score with the float eval_thresh (ops.box_solve passes 0.05)."""
    g = gold
    got = g["score_values"].astype(np.float32) > np.float32(0.05)
    np.testing.assert_array_equal(got, g["score_pass"])
    assert list(g["score_pass"]) == [False, False, True]


def test_oracle_infer_boundary_vs_reference(gold):
    g = gold
    off = g["ib_offsets"]
    assert len(off) - 1 == len(g["ib_names"]) >= 25
    for p, name in enumerate(g["ib_names"]):
        b = g["ib_boxes"][off[p]:off[p + 1]]
        lr = BS.infer_boundary((375, int(g["ib_im_w"][p])), b)
        np.testing.assert_array_equal(lr, g["ib_left_right"][off[p]:off[p + 1]], err_msg=str(name))
