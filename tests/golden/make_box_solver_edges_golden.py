"""Mint tests/golden/box_solver_edges.npz from the REFERENCE's own solver code (run in the build container only).

    python tests/golden/make_box_solver_edges_golden.py

box_estimator.py and kitti_utils.py are executed from where they lie, with the runtime patches of make_golden.py (10)
(py2 implicit import, `scipy.array` removed from scipy); nothing is copied.  Two groups of cases:

* status decisions of `solve_x_y_z_theta_from_kpt`, called exactly as test_net.py:287-295 calls it: `box_left` and
  `box_right` float32 numpy rows, `kpts` a float32 torch row, `alpha = math.atan2` of two float32 elements.  Each of
  the three rejection rules of box_estimator.py:187 sits at threshold - ulp, at the threshold and at threshold + ulp,
  plus pairs where the float32 difference rounds up to the threshold while the exact difference lies below it (found
  by the search below).  Only the status is stored: end points are compared by stationarity, not digit by digit
  (tests/test_box_solver.py explains why).  Also stored: the score test of test_net.py:285 at float32(0.05) and one
  float up, and a far detection that the reference drops by its `z > 100` rule.
* `infer_boundary` on hand-built occlusion patterns.  The reference ran it under numpy 1.x, where `1050.0 / x` of a
  float32 numpy scalar is a float64; numpy 2 (NEP 50) would compute it in float32.  The boxes are therefore passed as
  float64 arrays holding float32 values, which is the numpy 1.x arithmetic (and the product's).
"""
import math as m
import os
import sys
import types

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", ".."))

from oracle import ref_shim  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
f32 = np.float32
IM_SHAPE = (375, 1242, 3)


def load_reference():
    src = open(os.path.join(ref_shim.REF, "lib/model/utils/box_estimator.py")).read()
    src = src.replace("import kitti_utils as utils", "utils = None").replace("scipy.array", "np.array")
    be = types.ModuleType("box_estimator")
    exec(compile(src, "box_estimator.py", "exec"), be.__dict__)
    try:
        import cv2  # noqa: F401
    except ImportError:                                   # kitti_utils imports cv2; infer_boundary does not use it
        sys.modules["cv2"] = types.ModuleType("cv2")
    ku = types.ModuleType("kitti_utils")
    exec(compile(open(os.path.join(ref_shim.REF, "lib/model/utils/kitti_utils.py")).read(), "kitti_utils.py", "exec"),
         ku.__dict__)
    return be, ku


def project(p2, p3, x, y, z, w, h, l, th, kt):
    """a 3D box (bottom centre x, y, z; w, h, l; yaw th) -> float32 box_left, box_right, kpts [u, kt, 0.9, x1, x2],
    (sin, cos) of its viewpoint angle"""
    c, s = np.cos(th), np.sin(th)
    xs = np.array([-w / 2, -w / 2, w / 2, w / 2] * 2)
    ys = np.array([0, 0, 0, 0, -h, -h, -h, -h])
    zs = np.array([-l / 2, l / 2, l / 2, -l / 2] * 2)
    X, Y, Z = c * xs + s * zs + x, ys + y, -s * xs + c * zs + z
    u, v = p2[0, 0] * X / Z + p2[0, 2], p2[1, 1] * Y / Z + p2[1, 2]
    d = (p2[0, 3] - p3[0, 3]) / Z
    box_l = np.array([u.min(), v.min(), u.max(), v.max()])
    box_r = np.array([(u - d).min(), v.min(), (u - d).max(), v.max()])
    vw, vl = [(-w, -l), (-w, l), (w, l), (w, -l)][kt]
    Xk, Zk = x + c * vw / 2 + s * vl / 2, z - s * vw / 2 + c * vl / 2
    kp = np.array([p2[0, 0] * Xk / Zk + p2[0, 2], kt, 0.9, box_l[0], box_l[2]])
    alpha = th - m.pi / 2 + m.atan2(-x, z)
    return box_l.astype(f32), box_r.astype(f32), kp.astype(f32), np.array([np.sin(alpha), np.cos(alpha)], f32)


def disagreement_pairs(thresh, lo_range, count, seed):
    """float32 (a, b) with a in lo_range, b - a < thresh exactly, float32(b - a) == thresh"""
    rs = np.random.RandomState(seed)
    out = []
    while len(out) < count:
        a = f32(rs.uniform(*lo_range))
        b = f32(float(a) + thresh)
        while float(b) - float(a) >= thresh:
            b = np.nextafter(b, f32(-np.inf))
        if f32(b - a) == f32(thresh) and float(b) - float(a) < thresh:
            out.append((a, b))
    return out


def status_cases(be, p2, p3):
    """-> list of (name, box_left, box_right, kpts, sin_cos, dim, score)"""
    cases = []
    up, down = lambda v: np.nextafter(f32(v), f32(np.inf)), lambda v: np.nextafter(f32(v), f32(-np.inf))

    def add(name, geo, edit=None, score=0.9):
        box_l, box_r, kp, sc = project(p2, p3, *geo)
        if edit:
            edit(box_l, box_r, kp)
        cases.append((name, box_l, box_r, kp, sc, np.array(geo[3:6], f32), f32(score)))
    # keypoint borders: kpts[4] - kpts[3] vs 3 (the borders only enter the rule, any box will do)
    car = (1.0, 1.65, 18.0, 1.6, 1.5, 3.9, 0.6, 1)

    def kp_edit(k3, k4):
        def e(bl, br, kp):
            kp[3], kp[4] = k3, k4
        return e
    for name, k4 in (("kp_below", down(103.0)), ("kp_at", f32(103.0)), ("kp_above", up(103.0))):
        add(name, car, kp_edit(f32(100.0), k4))
    for j, (a, b) in enumerate(disagreement_pairs(3.0, (1.0, 2.0), 3, 1)):
        add("kp_f32_%d" % j, car, kp_edit(a, b))

    # box width x2 - x1 vs 10: a narrow object, at u ~ 100 and at the left edge (x1 < 4, so truncated there)
    def w_edit(x1, x2):
        def e(bl, br, kp):
            d = bl[0] - br[0]
            bl[0], bl[2] = x1, x2
            br[0], br[2] = f32(x1 - d), f32(x2 - d)
            kp[0] = f32((float(x1) + float(x2)) / 2)
        return e
    narrow = (-12.05, 1.65, 17.0, 0.2, 1.5, 0.2, 0.3, 2)
    for name, x2 in (("w_below", down(110.0)), ("w_at", f32(110.0)), ("w_above", up(110.0))):
        add(name, narrow, w_edit(f32(100.0), x2))
    edge = (-13.9, 1.65, 17.0, 0.2, 1.5, 0.2, 0.3, 2)
    for j, (a, b) in enumerate(disagreement_pairs(10.0, (2.0, 4.0), 3, 2)):
        add("w_f32_%d" % j, edge, w_edit(a, b))

    # box height y2 - y1 vs 10: a low object, at v ~ 100 and at the top edge (y1 < 4)
    def h_edit(y1, y2):
        def e(bl, br, kp):
            bl[1], bl[3] = y1, y2
            br[1], br[3] = y1, y2
        return e
    low = (1.0, -0.51, 20.0, 1.2, 0.28, 1.2, 0.6, 1)
    for name, y2 in (("h_below", down(110.0)), ("h_at", f32(110.0)), ("h_above", up(110.0))):
        add(name, low, h_edit(f32(100.0), y2))
    top = (1.0, -4.47, 20.0, 1.2, 0.28, 1.2, 0.6, 1)
    for j, (a, b) in enumerate(disagreement_pairs(10.0, (2.0, 4.0), 3, 3)):
        add("h_f32_%d" % j, top, h_edit(a, b))

    # far: the box implies z ~ 200 m (large dims, 1 px disparity); the reference drops it by `res.x[2] > 100`
    def far_edit(bl, br, kp):
        br[0], br[2] = bl[0] - f32(1.0), bl[2] - f32(1.0)
    add("far", (2.0, 1.65, 200.0, 3.0, 3.0, 8.0, 0.6, 1), far_edit)
    return cases


def solve_status(be, p2, p3, case):
    """the call of test_net.py:287-295 on one detection.  With today's scipy, an objective that returns a 0-d torch
    tensor (the keypoint is a torch element) fails inside `minimize`, so a detection that passes the rules raises
    there; its status then comes from a second call with the same float32 values as a numpy row (the rules see the
    same float32 differences)."""
    name, box_l, box_r, kp, sc, dim, score = case
    calib = types.SimpleNamespace(p2=p2, p3=p3)
    sin_alpha, cos_alpha = torch.tensor(sc[0]), torch.tensor(sc[1])
    alpha = m.atan2(sin_alpha, cos_alpha)
    args = (IM_SHAPE, calib, alpha, dim.copy(), box_l.copy(), box_r.copy())
    try:
        status, state = be.solve_x_y_z_theta_from_kpt(*args, torch.from_numpy(kp.copy()))
        return int(status), (None if np.isscalar(state) else np.asarray(state, np.float64))
    except AttributeError:          # past the rules, in scipy (a truncated box has no keypoint term and runs through)
        pass
    status, state = be.solve_x_y_z_theta_from_kpt(*args, kp.copy())
    return int(status), np.asarray(state, np.float64)


def ib_patterns():
    """(name, im_w, boxes [n,4] float32) in kept order"""
    rs = np.random.RandomState(9)
    B = lambda rows: np.array(rows, f32).reshape(-1, 4)
    pats = [
        ("nested_near_first", 1242, B([[100, 50, 400, 300], [200, 80, 300, 200]])),
        ("nested_far_first", 1242, B([[200, 80, 300, 200], [100, 50, 400, 300]])),
        ("shared_column", 1242, B([[100, 60, 200, 250], [200, 70, 300, 180], [200.5, 90, 260, 150]])),
        ("shared_column_frac", 1242, B([[100, 60, 200.9, 180], [200.2, 70, 300, 250]])),
        ("equal_bottoms", 1242, B([[100, 50, 300, 250], [200, 60, 400, 250], [250, 70, 500, 250]])),
        ("three_paint_desc", 1242, B([[100, 10, 300, 300], [150, 10, 320, 250], [180, 10, 340, 200], [190, 10, 360, 150]])),
        ("three_paint_asc", 1242, B([[190, 10, 360, 150], [180, 10, 340, 200], [150, 10, 320, 250], [100, 10, 300, 300]])),
        ("three_paint_mixed", 1242, B([[180, 10, 340, 200], [100, 10, 300, 300], [190, 10, 360, 150], [150, 10, 320, 250]])),
        ("both_ends_occluded", 1242, B([[150, 40, 220, 300], [280, 40, 350, 300], [200, 60, 300, 150]])),
        ("both_ends_far_first", 1242, B([[200, 60, 300, 150], [150, 40, 220, 300], [280, 40, 350, 300]])),
        ("im_w_edges", 1242, B([[0, 30, 50, 200], [1200, 30, 1242, 220], [0, 40, 1242, 120], [1241.5, 10, 1242, 300]])),
        ("fractional", 1242, B([[100.7, 20, 200.3, 180], [200.9, 30, 250.99, 220], [150.5, 25, 201.0, 160],
                                [99.999, 10, 100.001, 370]])),
        ("degenerate", 1242, B([[300, 40, 250, 200], [260, 30, 400, 180], [280, 50, 279.5, 300]])),
    ]
    for n, w in ((1, 1242), (2, 1242), (100, 1242), (300, 1242), (1, 1), (2, 1), (100, 1), (300, 1), (1, 4094),
                 (2, 4094), (100, 4094), (300, 4094)):
        q = lambda v: np.round(v * 8) / 8                    # eighths of a pixel: fractional, and the file stays small
        x1 = q(rs.rand(n) * w)
        x2 = np.minimum(x1 + q(rs.rand(n) * min(w, 400)), w)
        y1 = np.floor(rs.rand(n) * 300)
        y2 = y1 + 5 + np.floor(rs.rand(n) * 8) * 10          # few distinct bottoms: depth ties occur
        pats.append(("rand_%d_w%d" % (n, w), w, np.stack([x1, y1, x2, y2], 1).astype(f32)))
    return pats


def main():
    be, ku = load_reference()
    cal = np.load(os.path.join(HERE, "calibration.npz"))
    p2, p3 = cal["p2"][0], cal["p3"][0]
    out = {"p2": p2, "p3": p3, "im_shape": np.array(IM_SHAPE)}
    cases = status_cases(be, p2, p3)
    st = []
    for c in cases:
        s, state = solve_status(be, p2, p3, c)
        bl, kp = c[1], c[3]
        f32_rule = bool(kp[4] - kp[3] < 3 or bl[2] - bl[0] < 10 or bl[3] - bl[1] < 10)
        f64_rule = (float(kp[4]) - float(kp[3]) < 3 or float(bl[2]) - float(bl[0]) < 10 or
                    float(bl[3]) - float(bl[1]) < 10)
        z = "-" if state is None else "%.2f" % state[2]
        print("%-12s status %d  float32 rule %s  float64 rule %s  z %s" % (c[0], s, f32_rule, f64_rule, z))
        if c[0] == "far":
            assert s == 0 and not f32_rule and state[2] > 100
        else:       # each case is decided by the rule alone: a solved detection is a near one
            assert s == (0 if f32_rule else 1), c[0]
        st.append(s)
    for k, j in (("st_name", 0), ("st_box_left", 1), ("st_box_right", 2), ("st_kpts", 3), ("st_sincos", 4),
                 ("st_dim", 5), ("st_score", 6)):
        out[k] = np.array([c[j] for c in cases])
    out["st_status"] = np.array(st, np.int32)
    # test_net.py:285, `cls_dets_left[detect_idx, -1] > eval_thresh` on a float32 tensor element
    sc = np.array([np.nextafter(f32(0.05), f32(0)), f32(0.05), np.nextafter(f32(0.05), f32(1))], f32)
    out["score_values"] = sc
    out["score_pass"] = np.array([bool(torch.from_numpy(sc)[i] > 0.05) for i in range(3)])
    print("score > 0.05:", out["score_pass"])
    # infer_boundary
    pats = ib_patterns()
    boxes, lr, off, imw, names = [], [], [0], [], []
    n_f32 = 0
    for name, w, b in pats:
        ref = ku.infer_boundary((375, w, 3), b.astype(np.float64))
        n_f32 += not np.array_equal(ref, ku.infer_boundary((375, w, 3), b))
        boxes.append(b)
        lr.append(ref)
        off.append(off[-1] + len(b))
        imw.append(w)
        names.append(name)
    print("infer_boundary: %d patterns, %d boxes; %d would differ with numpy 2's float32 depth"
          % (len(pats), off[-1], n_f32))
    out.update(ib_boxes=np.concatenate(boxes), ib_left_right=np.concatenate(lr).astype(f32),
               ib_offsets=np.array(off, np.int32), ib_im_w=np.array(imw, np.int32), ib_names=np.array(names))
    np.savez_compressed(os.path.join(HERE, "box_solver_edges.npz"), **out)
    print("wrote box_solver_edges.npz")


if __name__ == "__main__":
    main()
