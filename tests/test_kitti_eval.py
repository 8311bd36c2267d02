"""CPU: the KITTI label / result parser, the oracle's BEV intersection against scipy's polygon areas, and the oracle's
restatement of the devkit's evaluate_object (DESIGN.md §9) on hand-built cases with their counts written out.  The
cases (CASES) are also run on the device by test_gpu_kitti_eval.py."""
import math
import os

import numpy as np
import pytest

from oracle import kitti_eval as O
from stereo_rcnn_b200 import kitti_eval as K

EASY, MOD, HARD = 0, 1, 2


def cfg(metric, d, bar=0, n_bars=2):
    return (metric * n_bars + bar) * 3 + d


# ------------------------------------------------------------------------------------------------ parser ----
LABEL = ("Car 0.00 0 -1.58 587.01 173.33 614.12 200.12 1.65 1.67 3.64 -0.65 1.71 46.70 -1.59\n"
         "DontCare -1 -1 -10 503.89 169.71 590.61 190.13 -1 -1 -1 -1000 -1000 -1000 -10\n")
RESULT = "Car -1 -1 -1.50 580.0 170.0 610.0 201.0 1.6 1.7 3.6 -0.6 1.7 46.0 -1.55 0.93\n"


def test_read_objects_label_and_result(tmp_path):
    types, rows = K.read_objects(LABEL)
    assert types == ["Car", "DontCare"] and rows.shape == (2, 15) and rows.dtype == np.float64
    assert rows[0, 3] == 587.01 and rows[1, 13] == -10.0 and np.isnan(rows[:, 14]).all()
    p = tmp_path / "000001.txt"
    p.write_text(RESULT)
    types, rows = K.read_objects(str(p))
    assert types == ["Car"] and rows[0, 14] == 0.93 and rows[0, 13] == -1.55
    assert K.read_objects("")[1].shape == (0, 15)
    codes, packed = K.pack_rows(*K.read_objects(LABEL + "Pedestrian" + RESULT[3:-6] + "\n"), False)
    assert codes.tolist() == [0, 2, 3] and packed.shape == (3, 16)
    assert packed[0, 13] == np.cos(-1.59) and packed[0, 14] == np.sin(-1.59) and packed[0, 15] == 0.0


@pytest.mark.parametrize("bad, what", [
    (LABEL + "Car 0 0 1 2 3\n", "line 3: 6 fields"),
    ("Car 0.00 0 -1.58 587.01 x 614.12 200.12 1.65 1.67 3.64 -0.65 1.71 46.70 -1.59\n", "line 1: a field"),
    ("Car 0.00 0 -1.58 587.01 nan 614.12 200.12 1.65 1.67 3.64 -0.65 1.71 46.70 -1.59\n", "line 1: a field is not"),
    (LABEL + RESULT, "line 3: 16 fields"),
])
def test_read_objects_refuses_malformed_lines(tmp_path, bad, what):
    p = tmp_path / "bad.txt"
    p.write_text(bad)
    with pytest.raises(ValueError, match=what) as e:
        K.read_objects(str(p))
    assert str(p) in str(e.value)
    with pytest.raises(ValueError, match="<text> " + what):
        K.read_objects(bad)


def test_evaluate_dirs_needs_every_label_file(tmp_path):
    with pytest.raises(FileNotFoundError, match="000007"):
        K.evaluate_dirs(str(tmp_path), str(tmp_path), ["000007"], "cpu")


def test_kitti_eval_refuses_bad_bars_and_unscored_results():
    with pytest.raises(ValueError):
        K.KittiEval("cpu", (0.7, 1.5))
    with pytest.raises(ValueError, match="no score"):
        K.KittiEval("cpu").add(LABEL, LABEL)


# ------------------------------------------------------------------------------------------- BEV geometry ----
def bev_row(x, z, l, w, ry):
    r = [0.0] * 16
    r[O.X], r[O.Z], r[O.L], r[O.W], r[O.COS], r[O.SIN] = x, z, l, w, math.cos(ry), math.sin(ry)
    return r


def scipy_area(a, b):
    """area of the intersection of two rectangles: the halfspaces of both, scipy's HalfspaceIntersection around the
    Chebyshev centre, ConvexHull of the vertices"""
    from scipy.optimize import linprog
    from scipy.spatial import ConvexHull, HalfspaceIntersection
    hs = []
    for r in (a, b):
        px, pz = O.bev_corners(r)
        for k in range(4):
            ex, ez = px[(k + 1) % 4] - px[k], pz[(k + 1) % 4] - pz[k]
            hs.append([ez, -ex, ex * pz[k] - ez * px[k]])
    hs = np.array(hs)
    norm = np.linalg.norm(hs[:, :2], axis=1)
    lp = linprog([0, 0, -1], A_ub=np.c_[hs[:, :2], norm], b_ub=-hs[:, 2], bounds=[(None, None)] * 2 + [(0, None)])
    if lp.x is None or lp.x[2] < 1e-9:                 # disjoint, or touching only
        return 0.0
    pts = HalfspaceIntersection(hs, lp.x[:2]).intersections
    return ConvexHull(pts).volume


def bev_pairs():
    rs = np.random.RandomState(5)
    pairs = []
    for _ in range(300):
        a = bev_row(rs.uniform(-2, 2), rs.uniform(-2, 2), rs.uniform(0.5, 5), rs.uniform(0.5, 3), rs.uniform(-4, 4))
        b = bev_row(rs.uniform(-2, 2), rs.uniform(-2, 2), rs.uniform(0.5, 5), rs.uniform(0.5, 3), rs.uniform(-4, 4))
        pairs.append((a, b))
    base = bev_row(1.0, 20.0, 4.0, 2.0, 0.3)
    c, s = math.cos(0.3), math.sin(0.3)
    pairs += [
        (base, base),                                                              # identical
        (base, bev_row(1.0 + 4.0 * c, 20.0 - 4.0 * s, 4.0, 2.0, 0.3)),              # sharing an edge
        (base, bev_row(1.0, 20.0, 2.0, 1.0, 1.1)),                                 # nested
        (bev_row(0, 0, 2, 2, 0), bev_row(2, 2, 2, 2, 0)),                          # touching at a corner
        (bev_row(0, 0, 2, 2, 0), bev_row(2, 2, 2, 2, math.pi / 4)),                # a corner inside
        (bev_row(0, 0, 2, 2, 0), bev_row(7, 1, 2, 2, 0.2)),                        # disjoint
        (bev_row(0, 0, 2, 2, 0), bev_row(2.5, 0, 2, 2, math.pi / 4)),              # disjoint, circles overlap
        (bev_row(0, 0, 4, 1, 0), bev_row(0, 0, 4, 1, math.pi / 2)),                # a cross
        (bev_row(0, 0, 4, 1, math.pi), bev_row(0, 0, 4, 1, -math.pi)),             # across +-pi
    ]
    return pairs


def test_bev_intersection_matches_scipy():
    for k, (a, b) in enumerate(bev_pairs()):
        got, ref = O.bev_intersection(a, b), scipy_area(a, b)
        assert abs(got - ref) <= 1e-9 * ref + 1e-12, (k, got, ref)
        assert abs(O.bev_intersection(b, a) - ref) <= 1e-9 * ref + 1e-12, k


def test_dontcare_rows_have_no_bev_overlap():
    d = bev_row(-1000.0, -1000.0, -1.0, -1.0, -10.0)
    assert O.bev_intersection(d, d) == pytest.approx(1.0)
    assert O.bev_intersection(bev_row(1.0, 20.0, 4.0, 2.0, 0.3), d) == 0.0


# ------------------------------------------------------------------------------------------ evaluate_object ----
def row(box, y=1.6, z=30.0, x=0.0, occ=0, trunc=0.0, alpha=0.0, score=0.0, h=1.5, w=1.6, l=3.9, ry=0.0):
    r = [0.0] * 16
    r[O.TRUNC], r[O.OCC], r[O.ALPHA] = trunc, occ, alpha
    r[O.X1], r[O.Y1], r[O.X2], r[O.Y2] = box
    r[O.H], r[O.W], r[O.L], r[O.X], r[O.Y], r[O.Z] = h, w, l, x, y, z
    r[O.COS], r[O.SIN], r[O.SCORE] = math.cos(ry), math.sin(ry), score
    return r


DONTCARE_ROW = row((200.0, 0.0, 300.0, 50.0), h=-1, w=-1, l=-1, x=-1000, y=-1000, z=-1000, ry=-10.0)


def image(gts=(), dets=()):
    """gts / dets: (code, row) -> the oracle's image tuple"""
    g = np.array([r for _c, r in gts], np.float64).reshape(-1, 16)
    d = np.array([r for _c, r in dets], np.float64).reshape(-1, 16)
    return g, np.array([c for c, _r in gts], np.int32), d, np.array([c for c, _r in dets], np.int32)


def anchor():
    """one easy Car matched exactly, far from everything else: every case has a threshold (its score, 0.5)"""
    r = row((800.0, 100.0, 900.0, 160.0), x=12.0, z=10.0)
    return image([(0, r)], [(0, _d(r, score=0.5))])


def with_anchor(*imgs):
    return [anchor()] + list(imgs)


def _d(r, **kw):
    r = list(r)
    for k, v in kw.items():
        r[getattr(O, k.upper())] = v
    return r


CAR60 = row((0.0, 0.0, 100.0, 60.0))
# name -> (images, bars, [(config, tp, fp, fn, n_thresholds)] at the last (lowest) threshold)
CASES = {
    "gt_height_40_ignored_at_easy": (
        with_anchor(image([(0, row((0.0, 0.0, 100.0, 40.0)))], [(0, _d(row((0.0, 0.0, 100.0, 40.0)), score=0.9))])),
        (0.7, 0.5), [(cfg(0, EASY), 1, 0, 0, 1), (cfg(0, MOD), 2, 0, 0, 2)]),
    "det_height_25_kept_at_moderate": (
        with_anchor(image([(0, row((0.0, 0.0, 100.0, 26.0)))], [(0, _d(row((0.0, 0.0, 100.0, 25.0)), score=0.9))])),
        (0.7, 0.5), [(cfg(0, EASY), 1, 0, 0, 1), (cfg(0, MOD), 2, 0, 0, 2)]),
    "truncation_015_is_easy": (
        with_anchor(image([(0, row((0.0, 0.0, 100.0, 60.0), trunc=0.15))], [(0, _d(CAR60, score=0.9))])),
        (0.7, 0.5), [(cfg(0, EASY), 2, 0, 0, 2)]),
    "occlusion_1_ignored_at_easy": (
        with_anchor(image([(0, row((0.0, 0.0, 100.0, 60.0), occ=1))], [(0, _d(CAR60, score=0.9))])),
        (0.7, 0.5), [(cfg(0, EASY), 1, 0, 0, 1), (cfg(0, MOD), 2, 0, 0, 2)]),
    "van_matched_is_not_a_false_positive": (
        with_anchor(image([(1, CAR60)], [(0, _d(CAR60, score=0.9))])),
        (0.7, 0.5), [(cfg(0, EASY), 1, 0, 0, 1), (cfg(1, MOD), 1, 0, 0, 1), (cfg(2, HARD), 1, 0, 0, 1)]),
    "unmatched_detection_is_a_false_positive": (
        with_anchor(image([], [(0, _d(CAR60, score=0.9))])),
        (0.7, 0.5), [(cfg(0, EASY), 1, 1, 0, 1)]),
    "short_detection_taken_in_pass_1": (
        with_anchor(image([(0, row((0.0, 0.0, 100.0, 30.0)))],
                          [(0, _d(row((0.0, 0.0, 100.0, 24.0)), score=0.9)), (0, _d(row((0.0, 0.0, 100.0, 30.0)), score=0.8))])),
        (0.7, 0.5), [(cfg(0, MOD), 2, 0, 0, 1)]),
    "false_positive_in_dontcare_2d_only": (
        with_anchor(image([(2, DONTCARE_ROW)], [(0, row((210.0, 5.0, 290.0, 45.0), x=-8.0, z=40.0, score=0.9))])),
        (0.7, 0.5), [(cfg(0, EASY), 1, 0, 0, 1), (cfg(1, EASY), 1, 1, 0, 1), (cfg(2, EASY), 1, 1, 0, 1)]),
    "iou_exactly_at_the_bar": (
        with_anchor(image([(0, row((0.0, 0.0, 100.0, 50.0)))], [(0, row((0.0, 0.0, 200.0, 50.0), score=0.9))])),
        (0.5,), [(cfg(0, EASY, 0, 1), 1, 1, 1, 1), (cfg(2, EASY, 0, 1), 2, 0, 0, 2)]),
    "score_and_overlap_ties_first_row_wins": (
        with_anchor(image([(0, _d(CAR60, alpha=0.4))], [(0, _d(CAR60, score=0.9, alpha=0.4)),
                                                         (0, _d(CAR60, score=0.9, alpha=0.4 + math.pi))])),
        (0.7, 0.5), [(cfg(0, EASY), 2, 1, 0, 2)]),
    "no_gt_in_the_split": (
        [image([], [(0, _d(CAR60, score=0.9))]), image([(2, DONTCARE_ROW)], [(0, _d(CAR60, score=0.7))])],
        (0.7, 0.5), [(cfg(0, EASY), 0, 0, 0, 0), (cfg(2, HARD), 0, 0, 0, 0)]),
    "images_without_gt_or_detections": (
        with_anchor(image([], [(0, _d(CAR60, score=0.9))]), image([(0, CAR60)], []), image([], [])),
        (0.7, 0.5), [(cfg(0, EASY), 1, 1, 1, 1), (cfg(2, MOD), 1, 1, 1, 1)]),
}


def test_iou_at_the_bar_is_exactly_half():
    assert O.overlap_2d(row((0.0, 0.0, 2.0, 1.0)), row((0.0, 0.0, 1.0, 1.0))) == 0.5


@pytest.mark.parametrize("name", sorted(CASES))
def test_hand_cases(name):
    images, bars, expect = CASES[name]
    r = O.evaluate(images, bars)
    for c, tp, fp, fn, nt in expect:
        t = max(int(r["n_thresholds"][c]) - 1, 0)
        got = (int(r["tp"][c, t]), int(r["fp"][c, t]), int(r["fn"][c, t]), int(r["n_thresholds"][c]))
        assert got == (tp, fp, fn, nt), (name, c, got)
    if name == "score_and_overlap_ties_first_row_wins":
        assert r["sim"][0, 0] == 1.0 and r["sim"][0, 1] == 2.0      # the first detection's alpha, not the second's
    if name == "no_gt_in_the_split":
        assert (r["ap"] == 0).all() and (r["n_gt"] == 0).all()


def exact_split(n):
    """n easy Cars, each matched exactly by one detection, with distinct scores"""
    imgs = []
    for k in range(n):
        r = row((0.0, 0.0, 100.0, 60.0), z=10.0 + k)
        imgs.append(image([(0, r)], [(0, _d(r, score=0.5 + k / 100.0))]))
    return imgs


def test_worked_cases():
    r = O.evaluate(exact_split(1))
    assert np.allclose(r["ap"][:, [0, 2]], 100.0 / 11.0, rtol=0, atol=1e-12) and (r["ap"][:, [1, 3]] == 0).all()
    r = O.evaluate(exact_split(41))
    assert (r["n_thresholds"] == 41).all() and np.allclose(r["ap"], 100.0, rtol=0, atol=1e-12)


def test_thresholds_rule():
    assert O.thresholds([], 0) == []
    assert len(O.thresholds(list(np.linspace(1, 0, 200)), 200)) == 41
    assert O.thresholds([0.9, 0.8], 100) == [0.9, 0.8]         # the last score is always taken


def test_package_and_oracle_pack_the_same_rows():
    """the parser and packer feed the oracle in the tests and the device in the product"""
    types, rows = K.read_objects(RESULT)
    codes, packed = K.pack_rows(types, rows, True)
    assert codes.tolist() == [0] and packed[0, O.SCORE] == 0.93 and packed[0, O.Y2] == 201.0
    assert os.path.basename(O.__file__) == "kitti_eval.py"
