"""Mint tests/golden/kitti_annotations.npz from the REFERENCE's own roidb code (run in the build container only).

    python tests/golden/make_kitti_annotations_golden.py

kitti_utils.read_obj_data, kitti.remove_occluded_keypoints / _load_kitti_annotation, imdb.append_flipped_images and
roidb.filter_roidb are executed from where they lie through oracle/ref_shim.py (nothing copied).  Runtime shims only:
`cv2.imread` becomes a lookup of the image shape, `cPickle` a stub module, `from datasets.factory import get_imdb` a
stub (filter_roidb does not use it), and the imdb is built without reading a split file.

Two kinds of case, written as a KITTI folder of label and calibration texts with PNG headers:
  * exact cases: ry = -pi/2 written as repr(), so the orientation is exactly 0, with dyadic calibration, dimensions and
    positions; every product and sum is exact, so every summation order (the reference's BLAS included) gives the
    same bits.  The boundary cases are built this way.
  * seeded cases: KITTI-like calibrations and objects.  The reference's BLAS products may round differently from the
    oracle's sequential order, so the maker records the smallest distance of a box edge to an integer (the int()
    decisions) and of a keypoint to its pruning bars (min_margin, in pixels), and refuses a seed where it is below 1e-6.
Stored: the texts, the image sizes, the reference's kept rows in sb_kitti_annotations' layout, its statuses (1 + the
object index of an IndexError, counted over the used lines), and the flip + filter of the non-raising entries.
"""
import math
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", ".."))
sys.path.insert(0, HERE)

from oracle import ref_shim  # noqa: E402
from make_calibration_golden import kitti_text  # noqa: E402

RY0 = repr(-math.pi / 2)                      # m.pi/2 + RY0 == 0.0 exactly
PNG_SIG = b"\x89PNG\r\n\x1a\n"


def png_header(h, w):
    return PNG_SIG + b"\x00\x00\x00\rIHDR" + w.to_bytes(4, "big") + h.to_bytes(4, "big") + b"\x08\x02\x00\x00\x00"


# ------------------------------------------------------------------------------------------------------ exact cases
# P2 = [[512, 0, 640, 32], [0, 512, 192, 0], [0, 0, 1, 0]], P3[0,3] = -256, P0[0,3] = 0: t = 1/16, and a corner at a
# dyadic depth z projects to u = (512 x + 640 z) / z on the left: one rounding, in any order
EXACT_CALIB = kitti_text(512.0, 640.0, 192.0, (0.0, 0.0, 0.0), (-256.0, 0.0, 0.0), (32.0, 0.0, 0.0),
                         (-256.0, 0.0, 0.0))
T = 1.0 / 16.0


def line(typ, x, y, z, w, h, l, trunc=0.0, occ=0, alpha=0.25, ry=RY0):
    return "%s %s %d %s 0.00 0.00 0.00 0.00 %s %s %s %s %s %s %s" % (
        typ, repr(float(trunc)), occ, repr(float(alpha)), repr(float(h)), repr(float(w)), repr(float(l)),
        repr(float(x)), repr(float(y)), repr(float(z)), ry)


def car(u1, u2, zn, typ="Car", y=1.5, h=1.5, **kw):
    """an object 1 m long whose left box spans exactly u1 .. u2 before clamping, its near corners at depth zn"""
    zf = zn + 1.0
    a = (u1 - 640.0) * (zn if u1 < 640 else zf) / 512.0
    b = (u2 - 640.0) * (zf if u2 < 640 else zn) / 512.0
    assert a <= b, (u1, u2)
    return line(typ, (a + b) / 2.0 - T, y, (zn + zf) / 2.0, b - a, h, zf - zn, **kw)


def box(a, b, zn, zf, typ="Car", y=1.5, h=1.5, **kw):
    """an object whose corners lie at x = a and b (camera 2) and depths zn and zf"""
    return line(typ, (a + b) / 2.0 - T, y, (zn + zf) / 2.0, b - a, h, zf - zn, **kw)


# a kept keypoint exactly on each pruning bar of each camera (the comparisons are strict).  With corners at depths 16
# and 32 a corner projects to u = 640 + 32 x (near) / 640 + 16 x (far) on the left and to 622 + 32 x / 631 + 16 x on
# the right; the middle keypoint of three sits 3 px from the extreme one, or 5 px past the column where a nearer Van
# (depths 8 and 16: 640 + 64 x / 640 + 32 x on the left, 604 + 64 x / 622 + 32 x on the right) starts or ends
KEYPOINT_BARS = (
    ("kp_left_lk3", [box(3 / 16, 1.0, 16, 32)]),                                    # 646 = 643 + 3
    ("kp_right_lk3", [box(3 / 4, 2.0, 16, 32)]),                                    # 646 = 643 + 3
    ("kp_left_rk3", [box(-1.0, -3 / 16, 16, 32)]),                                  # 634 = 637 - 3
    ("kp_right_rk3", [box(-1.0, 3 / 8, 16, 32)]),                                   # 634 = 637 - 3
    ("kp_left_vl5", [box(-0.625, 0.2109375, 8, 16, "Van"), box(1 / 4, 2.0, 16, 32)]),        # 648 = 653 - 5
    ("kp_left_vr5", [box(-0.1796875, 0.625, 8, 16, "Van"), box(-2.0, -1 / 4, 16, 32)]),      # 632 = 627 + 5
    ("kp_right_vl5", [box(-1 / 16, 0.8046875, 8, 16, "Van"), box(7 / 8, 2.0, 16, 32)]),      # 650 = 655 - 5
    ("kp_right_vr5", [box(0.2890625, 1.1875, 8, 16, "Van"), box(-1.0, 1 / 8, 16, 32)]),      # 626 = 621 + 5
)


def exact_cases():
    c = []
    add = lambda name, lines, hw=(375, 1242): c.append((name, "".join(l + "\n" for l in lines), EXACT_CALIB, hw))
    add("tie", [car(300, 400, 16), car(300, 400, 16)])
    add("chain_far_first", [car(200, 420, 64), car(300, 520, 32), car(400, 620, 16)])
    add("chain_near_first", [car(400, 620, 16), car(300, 520, 32), car(200, 420, 64)])
    add("one_end_hidden", [car(500, 700, 16), car(600, 900, 32)])
    add("both_hidden", [car(500, 900, 16), car(600, 800, 32)])
    add("edges_0_w1", [car(-100, 150, 16), car(1100, 1400, 16)])
    add("edge_1259", [car(1100, 1400, 16)], (375, 1260))
    add("integer_x", [car(100, 300, 16), car(700.0 - 2.0 ** -10, 900.0 - 2.0 ** -10, 16)])
    add("height_10", [car(100, 300, 16, y=0.3125, h=0.3125), car(500, 700, 16, y=10.03125 / 32, h=10.03125 / 32)])
    for u1 in (638.0, 637.5, 637.0):                          # visible widths 3, 3.5 and 4 (a narrow box straddles cx)
        add("visible_%s" % (641.0 - u1), [car(u1, 641.0, 16)])
    add("occ_trunc", [car(100, 300, 16, occ=3), car(400, 600, 16, trunc=0.98), car(700, 900, 16, occ=2,
                                                                                          trunc=0.96875)])
    add("behind_corners", [line("Car", 0.5, 1.5, 4.0, 2.0, 1.5, 16.0), line("Car", -60.0, 1.5, 24.0, 4.0, 1.5, 16.0)])
    add("van_hides_car", [car(300, 700, 16, typ="Van"), car(400, 600, 32),
                          car(800, 1000, 32), line("DontCare", -1000, -1000, -1000, -1, -1, -1, trunc=-1, occ=-1,
                                                       alpha=-10, ry="-10"),
                          "Pedestrian 0.00 0 0.25 0 0 0 0 1.75 0.5 0.75 %s 1.5 8.0 %s" % (repr(200.0 / 32 - T), RY0)])
    add("past_1259", [car(1100, 1300, 16)], (375, 1392))
    add("behind_camera", [car(100, 300, 16), line("Car", 0.0, 1.5, -10.0, 2.0, 1.5, 4.0)])
    add("behind_then_past", [line("Car", 0.0, 1.5, -10.0, 2.0, 1.5, 4.0), car(1100, 1300, 16)], (375, 1392))
    add("no_used", [line("Pedestrian", 0.0, 1.5, 16.0, 0.5, 1.75, 0.75), line("DontCare", 0, 0, 0, 0, 0, 0)])
    add("none_kept", [car(100, 300, 16, typ="Van"), car(400, 600, 16, typ="Truck"),
                      car(700, 900, 16, typ="Misc")])
    add("empty", [])
    add("wholly_right_after_behind", [line("Car", 0.0, 1.5, -10.0, 2.0, 1.5, 4.0), car(1395, 1450, 16)], (375, 1392))
    add("wholly_right_then_past", [car(1395, 1450, 16), car(1100, 1300, 16)], (375, 1392))
    add("corner_at_depth_0", [box(-1.0, 1.0, 0.0, 16.0), car(100, 300, 16)])     # u = +-512 / 0 and 0 / 0
    for name, lines in KEYPOINT_BARS:
        add(name, lines)
    rs = np.random.RandomState(7)
    many = []
    for _ in range(100):
        u1 = float(rs.randint(-40, 1240))
        zn = float(2 ** rs.randint(3, 7))
        r = zn / (zn + 1.0) if u1 < 640 else (zn + 1.0) / zn      # the narrowest box the 1 m depth allows
        u2 = max(u1 + float(rs.randint(4, 160)) + 0.5, math.ceil(640.0 + (u1 - 640.0) * r) + 1.0)
        many.append(car(u1, u2, zn, typ=("Car", "Car", "Van")[rs.randint(3)]))
    add("hundred", many)
    for w in (1224, 1241, 1242, 1261):
        add("width_%d" % w, [car(1000, 1500, 16), car(100, 260, 32)], (375, w))
    return c


# ----------------------------------------------------------------------------------------------------- seeded cases
def seeded_cases(n, seed):
    rs = np.random.RandomState(seed)
    c = []
    for i in range(n):
        f = 7.0e2 + rs.rand() * 30
        cx, cy = 6.0e2 + rs.rand() * 10, 1.8e2 + rs.rand() * 8
        text = kitti_text(f, cx, cy, (0.0, 0.0, 0.0), (-3.8e2 - rs.rand() * 8, 0.0, 0.0),
                          (4.5e1 + rs.rand(), -0.3 * rs.rand(), 4.9e-3 * rs.rand()),
                          (-3.3e2 - rs.rand() * 8, 2.3 + 0.1 * rs.rand(), 3.2e-3 * rs.rand()))
        hw = ((375, 1242), (370, 1224))[i % 2]
        lines = []
        for _ in range(rs.randint(0, 14)):
            typ = ("Car", "Car", "Car", "Van", "Truck", "Pedestrian", "DontCare", "Cyclist", "Misc")[rs.randint(9)]
            z = 4.0 + rs.rand() * 60
            x = (rs.rand() * 2 - 1) * z * 0.7
            lines.append("%s %.2f %d %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f" % (
                typ, rs.choice([0.0, 0.0, 0.3, 0.99]), rs.randint(0, 4), (rs.rand() * 2 - 1) * 3.1,
                0, 0, 0, 0, 1.3 + rs.rand() * 0.6, 1.5 + rs.rand() * 0.4, 3.2 + rs.rand() * 1.5,
                x, 1.4 + rs.rand() * 0.5, z, (rs.rand() * 2 - 1) * 3.14))
        c.append(("seed%d_%d" % (seed, i), "".join(l + "\n" for l in lines), text, hw))
    return c


# -------------------------------------------------------------------------------------------------- the reference
def load_reference(shapes):
    ref_shim.load()
    cv2 = types.ModuleType("cv2")
    cv2.imread = lambda path: types.SimpleNamespace(shape=shapes[os.path.basename(path)[:-4]] + (3,))
    sys.modules["cv2"] = cv2
    sys.modules["cPickle"] = types.ModuleType("cPickle")
    ku = ref_shim._exec_module("model.utils.kitti_utils", os.path.join(ref_shim.LIB, "model/utils/kitti_utils.py"))
    sys.modules["model.utils"].kitti_utils = ku
    ds = types.ModuleType("datasets")
    ds.__path__ = [os.path.join(ref_shim.LIB, "datasets")]
    sys.modules["datasets"] = ds
    imdb = ref_shim._exec_module("datasets.imdb", os.path.join(ref_shim.LIB, "datasets/imdb.py"))
    kitti = ref_shim._exec_module("datasets.kitti", os.path.join(ref_shim.LIB, "datasets/kitti.py"))
    rdb = ref_shim._exec_module("roi_data_layer.roidb", os.path.join(ref_shim.LIB, "roi_data_layer/roidb.py"), [
        ("from datasets.factory import get_imdb", "get_imdb = None")])
    return imdb, kitti, rdb


FIELDS = (("boxes_left", 4), ("boxes_right", 4), ("boxes_merge", 4), ("dim_orien", 4), ("kpts", 6), ("kpts_right", 6),
          ("truncation", 1), ("occlusion", 1))


def occlusion_pass(db, objs, ix):
    """the reference's remove_occluded_keypoints(objs, left=(ix == 0)) -> (survivors, the smallest distance of a box
    edge to an integer and of a keypoint to its pruning bars, the bars (name, ix) on which a kept keypoint lies)"""
    before = {id(o): np.array(o.boxes[ix].keypoints, np.float64) for o in objs}
    out = db.remove_occluded_keypoints(objs, left=(ix == 0))
    m, hits = np.inf, set()
    for o in out:
        b = o.boxes[ix]
        for x in (b.box[0], b.box[2]):
            fr = x - math.floor(x)
            if fr != 0.0:
                m = min(m, fr, 1.0 - fr)
        kp = [k for k in before[id(o)] if k != -1]
        if not kp:
            continue
        lk, rk = min(kp), max(kp)
        bars = (("vl-5", b.visible_left - 5), ("vr+5", b.visible_right + 5), ("lk+3", lk + 3), ("rk-3", rk - 3))
        for k in kp:
            for name, bar in bars:
                if k not in (lk, rk) or name in ("vl-5", "vr+5"):
                    m = min(m, abs(k - bar))
        for k in b.keypoints:
            for name, bar in bars:
                if k != -1 and k == bar:
                    hits.add((name, ix))
    return out, m, hits


def kept(o):
    """_load_kitti_annotation's filter (kitti.py:215-219)"""
    b0, b1 = o.boxes[0], o.boxes[1]
    return (o.truncate < 0.98 and o.occlusion < 3 and b0.box[3] - b0.box[1] > 10 and o.cls == "Car" and
            b0.visible_right - b0.visible_left > 3 and b1.visible_right - b1.visible_left > 3)


def main():
    cases = exact_cases()
    n_exact = len(cases)
    cases += seeded_cases(40, 11)
    shapes = {"%06d" % i: hw for i, (_n, _l, _c, hw) in enumerate(cases)}
    imdb_mod, kitti_mod, rdb = load_reference(shapes)
    with tempfile.TemporaryDirectory() as root:
        for sub in ("label_2", "calib", "image_2", "image_3"):
            os.makedirs(os.path.join(root, "training", sub))
        for i, (_n, lab, cal, hw) in enumerate(cases):
            idx = "%06d" % i
            with open(os.path.join(root, "training", "label_2", idx + ".txt"), "w") as f:
                f.write(lab)
            with open(os.path.join(root, "training", "calib", idx + ".txt"), "w") as f:
                f.write(cal)
            for side in ("image_2", "image_3"):
                with open(os.path.join(root, "training", side, idx + ".png"), "wb") as f:
                    f.write(png_header(*hw))
        db = kitti_mod.kitti.__new__(kitti_mod.kitti)
        imdb_mod.imdb.__init__(db, "kitti_train", ("__background__", "Car"))
        db._image_set, db._kitti_path, db._data_path = "train", root, root
        db._class_to_ind = dict(zip(db.classes, range(db.num_classes)))
        db._image_ext = ".png"
        ku = sys.modules["model.utils.kitti_utils"]
        out = {k: [] for k, _w in FIELDS}
        n_kept, status, roidb, ok, min_margin, bar_hits = [], [], [], [], np.inf, []
        for i, (name, lab, cal, hw) in enumerate(cases):
            idx = "%06d" % i
            try:
                e = db._load_kitti_annotation(idx)
                s = 0
            except IndexError as exc:
                # the object the reference stopped at: the loop variable of remove_occluded_keypoints' frame, found
                # again among the image's objects by its class, position and dimensions
                tb = exc.__traceback__
                while tb.tb_frame.f_code.co_name != "remove_occluded_keypoints":
                    tb = tb.tb_next
                loc = tb.tb_frame.f_locals
                o = loc["objects"][loc["i"]]
                calib = ku.read_obj_calibration(os.path.join(root, "training", "calib", idx + ".txt"))
                objs = ku.read_obj_data(os.path.join(root, "training", "label_2", idx + ".txt"), calib, hw)
                s = 1 + [k for k, p in enumerate(objs) if p.cls == o.cls and (p.pos == o.pos).all() and
                         (p.dim == o.dim).all()][0]
                e = None
            if e is not None:
                calib = ku.read_obj_calibration(os.path.join(root, "training", "calib", idx + ".txt"))
                objs = ku.read_obj_data(os.path.join(root, "training", "label_2", idx + ".txt"), calib, hw)
                left, m0, _h = occlusion_pass(db, objs, 0)
                right, m1, _h = occlusion_pass(db, left, 1)
                if i >= n_exact:
                    min_margin = min(min_margin, m0, m1)
                elif name.startswith("kp_"):
                    # the case puts a keypoint of a kept object on its bar: replay both passes on the kept object
                    objs = ku.read_obj_data(os.path.join(root, "training", "label_2", idx + ".txt"), calib, hw)
                    left, _m, h0 = occlusion_pass(db, objs, 0)
                    right, _m, h1 = occlusion_pass(db, left, 1)
                    side, bar = name[3:].split("_")
                    want = ({"lk3": "lk+3", "rk3": "rk-3", "vl5": "vl-5", "vr5": "vr+5"}[bar], side == "right")
                    assert want in h0 | h1 and any(kept(o) for o in right), (name, h0, h1)
                    bar_hits.append(name)
            status.append(s)
            n = 0 if e is None else len(e["gt_classes"])
            n_kept.append(n)
            for k, w in FIELDS:
                out[k].append(np.zeros((0, w), np.float32) if e is None else np.asarray(e[k], np.float32).reshape(n, w))
            if e is not None:
                assert (e["gt_classes"] == 1).all() and e["flipped"] is False
                roidb.append(e)
                ok.append(i)
            print("%-18s status %d kept %d" % (name, s, n))
        assert min_margin > 1e-6, min_margin
        assert len(bar_hits) == len(KEYPOINT_BARS), bar_hits
        # flip and filter, as combined_roidb('kitti_train') runs them, on the entries that did not raise
        db._roidb = [dict(e) for e in roidb]
        db._image_index = ["%06d" % i for i in ok]
        db._get_widths = lambda: [cases[i][3][1] for i in ok]
        db.append_flipped_images()
        flipped = rdb.filter_roidb(list(db.roidb))
        kept_src = [int(db._image_index[[j for j, x in enumerate(db.roidb) if x is e][0]]) for e in flipped]
        flip = {k: np.concatenate([np.asarray(e[k], np.float32).reshape(-1, w) for e in flipped])
                for k, w in FIELDS[:5]}
    rows = lambda k, w: np.concatenate(out[k]).reshape(-1, w)
    np.savez_compressed(
        os.path.join(HERE, "kitti_annotations.npz"),
        names=np.array([c[0] for c in cases]), labels=np.array([c[1] for c in cases]),
        calibs=np.array([c[2] for c in cases]), image_hw=np.array([c[3] for c in cases], np.int32),
        n_exact=n_exact, status=np.array(status, np.int32), n_kept=np.array(n_kept, np.int32),
        min_margin=min_margin, bar_cases=np.array(bar_hits), flip_source=np.array(kept_src, np.int32),
        flip_flipped=np.array([bool(e["flipped"]) for e in flipped]),
        flip_n=np.array([len(e["gt_classes"]) for e in flipped], np.int32),
        **{k: rows(k, w) for k, w in FIELDS}, **{"flip_" + k: v for k, v in flip.items()})
    print("wrote kitti_annotations.npz: %d cases (%d exact), min margin %.3g px" % (len(cases), n_exact, min_margin))


if __name__ == "__main__":
    main()
