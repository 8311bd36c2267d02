"""CPU: oracle/kitti_annotations.py against the reference golden (tests/golden/make_kitti_annotations_golden.py) --
bit for bit on the exact cases, within 4 ulp with identical decisions on the seeded ones -- train_roidb's flip and
filter against the reference's append_flipped_images + filter_roidb, and the host refusals of kitti_data."""
import os

import numpy as np
import pytest

from oracle import kitti_annotations as OA
from stereo_rcnn_b200 import kitti_data as KD
from stereo_rcnn_b200 import ops
from stereo_rcnn_b200 import synth
from stereo_rcnn_b200 import train as TR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "kitti_annotations.npz")
FIELDS = (("boxes_left", 0, 4), ("boxes_right", 4, 8), ("boxes_merge", 8, 12), ("dim_orien", 12, 16),
          ("kpts", 16, 22), ("kpts_right", 22, 28), ("truncation", 28, 29), ("occlusion", 29, 30))


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def golden_rows(g):
    """the reference's kept rows of every case in sb_kitti_annotations' layout, and the per-case row offsets"""
    out = np.concatenate([g[k].reshape(len(g[k]), -1) for k, _lo, _hi in FIELDS], axis=1)
    off = np.concatenate([[0], np.cumsum(g["n_kept"])])
    return out, off


def oracle_case(g, i):
    rows, codes, cal, _lines = KD.pack_image(str(g["labels"][i]), ops.read_calibration(str(g["calibs"][i])))
    return OA.image(rows, codes, cal, int(g["image_hw"][i][0]), int(g["image_hw"][i][1]))


def ulps(a, b):
    a, b = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    a = np.where(a < 0, -(a & 0x7FFFFFFF), a)
    b = np.where(b < 0, -(b & 0x7FFFFFFF), b)
    return np.abs(a - b)


def test_oracle_equals_the_reference_bit_for_bit_on_the_exact_cases(gold):
    out, off = golden_rows(gold)
    for i in range(int(gold["n_exact"])):
        got, status = oracle_case(gold, i)
        assert status == gold["status"][i], gold["names"][i]
        assert np.array_equal(got.view(np.uint32), out[off[i]:off[i + 1]].view(np.uint32)), gold["names"][i]


def test_oracle_matches_the_reference_on_the_seeded_cases(gold):
    out, off = golden_rows(gold)
    assert gold["min_margin"] > 1e-6
    for i in range(int(gold["n_exact"]), len(gold["names"])):
        got, status = oracle_case(gold, i)
        want = out[off[i]:off[i + 1]]
        assert status == gold["status"][i] and got.shape == want.shape, gold["names"][i]
        for lo in (16, 22):                                  # the same keypoints dropped, the same integer vl / vr
            assert np.array_equal(got[:, lo:lo + 4] == -1, want[:, lo:lo + 4] == -1)
        assert ulps(got, want).max(initial=0) <= 4, gold["names"][i]


def test_the_boundary_cases_decide_as_the_spec_says(gold):
    names = list(gold["names"])
    st = dict(zip(names, gold["status"].tolist()))
    kept = dict(zip(names, gold["n_kept"].tolist()))
    assert st["past_1259"] == 1 and st["behind_camera"] == 2 and st["width_1261"] == 1
    assert st["behind_then_past"] == 2                      # painting fails before the end lookups
    assert kept["visible_3.0"] == 0 and kept["visible_3.5"] == 1 and kept["height_10"] == 1
    assert kept["occ_trunc"] == 1 and kept["both_hidden"] == 1 and kept["van_hides_car"] == 1
    assert kept["no_used"] == kept["none_kept"] == kept["empty"] == 0 and kept["edge_1259"] == 1
    # a box wholly right of the depth line paints nothing: the earlier object behind the camera fails first, and a
    # later box that paints past column 1259 fails before its end lookups
    assert st["wholly_right_after_behind"] == 1 and st["wholly_right_then_past"] == 2
    # each of the four pruning bars of each camera holds a kept keypoint of a kept object (checked by the maker)
    bars = sorted(str(n) for n in gold["bar_cases"])
    assert bars == sorted("kp_%s_%s" % (s, b) for s in ("left", "right") for b in ("lk3", "rk3", "vl5", "vr5"))
    assert all(kept[n] == 1 for n in bars)


def test_flip_and_filter_equal_the_reference(gold):
    out, off = golden_rows(gold)
    ok = [i for i in range(len(gold["names"])) if gold["status"][i] == 0]
    entries = []
    for i in ok:
        r = out[off[i]:off[i + 1]]
        e = {k: r[:, lo:hi].copy() for k, lo, hi in FIELDS[:6]}
        e["gt_classes"], e["flipped"], e["src"] = np.ones(len(r), np.int32), False, i
        entries.append(e)
    roidb = KD.filter_roidb(TR.append_flipped(entries, [int(gold["image_hw"][i][1]) for i in ok]))
    assert [e["src"] for e in roidb] == gold["flip_source"].tolist()
    assert [e["flipped"] for e in roidb] == gold["flip_flipped"].tolist()
    assert [len(e["gt_classes"]) for e in roidb] == gold["flip_n"].tolist()
    for k, _lo, _hi in FIELDS[:5]:
        got = np.concatenate([e[k] for e in roidb])
        assert np.array_equal(got.view(np.uint32), gold["flip_" + k].view(np.uint32)), k


# ----------------------------------------------------------------------------------------------------- host refusals
@pytest.fixture()
def folder(tmp_path):
    ids = synth.kitti_folder(str(tmp_path), 3, seed=4)
    return str(tmp_path), ids


def test_png_size_reads_the_header_and_refuses_other_files(folder, tmp_path):
    root, ids = folder
    assert KD.png_size(os.path.join(root, "training", "image_2", ids[1] + ".png")) == (370, 1224)
    bad = os.path.join(root, "training", "image_2", ids[0] + ".png")
    with open(bad, "wb") as f:
        f.write(b"\xff\xd8\xff\xe0" + b"\x00" * 40)            # a JPEG named .png
    with pytest.raises(ValueError, match=r"%s is not a PNG file" % bad):
        KD.Split(root, ids)


@pytest.mark.parametrize("sub,what", [("label_2", "label file"), ("calib", "calibration file"),
                                      ("image_2", "left image"), ("image_3", "right image")])
def test_missing_files_are_refused(folder, sub, what):
    root, ids = folder
    path = os.path.join(root, "training", sub, ids[2] + (".txt" if sub in ("label_2", "calib") else ".png"))
    os.remove(path)
    with pytest.raises(FileNotFoundError, match="no %s for image %s" % (what, ids[2])):
        KD.Split(root, ids)


def test_malformed_lines_are_refused_naming_the_file(folder):
    root, ids = folder
    lab = os.path.join(root, "training", "label_2", ids[0] + ".txt")
    with open(lab, "a") as f:
        f.write("Car 0.00 0 0.1 1 2 3 4 1.5 1.6 3.9 1.0 1.6 x 0.1\n")
    with pytest.raises(ValueError, match=r"%s line \d+: a field after the type is not a number" % lab):
        KD.Split(root, ids)
    with open(lab, "w") as f:
        f.write("Car 0.00 0 0.1 1 2 3 4\n")
    with pytest.raises(ValueError, match=r"%s line 1: 8 fields" % lab):
        KD.Split(root, ids)
    with open(lab, "w") as f:
        f.write("")
    cal = os.path.join(root, "training", "calib", ids[1] + ".txt")
    with open(cal, "w") as f:
        f.write("P0: 1 2 3\nP1: 1\n")
    with pytest.raises(ValueError, match=r"%s: calibration line 1" % cal):
        KD.Split(root, ids)


def test_a_status_names_the_image_and_the_label_line(tmp_path, gold):
    i = list(gold["names"]).index("behind_then_past")
    d = tmp_path / "training"
    for sub in ("label_2", "calib", "image_2", "image_3"):
        (d / sub).mkdir(parents=True)
    text = "DontCare -1 -1 -10 0 0 0 0 -1 -1 -1 -1000 -1000 -1000 -10\n\n" + str(gold["labels"][i])
    (d / "label_2" / "000042.txt").write_text(text)
    (d / "calib" / "000042.txt").write_text(str(gold["calibs"][i]))
    h, w = (int(v) for v in gold["image_hw"][i])
    for sub in ("image_2", "image_3"):
        (d / sub / "000042.png").write_bytes(synth.png_bytes(np.zeros((h, w, 3), np.uint8)))
    split = KD.Split(str(tmp_path), ["000042"])
    _out, _n, status = OA.split(*split.arrays())
    assert status.tolist() == [2]
    with pytest.raises(ValueError, match=r"image 000042: the box of the object on line 4 of .*000042.txt reaches "
                                         r"past column 1259 .*the reference raises IndexError here"):
        split.check_status(status)
