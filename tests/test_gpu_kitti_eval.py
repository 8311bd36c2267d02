"""GPU: sb_kitti_overlaps and sb_kitti_eval against the oracle's restatement of the devkit's evaluate_object
(oracle/kitti_eval.py): overlaps bit for bit; counts, thresholds, precision, recall and AP bit for bit, AOS to 1e-12
(cos on the device); on the hand cases of test_kitti_eval.py, a seeded synthetic split, and an image whose overlap
matrix does not fit in shared memory.  And pipeline.evaluate(labels=...) against evaluate_dirs over its own files."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import kitti_eval as O
from stereo_rcnn_b200 import kitti_eval as K
from stereo_rcnn_b200 import ops as G
from stereo_rcnn_b200 import pipeline as PL
from stereo_rcnn_b200 import synth

from test_kitti_eval import CASES, bev_pairs, row
from test_gpu_evaluate import TARGET, calib, frame_pair, pipe, split  # noqa: F401  (pipe is a fixture)

pytestmark = pytest.mark.gpu
EXACT = ("thresholds", "n_thresholds", "tp", "fp", "fn", "precision", "recall", "n_gt")


def device_inputs(images):
    ev = K.KittiEval("cuda")
    for g, gc, d, dc in images:
        ev.images.append((np.asarray(gc, np.int32), np.asarray(g, np.float64).reshape(-1, 16),
                          np.asarray(dc, np.int32), np.asarray(d, np.float64).reshape(-1, 16)))
    return ev.device_inputs()


def device_eval(images, bars=(0.7, 0.5)):
    (gt, gc, det, dc, go, do, po), n_pairs = device_inputs(images)
    out = G.kitti_eval(gt, gc, det, dc, go, do, po, n_pairs, bars)
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items() if k != "_buffer"}


def assert_matches_oracle(images, bars=(0.7, 0.5)):
    got, ref = device_eval(images, bars), O.evaluate(images, bars)
    for k in EXACT:
        assert np.array_equal(got[k], ref[k]), k
    assert np.array_equal(got["ap"][:, :2], ref["ap"][:, :2])
    for k, v in (("sim", got["sim"]), ("aos", got["aos"]), ("ap_aos", got["ap"][:, 2:])):
        r = ref["ap"][:, 2:] if k == "ap_aos" else ref[k]
        assert np.allclose(v, r, rtol=1e-12, atol=1e-12), k
    return got


def images_of(split_text):
    ev = K.KittiEval("cpu")
    for g, d in split_text:
        ev.add(g, d)
    return [(g, gc, d, dc) for gc, g, dc, d in ev.images]


# ------------------------------------------------------------------------------------------------ overlaps ----
def box(rs):
    xs, ys = np.sort(rs.uniform(0, 200, 2)), np.sort(rs.uniform(0, 100, 2))
    return (xs[0], ys[0], xs[1], ys[1])


def overlap_sweep():
    """rows with the BEV pairs of the CPU test, plus random full rows: rotations across +-pi, heights with zero,
    partial and full vertical overlap, DontCare columns"""
    rs = np.random.RandomState(11)
    imgs = []
    for a, b in bev_pairs():
        a, b = list(a), list(b)
        a[O.X1:O.Y2 + 1], b[O.X1:O.Y2 + 1] = [0, 0, 10, 10], [5, 5, 15, 15]
        a[O.H], a[O.Y], b[O.H], b[O.Y] = 1.5, 1.6, 1.5, 1.6 + rs.choice([0.0, 0.7, 1.5, 2.0])
        imgs.append((np.array([b]), np.array([0], np.int32), np.array([a]), np.array([0], np.int32)))
    for _ in range(6):
        ng, nd = rs.randint(1, 9), rs.randint(1, 20)
        gts = [row(box(rs), y=rs.uniform(1, 2), h=rs.uniform(1, 2), x=rs.uniform(-2, 2), z=rs.uniform(10, 13),
                   ry=rs.uniform(-math.pi - 0.2, math.pi + 0.2)) for _g in range(ng)]
        dets = [list(gts[rs.randint(ng)]) for _d in range(nd)]
        for d in dets:
            d[O.X1:O.Y2 + 1] = list(np.array(d[O.X1:O.Y2 + 1]) + rs.randn(4) * 5)
            d[O.X] += rs.randn() * 0.5
            d[O.Y] += rs.choice([0.0, rs.randn() * 0.5, 3.0])
            ry = math.atan2(d[O.SIN], d[O.COS]) + rs.randn() * 0.4
            d[O.COS], d[O.SIN] = math.cos(ry), math.sin(ry)
        codes = rs.choice([0, 1, 2, 3], ng).astype(np.int32)
        imgs.append((np.array(gts), codes, np.array(dets), np.zeros(nd, np.int32)))
    imgs.append((np.zeros((0, 16)), np.zeros(0, np.int32), np.array(dets), np.zeros(len(dets), np.int32)))
    return imgs


def test_overlaps_bit_exact_vs_oracle():
    imgs = overlap_sweep()
    (gt, gc, det, _dc, go, do, po), n_pairs = device_inputs(imgs)
    got = [v.cpu().numpy() for v in G.kitti_overlaps(gt, gc, det, go, do, po, n_pairs)]
    po = po.cpu().numpy()
    nz = 0
    for k, (g, gcodes, d, _c) in enumerate(imgs):
        ref = O.overlaps(g, gcodes, d)
        for m in range(3):
            dev = got[m][po[k]:po[k + 1]].reshape(ref[m].shape)
            assert np.array_equal(dev.view(np.int64), ref[m].view(np.int64)), (k, m)
            nz += int((ref[m] > 0).sum())
    assert nz > 200


# ------------------------------------------------------------------------------------------------ matching ----
@pytest.mark.parametrize("name", sorted(CASES))
def test_eval_hand_cases(name):
    images, bars, _expect = CASES[name]
    assert_matches_oracle(images, bars)


def test_eval_worked_cases():
    from test_kitti_eval import exact_split
    got = assert_matches_oracle(exact_split(1))
    assert (got["ap"][:, 1] == 0).all() and np.allclose(got["ap"][:, 0], 100 / 11, rtol=0, atol=1e-12)
    got = assert_matches_oracle(exact_split(41))
    assert np.allclose(got["ap"], 100, rtol=0, atol=1e-12)


def test_eval_synthetic_split_and_run_to_run_identity():
    images = images_of(synth.kitti_split(300, seed=3))
    got = assert_matches_oracle(images, (0.7, 0.5, 0.3))
    assert (got["n_thresholds"] > 10).all() and (got["ap"][:, 0] > 0).all()
    again = device_eval(images, (0.7, 0.5, 0.3))
    for k in got:
        assert np.array_equal(got[k].view(np.uint8), again[k].view(np.uint8)), k


def test_eval_image_larger_than_shared_memory():
    """120 detections x 40 gt rows: 38 KB of overlaps per metric, matched from global memory, among small images"""
    big = synth.kitti_split(1, seed=9, n_cars=36, n_dets=120)
    split_text = synth.kitti_split(20, seed=8)
    images = images_of(split_text[:10] + big + split_text[10:])
    assert len(images[10][0]) * len(images[10][2]) * 8 > 8192
    assert_matches_oracle(images)


# ------------------------------------------------------------------------------------------ pipeline.evaluate ----
def test_evaluate_with_labels_scores_its_own_files(pipe, tmp_path):  # noqa: F811
    entries = split(8)
    frames = lambda e: frame_pair(*e["hw"], seed=e["seed"])
    cal = lambda e: calib(e["cal"], div=3.75)
    for empty in (False, True):
        plain, scored = str(tmp_path / ("plain%d" % empty)), str(tmp_path / ("scored%d" % empty))
        PL.evaluate(pipe, entries, frames, cal, plain, target_size=TARGET, empty_files=empty, log=lambda s: None)
        # labels: each written detection as a Car label, moved a little, and one missed Car per image
        label_dir = tmp_path / ("labels%d" % empty)
        label_dir.mkdir()
        rs = np.random.RandomState(4)
        for e in entries:
            p = os.path.join(plain, "data", e["image_id"] + ".txt")
            lines = open(p).read().splitlines() if os.path.exists(p) else []
            out = []
            for ln in lines:
                f = ln.split()[:15]
                for k in (4, 5, 6, 7):
                    f[k] = "%.2f" % (float(f[k]) + rs.randn() * 2.0)
                f[1], f[2] = "0.00", "0"
                out.append(" ".join(f))
            out.append("Car 0.00 0 0.1 10 100 90 180 1.5 1.6 3.9 -9 1.6 12 0.2")
            (label_dir / (e["image_id"] + ".txt")).write_text("\n".join(out) + "\n")
        labels = lambda e: str(label_dir / (e["image_id"] + ".txt"))
        summary = PL.evaluate(pipe, entries, frames, cal, scored, target_size=TARGET, empty_files=empty,
                              log=lambda s: None, labels=labels)
        files = sorted(os.listdir(os.path.join(plain, "data")))
        assert files == sorted(os.listdir(os.path.join(scored, "data")))
        for f in files:
            assert open(os.path.join(plain, "data", f)).read() == open(os.path.join(scored, "data", f)).read()
        ref = K.evaluate_dirs(str(label_dir), scored, [e["image_id"] for e in entries], "cuda")
        ap = summary["ap"]
        for m in ("bbox", "aos", "bev", "3d"):
            for bar in (0.7, 0.5):
                assert np.array_equal(ap[m][bar], ref[m][bar]), (m, bar)
        assert np.array_equal(ap["n_gt"], ref["n_gt"]) and ap["n_gt"][2] >= len(entries)
        assert ap["bbox"][0.5][2, 0] > 0
