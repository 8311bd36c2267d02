"""GPU: sb_kitti_eval and sb_kitti_overlaps at their edges, on the builders of test_kitti_eval_edges.py, against the
oracle (oracle/kitti_eval.py) with assert_matches_oracle's criteria: thresholds, counts, precision, recall, n_gt and
AP R11 / R40 bit for bit, sim and AOS to 1e-12; overlaps bit for bit.

* the threshold scan's 1024-image chunks (1023 to 3769 images), the rank kernel's 256-score blocks and ties, the
  threshold lanes (0 to 41 thresholds, assigned bits past word 0), the 8 KB staging limit, the pair search over empty
  images, overlap geometry at zero extents, quarter turns, thin, far, collinear and touching rectangles;
* on a light split the size of KITTI val: shuffled images, inserted empty images and a second run change nothing;
* KittiEval.result() against the documented configuration index c = (metric * n_bars + bar) * 3 + difficulty.
"""
import numpy as np
import pytest
import torch

from oracle import kitti_eval as O
from stereo_rcnn_b200 import kitti_eval as K
from stereo_rcnn_b200 import ops as G

import test_kitti_eval_edges as E
from test_gpu_kitti_eval import EXACT, assert_matches_oracle, device_eval, device_inputs

pytestmark = pytest.mark.gpu
BARS = (0.7, 0.5)


def assert_same(a, b, close=()):
    for k in a:
        if k in close:
            assert np.allclose(a[k], b[k], rtol=1e-12, atol=1e-12), k
        else:
            assert np.array_equal(a[k].view(np.uint8), b[k].view(np.uint8)), k


@pytest.fixture(scope="module")
def val():
    return E.val_split()


# ------------------------------------------------------------------------------------------------ scan chunks ----
@pytest.mark.parametrize("n", E.CHUNK_SIZES)
def test_chunks(n):
    got = assert_matches_oracle(E.chunk_split(n), BARS)
    assert (got["n_thresholds"] > E.LANES).all()


@pytest.mark.parametrize("variant", ["quiet_edges", "empty_ends"])
def test_chunk_variants(variant):
    n = 2060 if variant == "quiet_edges" else 2049
    assert_matches_oracle(E.chunk_split(n, **{variant: True}), BARS)


# ------------------------------------------------------------------------------------------------ rank ----
@pytest.mark.parametrize("kind", E.RANK_KINDS)
def test_rank_blocks(kind):
    imgs = E.rank_split(kind)
    assert_matches_oracle(imgs, BARS)
    if kind == "at_threshold":
        assert_matches_oracle(imgs, E.FOUR_BARS)


# ------------------------------------------------------------------------------------------------ lanes ----
@pytest.mark.parametrize("k", E.THRESHOLD_COUNTS)
@pytest.mark.parametrize("bars", [BARS, E.FOUR_BARS], ids=["two_bars", "four_bars"])
def test_threshold_counts(k, bars):
    got = assert_matches_oracle(E.threshold_split(k), bars)
    if bars == BARS:
        assert (got["n_thresholds"] == k).all()


def test_threshold_count_33_in_one_global_image():
    imgs = E.threshold_split(33, one_image=True)
    assert (assert_matches_oracle(imgs, BARS)["n_thresholds"] == 33).all()
    assert_matches_oracle(imgs, E.FOUR_BARS)


@pytest.mark.parametrize("bars", [BARS, E.FOUR_BARS], ids=["two_bars", "four_bars"])
def test_lane_second_threshold_starts_clear(bars):
    got = assert_matches_oracle(E.lane_split(), bars)
    assert (got["n_thresholds"].max() > E.LANES)


# ------------------------------------------------------------------------------------------------ staging ----
@pytest.mark.parametrize("bars", [BARS, E.FOUR_BARS], ids=["two_bars", "four_bars"])
def test_staging_edges(bars):
    assert_matches_oracle(E.stage_split(), bars)


def test_global_path_runs():
    assert_matches_oracle(E.global_run_split(), BARS)


# ------------------------------------------------------------------------------------------------ pair search ----
def test_empty_image_runs():
    imgs = E.pair_split()
    assert_matches_oracle(imgs, E.FOUR_BARS)
    (gt, gc, det, _dc, go, do, po), n_pairs = device_inputs(imgs)
    got = [v.cpu().numpy() for v in G.kitti_overlaps(gt, gc, det, go, do, po, n_pairs)]
    ref = [np.concatenate([O.overlaps(g, c, d)[m].ravel() for g, c, d, _ in imgs]) for m in range(3)]
    for m in range(3):
        assert np.array_equal(got[m].view(np.int64), ref[m].view(np.int64)), m


def test_no_pairs_with_gt_rows():
    got = assert_matches_oracle(E.no_pair_split(), E.FOUR_BARS)
    assert (got["n_thresholds"] == 0).all() and (got["n_gt"] > 0).all() and (got["ap"] == 0).all()


# ------------------------------------------------------------------------------------------------ geometry ----
def test_overlap_geometry_bit_exact():
    imgs = E.geometry_images()
    (gt, gc, det, _dc, go, do, po), n_pairs = device_inputs(imgs)
    got = [v.cpu().numpy() for v in G.kitti_overlaps(gt, gc, det, go, do, po, n_pairs)]
    po = po.cpu().numpy()
    for k, (g, c, d, _) in enumerate(imgs):
        ref = O.overlaps(g, c, d)
        for m in range(3):
            dev = got[m][po[k]:po[k + 1]].reshape(ref[m].shape)
            assert np.array_equal(dev.view(np.int64), ref[m].view(np.int64)), (k, m)
    assert_matches_oracle(imgs, E.FOUR_BARS)


# ------------------------------------------------------------------------------------------------ val size ----
def test_val_size_split(val):
    assert len(val) == 3769
    assert_matches_oracle(val, BARS)


def test_val_size_invariances(val):
    """no oracle: the image order changes no count, threshold, precision, recall or AP R11 / R40 (sim and AOS only
    by the order of their sums); empty images anywhere change nothing; two runs agree bit for bit"""
    ref = device_eval(val, BARS)
    assert_same(device_eval(val, BARS), ref)
    rs = np.random.RandomState(3)
    perm = rs.permutation(len(val))
    shuffled = device_eval([val[i] for i in perm], BARS)
    assert_same({k: v for k, v in shuffled.items() if k != "ap"}, ref, close=("sim", "aos"))
    assert np.array_equal(shuffled["ap"][:, :2], ref["ap"][:, :2])
    assert np.allclose(shuffled["ap"][:, 2:], ref["ap"][:, 2:], rtol=1e-12, atol=1e-12)
    padded = list(val)
    for at in sorted(set(rs.randint(0, len(val), 40).tolist()) | {0, 1023, 1024, 2048, len(val)}, reverse=True):
        padded[at:at] = [E.image()] * (1 + at % 3)
    assert len(padded) > 3769 + 40
    assert_same(device_eval(padded, BARS), ref)


# ------------------------------------------------------------------------------------------------ result() ----
@pytest.mark.parametrize("bars", [(0.7,), (0.7, 0.5, 0.3), E.FOUR_BARS], ids=["one_bar", "three_bars", "four_bars"])
def test_result_table_follows_the_configuration_index(bars):
    imgs = E.table_split()
    ev = K.KittiEval("cuda", bars)
    for g, gc, d, dc in imgs:
        ev.images.append((np.asarray(gc, np.int32), np.asarray(g, np.float64).reshape(-1, 16),
                          np.asarray(dc, np.int32), np.asarray(d, np.float64).reshape(-1, 16)))
    table = ev.result()
    ref = O.evaluate(imgs, bars)
    nb = len(bars)
    for m, metric in enumerate(K.METRICS):
        for b, bar in enumerate(bars):
            for d in range(3):
                c = (m * nb + b) * 3 + d
                assert np.array_equal(table[metric][bar][d], ref["ap"][c, :2]), (metric, bar, d)
                if metric == "bbox":
                    assert np.allclose(table["aos"][bar][d], ref["ap"][c, 2:], rtol=1e-12, atol=1e-12), (bar, d)
                for k in EXACT:
                    if k != "n_gt":
                        assert np.array_equal(table["curves"][metric][bar][k][d], ref[k][c]), (metric, bar, d, k)
    assert np.array_equal(table["n_gt"], ref["n_gt"][:3])
    torch.cuda.synchronize()
