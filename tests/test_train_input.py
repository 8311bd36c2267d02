"""CPU: the training side of the input pipeline -- oracle/train_input.py against tests/golden/train_batch.npz (minted
from the reference's own append_flipped_images, get_minibatch and roibatchLoader.__getitem__), Philox4x32-10 against
the Random123 known-answer vectors, train.append_flipped against the golden and as an involution, the sampler order and
lr schedule of train.fit, and the argument checks of the four new entry points (SB_EINVAL before any CUDA call)."""
import os

import numpy as np
import pytest
import torch

from oracle import train_input as TI
from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import train as TR

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "train_batch.npz")
ROW_KEYS = ("boxes_left", "boxes_right", "boxes_merge", "dim_orien", "kpts")
GT_KEYS = ("gt_left", "gt_right", "gt_merge", "gt_dim_orien", "gt_kpts")
SB_EINVAL = -22
FAKE = 1 << 20                                            # never dereferenced: every refusal precedes the first call


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def golden_entry(g, i, padded=False):
    """entry i of the golden roidb (12 entries: 6 and their flips); padded: at the stored capacity of 40 rows"""
    n = int(g["n_rows"][i])
    e = {k: g[k][i] if padded else g[k][i][:n] for k in ROW_KEYS + ("gt_classes",)}
    if i < len(g["widths"]):
        e["kpts_right"] = g["kpts_right"][i] if padded else g["kpts_right"][i][:n]
    e["flipped"] = bool(g["flipped"][i])
    return e, n


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.int32), b.view(np.int32))


def test_golden_covers_the_edges(gold):
    g = gold
    s, wid = np.float32(g["scale"]), g["im_info"][:, 1]
    assert len(g["n_rows"]) == 12 and g["flipped"].sum() == 6
    assert (g["boxes_left"][:, :, 0] * s > wid[:, None]).any()                     # x1 beyond the blob's width
    k = g["kpts"] * s
    assert ((k > wid[:, None, None] - 1) & (g["gt_classes"] != 0)[:, :, None]).any() and (k == 100.0).any()
    assert ((g["kpts"] < 0) & (g["kpts"] > -1)).any()
    th = g["dim_orien"][:6, :, 3]
    assert (th > np.pi).any() and (th < -np.pi).any() and (th > 0).any() and (th < 0).any() and (th[3, :8] == 0).any()
    assert ((g["gt_classes"] == 0) & (np.arange(40) < g["n_rows"][:, None])).any()  # class-0 rows in use
    assert ((g["gt_classes"] != 0).sum(1) > 30).any() and (g["num_boxes"] == 0).any() and (g["num_boxes"] == 30).any()


def test_oracle_train_gt_equals_the_reference_bit_for_bit(gold):
    g = gold
    for i in range(12):
        for padded in (False, True):
            e, n = golden_entry(g, i, padded)
            words = g["words"][i] if padded else g["words"][i][:n]
            out = TI.train_gt(e, float(g["scale"]), int(g["im_info"][i, 1]), words, n)
            for k, o in zip(GT_KEYS, out[:5]):
                assert same_bits(o, g[k][i]), (i, k)
            assert out[5] == g["num_boxes"][i]
        # the stored permutation is the order the words give
        valid = (g["gt_classes"][i] != 0) & (np.arange(40) < n)
        nb = int(g["num_boxes"][i])
        assert np.array_equal(TI.word_order(g["words"][i], valid)[:nb], g["perm"][i][:nb])
    assert np.allclose(g["im_info"][:, 2], g["scale"]) and (g["im_info"][:, :2] == (32, 101)).all()


def test_oracle_pair_blobs_against_the_reference(gold):
    """the flip of the pair is exact (which frame, mirrored or not); the blob itself is within the bar of
    prep_image against cv2.resize (2 ulp of the largest tap)"""
    g = gold
    for j, i in enumerate(g["blob_entries"]):
        left, right = g["frames_left"][i % 6][:, :, ::-1], g["frames_right"][i % 6][:, :, ::-1]     # RGB -> BGR
        bl, br = TI.pair_blobs(left, right, float(g["scale"]), bool(g["flipped"][i]))
        for got, ref in ((bl, g["blob_left"][j]), (br, g["blob_right"][j])):
            assert got.shape == ref.shape and np.abs(got - ref).max() <= 2 * np.spacing(np.float32(160.0))
    assert g["flipped"][g["blob_entries"]].tolist() == [False, False, True, True]
    # the wrong pairing is far outside that bar
    bl, _ = TI.pair_blobs(g["frames_left"][0][:, :, ::-1], g["frames_right"][0][:, :, ::-1], 1.6, False)
    assert np.abs(bl - g["blob_left"][2]).max() > 1.0


PHILOX_KAT = [   # Random123 kat_vectors, philox4x32 10: counter / key -> output
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
]


def philox_scalar(ctr, key):
    """a second restatement, on Python integers"""
    c, k = list(ctr), list(key)
    for _ in range(10):
        p0, p1 = 0xD2511F53 * c[0], 0xCD9E8D57 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k[0], p1 & 0xFFFFFFFF, (p0 >> 32) ^ c[3] ^ k[1], p0 & 0xFFFFFFFF]
        k = [(k[0] + 0x9E3779B9) & 0xFFFFFFFF, (k[1] + 0xBB67AE85) & 0xFFFFFFFF]
    return tuple(c)


def test_philox_known_answers():
    for ctr, key, out in PHILOX_KAT:
        assert philox_scalar(ctr, key) == out
        assert tuple(int(v) for v in TI.philox4x32_10(np.array(ctr, np.uint32), np.array(key, np.uint32))) == out
    seed, step = 0x123456789ABCDEF0, (5 << 32) + 7
    w = TI.random_words(seed, step, 3, 10).view(np.uint32)
    for i in range(10):
        ref = philox_scalar((i // 4, 3, step & 0xFFFFFFFF, step >> 32), (seed & 0xFFFFFFFF, seed >> 32))
        assert int(w[i]) == ref[i % 4]


@pytest.mark.parametrize("impl", [TI.append_flipped, TR.append_flipped], ids=["oracle", "train"])
def test_append_flipped(gold, impl):
    g = gold
    base = [golden_entry(g, i)[0] for i in range(6)]
    both = impl(base, g["widths"])
    assert len(both) == 12 and all(a is b for a, b in zip(both[:6], base))
    for i in range(6, 12):
        ref, _ = golden_entry(g, i)
        assert both[i]["flipped"] is True and np.array_equal(both[i]["gt_classes"], ref["gt_classes"])
        for k in ROW_KEYS:
            assert same_bits(both[i][k], ref[k]), (i, k)
    # the flip of the flip: boxes and keypoints come back (quarter-pixel values: every step is exact)
    rs = np.random.RandomState(0)
    q = lambda *s: (rs.randint(0, 4 * 50, s) / 4.0).astype(np.float32)
    x1 = q(7)
    e = dict(boxes_left=np.stack([x1, q(7), x1 + 5, q(7)], 1), boxes_right=np.stack([x1 - 2, q(7), x1 + 3, q(7)], 1),
             boxes_merge=np.stack([x1 - 2, q(7), x1 + 5, q(7)], 1), kpts=q(7, 6), kpts_right=q(7, 6),
             dim_orien=np.array([[1.5, 1.6, 4.0, t] for t in (0.0, 0.5, -0.5, 2.0, -2.0, 3.0, -3.0)], np.float32),
             gt_classes=np.ones(7, np.int32), flipped=False, index="000123")
    twice = impl(impl([e], [1242])[1:], [1242])[1]
    assert twice["flipped"] is False and twice["index"] == "000123"
    for k in ("boxes_left", "boxes_right", "boxes_merge", "kpts", "kpts_right"):
        assert np.array_equal(twice[k], e[k]), k
    np.testing.assert_allclose(twice["dim_orien"], e["dim_orien"], atol=1e-6)


def test_sampler_order_and_lr_schedule():
    # trainval_net.py:81-101 at batch size 1: randperm(n) * 1 + [0], no leftover, one draw per epoch from one generator
    g, h = torch.Generator().manual_seed(11), torch.Generator().manual_seed(11)
    for _ in range(3):
        want = (torch.randperm(6, generator=h).view(-1, 1) * 1 + torch.arange(0, 1).view(1, 1)).view(-1).tolist()
        got = TR.epoch_order(6, g)
        assert got == want and sorted(got) == list(range(6))
    # trainval_net.py:189-191 with lr_decay_step 5: epochs 6 and 12 decay
    a, b = 1e-3 * 0.1, 1e-3 * 0.1 * 0.1
    want = [(1, 1e-3), (2, 1e-3), (3, 1e-3), (4, 1e-3), (5, 1e-3), (6, a), (7, a), (8, a), (9, a), (10, a), (11, a),
            (12, b), (13, b)]
    assert TR.lr_schedule(1e-3, 1, 13, 5, 0.1) == want
    # resumed after epoch 7 with the lr of epoch 7
    assert TR.lr_schedule(a, 8, 13, 5, 0.1) == want[7:]


@pytest.fixture(scope="module")
def lib():
    from stereo_rcnn_b200 import build
    build.build()
    return L.load()


def test_new_entry_points_reject_bad_arguments(lib):
    def pair(left=FAKE, right=FAKE, H=375, W=1242, scale=1.6, flip=FAKE, ol=FAKE, orr=FAKE):
        return lib.sb_prep_stereo_pair(left, right, H, W, scale, 1, flip, ol, orr, None)

    def gt(B=1, N=64, scale=1.6, width=1987, **null):
        a = [None if ("a%d" % i) in null else FAKE for i in range(14)]
        return lib.sb_train_gt(*a[:8], B, N, scale, width, *a[8:], None)

    def words(step=FAKE, out=FAKE, n=100):
        return lib.sb_random_words(1, step, 0, out, n, None)
    n0 = lib.sb_launch_count()
    bad = {"pair null left": pair(left=None), "pair null right": pair(right=None), "pair null flip": pair(flip=None),
           "pair null out_left": pair(ol=None), "pair null out_right": pair(orr=None), "pair H 0": pair(H=0),
           "pair W 0": pair(W=0), "pair scale 0": pair(scale=0.0), "pair scale < 0": pair(scale=-1.6),
           "pair scale nan": pair(scale=float("nan")), "pair rounds to no rows": pair(H=1, scale=0.25),
           "gt B 0": gt(B=0), "gt N 0": gt(N=0), "gt N 1025": gt(N=1025), "gt scale 0": gt(scale=0.0),
           "gt scale nan": gt(scale=float("nan")), "gt scale inf": gt(scale=float("inf")), "gt width 0": gt(width=0),
           "words null step": words(step=None), "words null out": words(out=None), "words n 0": words(n=0),
           "advance null": lib.sb_step_advance(None, None)}
    bad.update({"gt null pointer %d" % i: gt(**{"a%d" % i: True}) for i in range(14)})
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}
