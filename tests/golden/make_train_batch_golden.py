"""Mint tests/golden/train_batch.npz from the REFERENCE's own Python (run in the build container only).

    python tests/golden/make_train_batch_golden.py

A companion of make_golden.py for the training side of the input pipeline: the reference is imported from where it
lies through oracle/ref_shim.py (runtime shims only, nothing copied), run on a seeded synthetic roidb, and a small
input/output fixture is stored.  The GPU box has no reference checkout; tests there only read the committed fixture.
"""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", ".."))
torch.set_num_threads(1)

from oracle import ref_shim  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def train_batch_goldens():
    """the training side of the input pipeline: the reference's OWN `imdb.append_flipped_images` (imdb.py:117-176),
    `get_minibatch` (minibatch.py:23-131) and `roibatchLoader.__getitem__` (roibatchLoader.py:55-110), imported from
    where they lie, on a synthetic roidb of six entries and their flips.  Three things are supplied from outside:
    `scipy.misc.imread` (gone from scipy) is a lookup into the synthetic frames, the imdb is a subclass that holds the
    roidb and the widths, and cfg.TRAIN.SCALES is (32,) so that the 20x63 frames are scaled by 1.6.  The reference
    shuffles with numpy's global stream; the permutation it drew is recovered from the rows of its output (they are
    unique) and stored, with words that give that permutation under the (word, row index) order."""
    import importlib
    import types
    ref = ref_shim.load()
    cfg = ref.cfg
    f32 = np.float32
    Hf, Wf, N = 20, 63, 40
    rs = np.random.RandomState(12)
    frames = {}
    for i in range(6):
        for side in ("left", "right"):
            base = rs.randint(0, 256, (5, 9, 3)).astype(np.float32)
            im = np.kron(base, np.ones((4, 7, 1), np.float32))[:Hf, :Wf] + rs.randn(Hf, Wf, 3) * 9
            frames["%s%d" % (side, i)] = np.clip(im, 0, 255).astype(np.uint8)            # RGB, as imread gives
    misc = types.ModuleType("scipy.misc")
    misc.imread = lambda path: frames[path].copy()
    sys.modules["scipy.misc"] = misc
    imdb_mod = importlib.import_module("datasets.imdb")
    loader_mod = importlib.import_module("roi_data_layer.roibatchLoader")
    minibatch = importlib.import_module("roi_data_layer.minibatch")

    def entry(n, classes=None, x1_over=(), kpt_edge=False, thetas=None):
        x1 = (rs.rand(n) * 45).astype(f32)
        y1 = (rs.rand(n) * 10).astype(f32)
        bl = np.stack([x1, y1, x1 + 3 + (rs.rand(n) * 12).astype(f32), y1 + 2 + (rs.rand(n) * 7).astype(f32)], 1).astype(f32)
        for r in x1_over:                                   # x1 * 1.6 beyond the blob's width (minibatch.py:50)
            bl[r, 0], bl[r, 2] = 63.5, 64.25
        disp = (1 + rs.rand(n) * 6).astype(f32)
        br = bl.copy()
        br[:, [0, 2]] -= disp[:, None]
        bm = np.stack([np.minimum(bl[:, 0], br[:, 0]), bl[:, 1], np.maximum(bl[:, 2], br[:, 2]), bl[:, 3]], 1).astype(f32)
        do = np.stack([1.4 + 0.01 * np.arange(n) + rs.rand(n) * 0.005, 1.5 + rs.rand(n) * 0.3, 3.5 + rs.rand(n),
                       (rs.rand(n) * 2 - 1) * 3.1], 1).astype(f32)
        if thetas is not None:
            do[:len(thetas), 3] = thetas
        kp = (bl[:, [0]] + rs.rand(n, 6) * (bl[:, [2]] - bl[:, [0]])).astype(f32)
        kp[rs.rand(n, 6) < 0.25] = -1                        # kitti.py marks an invisible keypoint with -1
        if kpt_edge:                                          # k * 1.6 on both sides of 0 and of im_width - 1 = 100
            kp[0] = [-0.5, 0.0, 62.5, 62.6, 0.25, 63.0]
        kpr = kp - np.where(kp >= 0, disp[:, None], 0).astype(f32)
        cls = np.ones(n, np.int32) if classes is None else np.asarray(classes, np.int32)
        return dict(boxes_left=bl, boxes_right=br, boxes_merge=bm, dim_orien=do, kpts=kp.astype(f32),
                    kpts_right=kpr.astype(f32), gt_classes=cls, gt_overlaps=None, flipped=False)

    c38 = np.ones(38, np.int32)
    c38[[4, 17, 30]] = 0
    roidb = [entry(3), entry(38, classes=c38), entry(5, x1_over=(1,), kpt_edge=True),
             entry(8, thetas=[0.0, 0.3, -0.3, 3.5, -3.5, 3.1415927, -3.1415927, 6.0]), entry(4, classes=[0, 0, 0, 0]),
             entry(30)]
    base_n = len(roidb)

    class SynthImdb(imdb_mod.imdb):
        def __init__(self):
            imdb_mod.imdb.__init__(self, "synthetic", ("__background__", "Car"))
            self._roidb, self._image_index = roidb, list(range(base_n))

        def _get_widths(self):
            return [Wf] * base_n

    db = SynthImdb()
    db.append_flipped_images()
    roidb = db.roidb
    assert len(roidb) == 2 * base_n and all(e["flipped"] for e in roidb[base_n:])
    for i, e in enumerate(roidb):                            # what roidb.prepare_roidb adds (roidb.py)
        e["img_left"], e["img_right"] = "left%d" % (i % base_n), "right%d" % (i % base_n)
    scales0 = cfg.TRAIN.SCALES
    cfg.TRAIN.SCALES = (32,)
    loader = loader_mod.roibatchLoader(roidb, np.ones(len(roidb)), np.arange(len(roidb)), 1, 2, training=True)
    E = len(roidb)
    out = dict(frames_left=np.stack([frames["left%d" % i] for i in range(base_n)]),
               frames_right=np.stack([frames["right%d" % i] for i in range(base_n)]), widths=np.array([Wf] * base_n),
               n_rows=np.zeros(E, np.int32), flipped=np.array([e["flipped"] for e in roidb]),
               gt_classes=np.zeros((E, N), np.int32), words=np.zeros((E, N), np.uint32),
               perm=np.full((E, 30), -1, np.int32), num_boxes=np.zeros(E, np.int32), im_info=np.zeros((E, 3), f32),
               blob_entries=np.array([0, 2, 6, 8]), blob_left=[], blob_right=[], blob_sums=np.zeros((E, 2)))
    fields = (("boxes_left", 4), ("boxes_right", 4), ("boxes_merge", 4), ("dim_orien", 4), ("kpts", 6))
    for k, w in fields:
        out[k] = np.zeros((E, N, w), f32)
    out["kpts_right"] = np.zeros((base_n, N, 6), f32)
    names = ("gt_left", "gt_right", "gt_merge", "gt_dim_orien", "gt_kpts")
    for k in names:
        out[k] = np.zeros((E, 30, 6 if k == "gt_kpts" else 5), f32)
    for i, e in enumerate(roidb):
        n = len(e["gt_classes"])
        out["n_rows"][i] = n
        out["gt_classes"][i, :n] = e["gt_classes"]
        for k, _ in fields:
            assert e[k].dtype == np.float32
            out[k][i, :n] = e[k]
        if i < base_n:
            out["kpts_right"][i, :n] = e["kpts_right"]
        np.random.seed(3 + i)
        item = loader[i]
        dl, dr, info = item[0].numpy(), item[1].numpy(), item[2].numpy()
        for k, t in zip(names, item[3:8]):
            out[k][i] = t.numpy()
        nb = int(item[8])
        out["num_boxes"][i], out["im_info"][i] = nb, info
        out["blob_sums"][i] = dl.sum(dtype=np.float64), dr.sum(dtype=np.float64)
        if i in out["blob_entries"]:
            out["blob_left"].append(dl)
            out["blob_right"].append(dr)
        # the permutation: match the shuffled rows against the unshuffled rows of get_minibatch
        b = minibatch.get_minibatch([e], 2)
        rows = np.concatenate((b["gt_boxes_left"], b["gt_boxes_right"], b["gt_boxes_merge"], b["gt_dim_orien"],
                               b["gt_kpts"]), axis=1)
        got = np.concatenate([out[k][i] for k in names], axis=1)
        gt_inds = np.where(e["gt_classes"] != 0)[0]
        assert len(np.unique(rows[:, 15])) == len(rows)
        w = np.zeros(N, np.uint32)
        w[gt_inds] = 0xF0000000 + gt_inds                     # the rows the reference cut off come last
        for pos in range(nb):
            j = np.nonzero((rows == got[pos]).all(1))[0]
            assert len(j) == 1
            out["perm"][i, pos] = gt_inds[j[0]]
            w[gt_inds[j[0]]] = 7919 * pos + 5
        out["words"][i] = w
        print("train batch", i, "flipped" if e["flipped"] else "       ", "rows", n, "num_boxes", nb, "blob", dl.shape)
    cfg.TRAIN.SCALES = scales0
    out["blob_left"], out["blob_right"] = np.stack(out["blob_left"]), np.stack(out["blob_right"])
    np.savez_compressed(os.path.join(HERE, "train_batch.npz"), scale=1.6, **out)
    print("train batch golden written")


if __name__ == "__main__":
    train_batch_goldens()
