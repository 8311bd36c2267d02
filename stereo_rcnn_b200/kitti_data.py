"""The training roidb of a KITTI split, built on the device: what the reference's kitti.gt_roidb and
combined_roidb('kitti_train') hand its training loop, from root/training/{label_2,calib,image_2,image_3}.

* `annotations`  : the reference's gt_roidb entries (kitti_utils.read_obj_data, kitti.remove_occluded_keypoints for the
                   left and the right camera, kitti._load_kitti_annotation), one per image id, in order.
* `train_roidb`  : annotations, then train.append_flipped, the keys of roidb.prepare_roidb and roidb.filter_roidb;
                   its output goes straight into train.fit.

Reading the label and calibration texts and the PNG headers is host work (kitti_eval.read_objects,
ops.read_calibration); the projections, the occlusion reasoning and the filter run in sb_kitti_annotations, one CTA
per image, with one host-to-device copy of the packed split and one device-to-host copy of the results.  Images are
not decoded: (H, W) come from the PNG header, as the reference needs nothing else of the left image.  DESIGN.md §10
states the numerics.
"""
import math
import os

import numpy as np
import torch

from . import ops
from .kitti_eval import read_objects

USED_TYPES = ("Car", "Van", "Truck", "Misc")     # kitti_utils.read_obj_data's used_cls; only Car is kept
PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"
OUT_FIELDS = (("boxes_left", 0, 4), ("boxes_right", 4, 8), ("boxes_merge", 8, 12), ("dim_orien", 12, 16),
              ("kpts", 16, 22), ("kpts_right", 22, 28))


def png_size(path):
    """(H, W) of a PNG file from its IHDR chunk (bytes 16-23), without decoding it; anything else raises ValueError
    naming the file"""
    with open(path, "rb") as f:
        head = f.read(24)
    if len(head) < 24 or head[:8] != PNG_SIGNATURE or head[12:16] != b"IHDR":
        raise ValueError("%s is not a PNG file (the image size is read from the PNG header)" % path)
    w, h = int.from_bytes(head[16:20], "big"), int.from_bytes(head[20:24], "big")
    if w < 1 or h < 1:
        raise ValueError("%s: the PNG header gives a %dx%d image" % (path, w, h))
    return h, w


def _need(path, what, image_id):
    if not os.path.isfile(path):
        raise FileNotFoundError("no %s for image %s: %s" % (what, image_id, path))
    return path


def pack_image(label_text, calib, label_name="<text>"):
    """one image's label text and ops.Calibration -> (rows float64 [n,11], codes int32 [n], calib float64 [25],
    line numbers [n] of the used label lines).  Only Car, Van, Truck and Misc lines are used; ori = ry + pi/2 and its
    cosine and sine are Python floats (math, as the reference)."""
    try:
        types, vals = read_objects(label_text + "\n")
    except ValueError as e:
        raise ValueError(str(e).replace("<text>", label_name, 1)) from None
    line_no = [n for n, line in enumerate(label_text.splitlines(), 1) if line.split()]
    rows, codes, lines = [], [], []
    for t, v, n in zip(types, vals.tolist(), line_no):
        if t not in USED_TYPES:
            continue
        ori = v[13] + math.pi / 2
        rows.append([v[0], v[1], v[2], v[8], v[7], v[9], v[10], v[11], v[12], math.cos(ori), math.sin(ori)])
        codes.append(0 if t == "Car" else 1)
        lines.append(n)
    p2_2, p2_3 = calib.p2.copy(), calib.p3.copy()
    p2_2[0, 3] = calib.p2[0, 3] - calib.p2[0, 3]
    p2_3[0, 3] = calib.p3[0, 3] - calib.p2[0, 3]
    cal = np.concatenate([p2_2.reshape(-1), p2_3.reshape(-1), [calib.t_cam2_cam0_x]]).astype(np.float64)
    return (np.array(rows, np.float64).reshape(-1, ops.KITTI_ANN_IN), np.array(codes, np.int32), cal,
            np.array(lines, np.int64))


class Split(object):
    """a KITTI split packed for sb_kitti_annotations (host arrays): rows, codes, obj_off, calib, image_hw, and per
    image its id, label path, used label line numbers and image paths"""

    def __init__(self, root, image_ids):
        self.root, self.ids = root, [str(i) for i in image_ids]
        if not self.ids:
            raise ValueError("no image ids")
        rows, codes, cals, hws, self.lines, self.paths = [], [], [], [], [], []
        for i in self.ids:
            d = os.path.join(root, "training")
            lab = _need(os.path.join(d, "label_2", i + ".txt"), "label file", i)
            cpath = _need(os.path.join(d, "calib", i + ".txt"), "calibration file", i)
            left = _need(os.path.join(d, "image_2", i + ".png"), "left image", i)
            right = _need(os.path.join(d, "image_3", i + ".png"), "right image", i)
            with open(lab) as f:
                text = f.read()
            try:
                cal = ops.read_calibration(cpath)
            except ValueError as e:
                raise ValueError("%s: %s" % (cpath, e)) from None
            hw = png_size(left)
            r, c, k, ln = pack_image(text, cal, lab)
            rows.append(r)
            codes.append(c)
            cals.append(k)
            hws.append(hw)
            self.lines.append(ln)
            self.paths.append((lab, left, right))
        self.rows = np.concatenate(rows).reshape(-1, ops.KITTI_ANN_IN)
        self.codes = np.concatenate(codes).astype(np.int32)
        self.obj_off = np.concatenate([[0], np.cumsum([len(c) for c in codes])]).astype(np.int64)
        self.calib = np.stack(cals).astype(np.float64)
        self.image_hw = np.array(hws, np.int32).reshape(-1, 2)

    def arrays(self):
        return self.rows, self.codes, self.obj_off, self.calib, self.image_hw

    def to_device(self, device):
        """the packed split in one device buffer (one host-to-device copy) -> tensor views in arrays()' order"""
        arrs = self.arrays()
        segs, o = [], 0
        for a in arrs:
            segs.append(o)
            o += (a.nbytes + 7) // 8 * 8
        host = np.zeros(max(o, 8), np.uint8)
        for s, a in zip(segs, arrs):
            host[s:s + a.nbytes] = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
        buf = torch.from_numpy(host).to(device)
        dt = {np.dtype(np.float64): torch.float64, np.dtype(np.int64): torch.int64, np.dtype(np.int32): torch.int32}
        return [buf[s:s + (a.nbytes + 7) // 8 * 8].view(dt[a.dtype])[:a.size].view(a.shape) for s, a in zip(segs, arrs)]

    def outputs(self, device):
        """the output tensors of sb_kitti_annotations as views into one device buffer (one device-to-host copy)"""
        n, ni = len(self.codes), len(self.ids)
        buf = torch.zeros(n * ops.KITTI_ANN_OUT + 2 * ni, dtype=torch.float32, device=device)
        out = buf[:n * ops.KITTI_ANN_OUT].view(n, ops.KITTI_ANN_OUT)
        ints = buf[n * ops.KITTI_ANN_OUT:].view(torch.int32)
        return buf, (out, ints[:ni], ints[ni:])

    def check_status(self, status):
        """raise for the first image the reference cannot read"""
        for k, s in enumerate(np.asarray(status).tolist()):
            if s > 0:
                lab = self.paths[k][0]
                raise ValueError("image %s: the box of the object on line %d of %s reaches past column %d of the "
                                 "depth line; the reference raises IndexError here"
                                 % (self.ids[k], int(self.lines[k][s - 1]), lab, ops.KITTI_DEPTH_COLS - 1))
            if s != 0:
                raise ValueError("image %s: status %d of sb_kitti_annotations" % (self.ids[k], s))

    def entries(self, out, n_kept):
        """the reference's gt_roidb dicts from the host copies of out [n,30] and n_kept"""
        res = []
        for k in range(len(self.ids)):
            a = int(self.obj_off[k])
            r = out[a:a + int(n_kept[k])]
            e = {name: r[:, lo:hi].copy() for name, lo, hi in OUT_FIELDS}
            e["truncation"], e["occlusion"] = r[:, 28].copy(), r[:, 29].copy()
            e["gt_classes"] = np.ones(len(r), np.int32)
            e["flipped"] = False
            res.append(e)
        return res


def run(split, device):
    """sb_kitti_annotations over a Split: one copy in, one launch, one copy out -> (out [n,30], n_kept, status) numpy"""
    dev = torch.device(device)
    with torch.cuda.device(dev):
        views = split.to_device(dev)
        buf, out = split.outputs(dev)
        ops.kitti_annotations(*views, out=out)
        host = buf.cpu().numpy()
    n, ni = len(split.codes), len(split.ids)
    ints = host[n * ops.KITTI_ANN_OUT:].view(np.int32)
    return host[:n * ops.KITTI_ANN_OUT].reshape(n, ops.KITTI_ANN_OUT), ints[:ni], ints[ni:]


def annotations(root, image_ids, device):
    """the reference's gt_roidb (kitti.py:118-279) for root/training/{label_2,calib,image_2,image_3}/<id> -> one dict
    per image id, in order: boxes_left, boxes_right, boxes_merge [n,4], dim_orien [n,4] (w, h, l, alpha), kpts,
    kpts_right [n,6] (four keypoints, visible left, visible right), truncation, occlusion [n] float32, gt_classes [n]
    int32 (1, Car), flipped False.  The sparse gt_overlaps / subclass keys, which training does not read, are left
    out.  An image the reference would stop on (a box past column 1259 of its depth line, or entirely behind the
    camera) raises ValueError naming the image and the label line."""
    split = Split(root, image_ids)
    out, n_kept, status = run(split, device)
    split.check_status(status)
    return split.entries(out, n_kept)


def prepare(roidb, split, n_base):
    """roidb.prepare_roidb's keys: img_left, img_right, width, height (entry k and its flip share image k % n_base)"""
    for k, e in enumerate(roidb):
        j = k % n_base
        _lab, left, right = split.paths[j]
        e["img_left"], e["img_right"] = left, right
        e["height"], e["width"] = int(split.image_hw[j, 0]), int(split.image_hw[j, 1])
        e["image_id"] = split.ids[j]
    return roidb


def filter_roidb(roidb):
    """roidb.filter_roidb: drop the entries without rows, keep the order"""
    return [e for e in roidb if len(e["boxes_left"]) and len(e["boxes_right"]) and len(e["boxes_merge"])]


def train_roidb(root, image_ids, device, flipped=True):
    """what combined_roidb('kitti_train') hands trainval_net.py (roidb.py:88-131): annotations, then (with flipped,
    cfg.TRAIN.USE_FLIPPED) train.append_flipped with the left images' widths, prepare_roidb's keys (plus image_id)
    and filter_roidb.  Feed it to train.fit with frames(entry) decoding entry["img_left"] / entry["img_right"]."""
    from .train import append_flipped
    split = Split(root, image_ids)
    out, n_kept, status = run(split, device)
    split.check_status(status)
    roidb = split.entries(out, n_kept)
    n = len(roidb)
    if flipped:
        roidb = append_flipped(roidb, [int(w) for w in split.image_hw[:, 1]])
    return filter_roidb(prepare(roidb, split, n))
