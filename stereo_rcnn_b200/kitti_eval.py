"""KITTI average precision of a split, Car only: what the KITTI object devkit's evaluate_object reports (2D boxes,
orientation (AOS), bird's-eye view (BEV) and 3D, at easy / moderate / hard, AP|R11 and AP|R40), computed by
sb_kitti_eval on the device.  DESIGN.md §9 is the restatement of the devkit it follows.

* `read_objects`  : a KITTI label file (15 fields per line) or result file (16, the last the score) -> (types, rows).
* `KittiEval`     : add() one image's labels and results at a time, result() scores the split in one device call.
* `evaluate_dirs` : the devkit's job over directories: label_dir/<id>.txt and result_dir/data/<id>.txt.

Parsing text and packing rows is host work; the overlaps, the matchings, the thresholds and the curves run on the
device, with one host-to-device copy of the packed split and one device-to-host copy of the results.
"""
import math
import os

import numpy as np
import torch

from . import ops

METRICS = ("bbox", "bev", "3d")                   # the devkit's order of eval_class calls
DIFFICULTIES = ("easy", "moderate", "hard")
TYPE_CODES = {"Car": 0, "Van": 1, "DontCare": 2}  # relative to Car; every other type is 3


def read_objects(path_or_text):
    """parse a KITTI label or result file, given as a path or as its text (anything with a line break, or "") ->
    (types: list of str, rows: float64 [n, 15]) with the fields trunc, occ, alpha, x1, y1, x2, y2, h, w, l, x, y, z,
    ry, score; score is NaN on label lines (15 fields).  A line with another field count, a field that is not a finite
    number, or a mix of label and result lines raises ValueError naming the file and the line."""
    text, name = path_or_text, "<text>"
    if path_or_text != "" and "\n" not in path_or_text:
        name = path_or_text
        with open(path_or_text) as f:
            text = f.read()
    types, rows, width = [], [], None
    for n, line in enumerate(text.splitlines(), 1):
        tok = line.split()
        if not tok:
            continue
        if len(tok) not in (15, 16) or (width is not None and len(tok) != width):
            raise ValueError("%s line %d: %d fields; a label line has 15 and a result line 16, one kind per file"
                             % (name, n, len(tok)))
        width = len(tok)
        try:
            vals = [float(v) for v in tok[1:]]
        except ValueError:
            raise ValueError("%s line %d: a field after the type is not a number: %r" % (name, n, line)) from None
        if not all(math.isfinite(v) for v in vals):
            raise ValueError("%s line %d: a field is not finite: %r" % (name, n, line))
        types.append(tok[0])
        rows.append(vals + [math.nan] * (15 - len(vals)))
    return types, np.array(rows, np.float64).reshape(-1, 15)


def pack_rows(types, rows, scored):
    """(types, rows [n,15]) -> (codes int32 [n], the device rows float64 [n,16]: trunc, occ, alpha, x1, y1, x2, y2, h, w,
    l, x, y, z, cos(ry), sin(ry), score (0 unless scored))"""
    rows = np.asarray(rows, np.float64).reshape(-1, 15)
    codes = np.array([TYPE_CODES.get(t, 3) for t in types], np.int32)
    out = np.zeros((len(rows), ops.KITTI_ROW), np.float64)
    out[:, :13] = rows[:, :13]
    out[:, 13], out[:, 14] = np.cos(rows[:, 13]), np.sin(rows[:, 13])
    if scored:
        out[:, 15] = rows[:, 14]
    return codes, out


def _objects(x):
    return x if isinstance(x, tuple) else read_objects(x)


class KittiEval(object):
    """Scores a split image by image as the devkit's evaluate_object does (Car): add() every image, then result().
    min_overlaps: the IoU bars, each used for the 2D, BEV and 3D metrics (up to four)."""

    def __init__(self, device, min_overlaps=(0.7, 0.5)):
        self.device = torch.device(device)
        self.bars = tuple(float(b) for b in min_overlaps)
        if not 1 <= len(self.bars) <= 4 or not all(0.0 <= b <= 1.0 for b in self.bars):
            raise ValueError("min_overlaps: one to four bars in [0, 1]")
        self.images = []

    def add(self, gt, det):
        """one image: its labels and its results, each as text, a path, or read_objects' (types, rows)"""
        gt_types, gt_rows = _objects(gt)
        det_types, det_rows = _objects(det)
        if np.isnan(det_rows[:, 14]).any():
            raise ValueError("a detection has no score (a label line among the results)")
        self.images.append(pack_rows(gt_types, gt_rows, False) + pack_rows(det_types, det_rows, True))

    def packed(self):
        """the split in the device layout, as numpy arrays: gt rows, gt codes, det rows, det codes, gt_off, det_off,
        pair_off"""
        ng = np.array([len(c) for c, _r, _dc, _dr in self.images], np.int64)
        nd = np.array([len(dc) for _c, _r, dc, _dr in self.images], np.int64)
        off = [np.concatenate([[0], np.cumsum(v)]).astype(np.int64) for v in (ng, nd, ng * nd)]
        gt = np.concatenate([r for _c, r, _dc, _dr in self.images]).reshape(-1, ops.KITTI_ROW)
        gc = np.concatenate([c for c, _r, _dc, _dr in self.images]).astype(np.int32)
        det = np.concatenate([dr for _c, _r, _dc, dr in self.images]).reshape(-1, ops.KITTI_ROW)
        dc = np.concatenate([dc for _c, _r, dc, _dr in self.images]).astype(np.int32)
        return gt, gc, det, dc, off[0], off[1], off[2]

    def device_inputs(self):
        """packed() in one device buffer (one host-to-device copy) -> (tensor views in packed()'s order, n_pairs)"""
        arrs = self.packed()
        segs, o = [], 0
        for a in arrs:
            n = (a.nbytes + 7) // 8 * 8
            segs.append((o, a))
            o += n
        host = np.zeros(max(o, 8), np.uint8)
        for s, a in segs:
            host[s:s + a.nbytes] = a.view(np.uint8).reshape(-1)
        buf = torch.from_numpy(host).to(self.device)
        views = []
        for (s, a) in segs:
            t = torch.float64 if a.dtype == np.float64 else (torch.int64 if a.dtype == np.int64 else torch.int32)
            views.append(buf[s:s + (a.nbytes + 7) // 8 * 8].view(t)[:a.size].view(a.shape))
        return views, int(arrs[6][-1])

    def result(self):
        """score the split -> {"bbox" | "aos" | "bev" | "3d": {bar: float64 [3 difficulties, 2 (AP|R11, AP|R40)]},
        "n_gt": int [3], "curves": {"bbox" | "bev" | "3d": {bar: {thresholds, n_thresholds, tp, fp, fn, sim,
        precision, recall, aos: arrays with a leading difficulty axis}}}}.  AOS comes from the 2D matching."""
        if not self.images:
            raise ValueError("no images to evaluate")
        (gt, gc, det, dc, goff, doff, poff), n_pairs = self.device_inputs()
        with torch.cuda.device(self.device):
            out = ops.kitti_eval(gt, gc, det, dc, goff, doff, poff, n_pairs, self.bars)
            host = out["_buffer"].cpu()
        res = ops.kitti_eval_outputs(len(self.bars), "cpu")
        res["_buffer"].copy_(host)
        nb = len(self.bars)
        table = {k: {} for k in ("bbox", "aos", "bev", "3d")}
        curves = {k: {} for k in METRICS}
        for m, metric in enumerate(METRICS):
            for b, bar in enumerate(self.bars):
                c = slice((m * nb + b) * 3, (m * nb + b) * 3 + 3)
                ap = res["ap"][c].numpy()
                table[metric][bar] = ap[:, 0:2].copy()
                if metric == "bbox":
                    table["aos"][bar] = ap[:, 2:4].copy()
                curves[metric][bar] = {k: res[k][c].numpy().copy() for k, _t, _n in ops.KITTI_OUTPUTS
                                       if k not in ("ap", "n_gt")}
        table["n_gt"] = res["n_gt"][0:3].numpy().copy()
        table["curves"] = curves
        return table


def evaluate_dirs(label_dir, result_dir, image_ids, device, min_overlaps=(0.7, 0.5)):
    """The devkit's evaluation over directories: label_dir/<id>.txt (a missing one is an error) and
    result_dir/data/<id>.txt (a missing one means no detections), the layout pipeline.evaluate writes.
    -> KittiEval.result()"""
    ev = KittiEval(device, min_overlaps)
    for i in image_ids:
        lab = os.path.join(label_dir, "%s.txt" % i)
        if not os.path.isfile(lab):
            raise FileNotFoundError("no label file for image %s: %s" % (i, lab))
        res = os.path.join(result_dir, "data", "%s.txt" % i)
        ev.add(lab, res if os.path.isfile(res) else "")
    return ev.result()
