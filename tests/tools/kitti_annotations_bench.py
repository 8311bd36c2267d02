"""Time building the training roidb of a KITTI-train-sized synthetic split (3712 images at 375x1242 and 370x1224):
host parsing, the host-to-device copy, sb_kitti_annotations (CUDA events, warmed up, mean of 20 calls), the
device-to-host copy and assembling the dicts, and the sequential oracle on one host core for comparison.

    python tests/tools/kitti_annotations_bench.py [--images 3712] [--seed 0]

Lives under tests/tools because it imports the oracle.  Writes the split to a temporary directory; prints the card
and its power limit with the numbers, and one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", ".."))

from oracle import kitti_annotations as OA  # noqa: E402
from stereo_rcnn_b200 import kitti_data as KD  # noqa: E402
from stereo_rcnn_b200 import ops  # noqa: E402
from stereo_rcnn_b200 import synth  # noqa: E402


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=3712)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    torch.set_num_threads(1)
    dev = torch.device("cuda")
    res = {"card": torch.cuda.get_device_name(dev), "power_limit": power_limit(), "images": a.images}
    with tempfile.TemporaryDirectory() as root:
        ids = synth.kitti_folder(root, a.images, a.seed)
        t = time.perf_counter()
        split = KD.Split(root, ids)
        res["host_parse_ms"] = (time.perf_counter() - t) * 1e3
    res["rows"] = int(len(split.codes))
    torch.cuda.synchronize()
    t = time.perf_counter()
    views = split.to_device(dev)
    torch.cuda.synchronize()
    res["h2d_ms"] = (time.perf_counter() - t) * 1e3
    buf, out = split.outputs(dev)
    for _ in range(3):
        ops.kitti_annotations(*views, out=out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        ops.kitti_annotations(*views, out=out)
    e1.record()
    torch.cuda.synchronize()
    res["kernel_ms"] = e0.elapsed_time(e1) / 20
    t = time.perf_counter()
    host = buf.cpu().numpy()
    res["d2h_ms"] = (time.perf_counter() - t) * 1e3
    n, ni = len(split.codes), len(split.ids)
    o = host[:n * ops.KITTI_ANN_OUT].reshape(n, ops.KITTI_ANN_OUT)
    ints = host[n * ops.KITTI_ANN_OUT:].view(np.int32)
    t = time.perf_counter()
    split.check_status(ints[ni:])
    entries = split.entries(o, ints[:ni])
    res["assemble_ms"] = (time.perf_counter() - t) * 1e3
    res["kept_rows"] = int(sum(len(e["gt_classes"]) for e in entries))
    t = time.perf_counter()
    oo, on, ost = OA.split(*split.arrays())
    res["oracle_one_core_ms"] = (time.perf_counter() - t) * 1e3
    res["agree"] = bool(np.array_equal(oo.view(np.uint32), o.view(np.uint32)) and np.array_equal(on, ints[:ni]) and
                        np.array_equal(ost, ints[ni:]))
    print("%s at %s, %d images, %d used rows, %d kept" % (res["card"], res["power_limit"], a.images, res["rows"],
                                                          res["kept_rows"]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
