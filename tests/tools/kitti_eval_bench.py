"""Times sb_kitti_eval on a seeded synthetic split the size of KITTI val (3769 images, each about four Cars, a Van, a
Pedestrian, two DontCare rows and about 30 detections) and the oracle (oracle/kitti_eval.py, sequential Python on
one host core) on the same data, checks that they agree, and prints one JSON line with the card's name and power
limit read in the same run.

    python tests/tools/kitti_eval_bench.py [--images 3769] [--reps 20] [--no-oracle]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import kitti_eval as O                      # noqa: E402
from stereo_rcnn_b200 import kitti_eval as K            # noqa: E402
from stereo_rcnn_b200 import ops as G                   # noqa: E402
from stereo_rcnn_b200 import synth                      # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=3769)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--no-oracle", action="store_true")
    a = ap.parse_args()
    t0 = time.perf_counter()
    ev = K.KittiEval("cuda")
    for g, d in synth.kitti_split(a.images, seed=2017):
        ev.add(g, d)
    parse_s = time.perf_counter() - t0
    bars = ev.bars
    (gt, gc, det, dc, go, do, po), n_pairs = ev.device_inputs()
    L = G._l.load()
    n_img, ng, nd = go.numel() - 1, gc.numel(), dc.numel()
    out = G.kitti_eval(gt, gc, det, dc, go, do, po, n_pairs, bars)        # warm-up
    ov = torch.empty(3, n_pairs, dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn):
        fn()
        ev0.record()
        for _ in range(a.reps):
            fn()
        ev1.record()
        torch.cuda.synchronize()
        return ev0.elapsed_time(ev1) * 1e3 / a.reps

    s = G.stream_ptr()
    ov_us = timed(lambda: L.sb_kitti_overlaps(G.ptr(gt), G.ptr(gc), G.ptr(det), G.ptr(go), G.ptr(do), G.ptr(po),
                                              n_img, n_pairs, G.ptr(ov[0]), G.ptr(ov[1]), G.ptr(ov[2]), s))
    total_us = timed(lambda: G.kitti_eval(gt, gc, det, dc, go, do, po, n_pairs, bars, out=out))
    # per-stage device times: a profile of `reps` calls, in a run of its own after the timed window
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.reps):
            G.kitti_eval(gt, gc, det, dc, go, do, po, n_pairs, bars, out=out)
        torch.cuda.synchronize()
    stages = {}
    for e in prof.key_averages():
        for k in ("overlaps_kernel", "match_tp_kernel", "thresholds_scan_kernel", "thresholds_rank_kernel",
                  "match_curve_kernel", "curves_kernel"):
            if k in e.key:
                stages[k.replace("_kernel", "")] = round(e.device_time_total / a.reps, 1)
    res = dict(metric="kitti_eval", images=n_img, gt_rows=ng, det_rows=nd, pairs=n_pairs,
               configurations=9 * len(bars), device_us=round(total_us, 1), overlaps_us=round(ov_us, 1),
               stage_us=stages, host_parse_pack_s=round(parse_s, 2), card=card())
    got = {k: v.cpu().numpy() for k, v in out.items() if k != "_buffer"}
    res["ap_3d_07_R11"] = [round(float(v), 4) for v in got["ap"][2 * len(bars) * 3:2 * len(bars) * 3 + 3, 0]]
    if not a.no_oracle:
        images = [(g, gcs, d, dcs) for gcs, g, dcs, d in ev.images]
        t0 = time.perf_counter()
        ref = O.evaluate(images, bars)
        res["oracle_s"] = round(time.perf_counter() - t0, 2)
        exact = all(np.array_equal(got[k], ref[k]) for k in ("thresholds", "n_thresholds", "tp", "fp", "fn",
                                                            "precision", "recall", "n_gt"))
        exact = exact and np.array_equal(got["ap"][:, :2], ref["ap"][:, :2])
        close = all(np.allclose(got[k], ref[k], rtol=1e-12, atol=1e-12) for k in ("sim", "aos", "ap"))
        res["parity"] = bool(exact and close)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
