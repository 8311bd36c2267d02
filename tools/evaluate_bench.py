#!/usr/bin/env python
"""The test loop over a split (pipeline.evaluate) at KITTI frame sizes; one JSON line.

    python tools/evaluate_bench.py [--pairs 60] [--other 12]
    python -m torch.distributed.run --nproc-per-node N tools/evaluate_bench.py [--pairs 60] [--other 12]

A synthetic split of `--other` pairs at 370x1224 followed by `--pairs` pairs at 375x1242 (target size 600: blobs of
600x1985 and 600x1987), with the three calibrations of tests/golden/calibration.npz in turn.  The weights are
synth.make_state_dict(3) with the Car score biased up so that every image carries detections through the solver
stage.  Frames come from a small pool made before the timed runs, so the frames callback costs nothing here (a real
loop decodes PNGs there).  The 370x1224 pairs come first, so every (frame shape, slot) graph is captured in the first
entries.

Reports pairs/s of evaluate at inflight 1, 2 and 3 (one throughput=True pipeline), each over the
whole call (graph captures included) and in the steady state (from the frames call of the first entry after the
captures to the end of the call); next to them the eager per-pair loop a user would otherwise write
(step_with_solver on prepared blobs with host P2 / P3, results read back per pair); the host seconds spent writing
files; peak allocated device memory and the graphs of each run; and the card's name and power limit read in the same
run.  Result files go to a temporary directory that is removed afterwards.

Under torch.distributed.run (one process per GPU, NCCL) every rank evaluates its shard of the same split
(evaluate(world=N, dist=...)); the line then reports images/s of the whole sharded call with and without labels
(kitti_split's seeded label texts), next to each rank's loop seconds and rank 0's seconds in the end-of-loop gather,
in writing the files and in scoring.  At one process the same two runs go through the one-rank path, where the
writing and the scoring run inside the loop.  Rank 0 prints the line.
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

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from stereo_rcnn_b200 import ops, pipeline  # noqa: E402
from stereo_rcnn_b200.synth import kitti_split, make_state_dict  # noqa: E402

SHAPES = {"kitti": (375, 1242), "other": (370, 1224)}
CAL = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests", "golden", "calibration.npz")
POOL = 4


def frame(h, w, seed):
    rs = np.random.RandomState(seed)
    base = rs.randint(0, 256, (h // 8 + 2, w // 8 + 2, 3)).astype(np.float32)
    im = np.kron(base, np.ones((8, 8, 1), np.float32))[:h, :w] + rs.randn(h, w, 3) * 6
    return np.clip(im, 0, 255).astype(np.uint8)


def make_split(n_kitti, n_other):
    g = np.load(CAL)
    cals = [ops.read_calibration(str(t)) for t in g["texts"]]
    pool = {}
    for name, (h, w) in SHAPES.items():
        for s in range(POOL):
            left = frame(h, w + 12, 1000 * len(name) + s)
            pool[name, s] = (np.ascontiguousarray(left[:, 12:]), np.ascontiguousarray(left[:, :w]))
    entries = [dict(image_id="%06d" % k, shape="other" if k < n_other else "kitti", pool=k % POOL, cal=k % len(cals))
               for k in range(n_other + n_kitti)]
    return entries, pool, cals


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                               "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        return None


def run_evaluate(pipe, entries, pool, cals, inflight, steady_from):
    stamps = {}

    def frames(e):
        k = int(e["image_id"])
        stamps.setdefault(k, time.perf_counter())
        return pool[e["shape"], e["pool"]]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    with tempfile.TemporaryDirectory() as d:
        t0 = time.perf_counter()
        s = pipeline.evaluate(pipe, entries, frames, lambda e: cals[e["cal"]], d, inflight=inflight, log=lambda m: None)
        t1 = time.perf_counter()
    n = len(entries)
    return dict(pairs_per_s=round(n / (t1 - t0), 2),
                steady_pairs_per_s=round((n - steady_from) / (t1 - stamps[steady_from]), 2),
                write_s=round(s["write_s"], 4), graphs=s["graphs"], lines=s["lines"], files=s["files"],
                peak_alloc_gb=round(torch.cuda.max_memory_allocated() / 2 ** 30, 2))


def run_split(pipe, entries, pool, cals, labels, world, dist, inflight=2):
    """one evaluate over the split, sharded over the ranks at world > 1; host clock from a barrier to the return"""
    lab = None if labels is None else (lambda e: labels[int(e["image_id"]) % len(labels)])
    with tempfile.TemporaryDirectory() as d:
        torch.cuda.synchronize()
        if world > 1:
            dist.barrier()
        t0 = time.perf_counter()
        s = pipeline.evaluate(pipe, entries, lambda e: pool[e["shape"], e["pool"]], lambda e: cals[e["cal"]], d,
                              inflight=inflight, log=lambda m: None, labels=lab, world=world, dist=dist)
        t1 = time.perf_counter()
    out = dict(images_per_s=round(len(entries) / (t1 - t0), 2), call_s=round(t1 - t0, 3), inflight=inflight,
               graphs=s["graphs"], files=s["files"])
    for k in ("gather_s", "write_s", "score_s"):
        if k in s:
            out[k] = round(s[k], 4)
    if "loop_s" in s:
        out["loop_s"] = [round(t, 3) for t in s["loop_s"]]
        out["rank_images"] = s["rank_images"]
    if "ap" in s:
        out["car_ap_r11_moderate_2d"] = round(float(s["ap"]["bbox"][0.7][1, 0]), 2)
    return out


def run_eager(pipe, entries, pool, cals):
    """the per-pair loop without evaluate: blobs prepared beforehand, step_with_solver with host P2 / P3, results read
    back per pair (what writing the files needs)"""
    flip = torch.zeros(1, dtype=torch.int32, device="cuda")
    blobs = {}
    for (name, s), (left, right) in pool.items():
        hw = SHAPES[name]
        bl, br = ops.prep_stereo_pair(torch.from_numpy(left).cuda(), torch.from_numpy(right).cuda(),
                                      pipeline.frame_scale(hw), flip, rgb_input=True)
        blobs[name, s] = (bl[None], br[None])

    def one(e):
        hw, c = SHAPES[e["shape"]], cals[e["cal"]]
        out = pipe.step_with_solver(*blobs[e["shape"], e["pool"]], c.p2, c.p3, hw,
                                    scale=np.float32(pipeline.frame_scale(hw)))
        return int(out["n_solved"].item()), out["final"].cpu()
    for e in entries[:6]:
        one(e)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    solved = [one(e)[0] for e in entries]
    t1 = time.perf_counter()
    return dict(pairs_per_s=round(len(entries) / (t1 - t0), 2), mean_n_solved=round(float(np.mean(solved)), 2))


def run(args):
    world = int(os.environ.get("WORLD_SIZE", "1"))
    dist = None
    if world > 1:
        import torch.distributed as dist
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", 0)))
        dist.init_process_group("nccl", device_id=torch.device("cuda", torch.cuda.current_device()))
    dev = torch.device("cuda", torch.cuda.current_device())
    sd = make_state_dict(3)
    b = sd["RCNN_cls_score.bias"].clone()
    b[1] += 4.0
    sd["RCNN_cls_score.bias"] = b
    entries, pool, cals = make_split(args.pairs, args.other)
    labels = [t for t, _d in kitti_split(16, seed=7)]
    steady_from = args.other + 6                           # every (shape, slot) graph exists from here on
    res = {}
    with torch.no_grad():
        pipe = pipeline.StereoPipeline(sd, dev, throughput=True)
        if world == 1:
            res = {"inflight%d" % k: run_evaluate(pipe, entries, pool, cals, k, steady_from) for k in (1, 2, 3)}
            res["eager_step_with_solver"] = run_eager(pipe, entries, pool, cals)
        run_split(pipe, entries[:2 * world], pool, cals, None, world, dist)        # loads the modules on every rank
        res["split_no_labels"] = run_split(pipe, entries, pool, cals, None, world, dist)
        res["split_labels"] = run_split(pipe, entries, pool, cals, labels, world, dist)
    if world > 1:
        rank = dist.get_rank()
        dist.destroy_process_group()
        if rank:
            return
    print(json.dumps({
        "metric": "evaluate_pairs_per_s" if world == 1 else "evaluate_images_per_s_sharded",
        "value": res["inflight1"]["steady_pairs_per_s"] if world == 1 else res["split_no_labels"]["images_per_s"],
        "unit": "pairs/s", "higher_is_better": True, "gpus": world, "pairs": len(entries),
        "frames": {k: [sum(e["shape"] == k for e in entries), list(v)] for k, v in SHAPES.items()},
        "calibrations": len(cals), "gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit(), **res}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=60, help="pairs at 375x1242")
    ap.add_argument("--other", type=int, default=12, help="pairs at 370x1224, first in the split")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
