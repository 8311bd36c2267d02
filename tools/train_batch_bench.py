#!/usr/bin/env python
"""The data-parallel training step at B stereo pairs per GPU (SURVEY §8d config 4: trainval_net.py's step, batch 16
over 8 GPUs = 2 pairs per GPU); one JSON line from rank 0.

    python -m torch.distributed.run --nproc-per-node N tools/train_batch_bench.py --pairs-per-gpu B \
        [--steps K] [--warmup W] [--fit-shapes S]

Each rank trains on B synthetic 375x1242 camera frame pairs (600x1987 blobs) with 8 ground-truth boxes per image
through Trainer.step_from_frames: replayed from a CUDA graph at one rank, eager at several (what train.fit runs).
Reports global pairs/s and ms per step (CUDA events, the slowest rank), the gradient all-reduce alone
(GradientBuckets.all_reduce over the trainer's own buckets, CUDA events), the peak allocated memory of every rank,
the skip count, and the card's name and power limit read in the same run.  --fit-shapes S (one rank only) adds the
peak memory of one train.fit epoch over S KITTI frame shapes, two batches each: the engine keeps workspaces and a
captured step per shape, so this is what decides whether B pairs fit on the card.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from stereo_rcnn_b200 import train  # noqa: E402
from stereo_rcnn_b200.engine import GraphRunner, StereoRCNNEngine  # noqa: E402
from stereo_rcnn_b200.parallel import max_over_ranks  # noqa: E402
from stereo_rcnn_b200.synth import make_state_dict  # noqa: E402

FRAME = (375, 1242)
KITTI_SHAPES = [(375, 1242), (370, 1224), (374, 1238), (376, 1241)]
N_BOXES = 8


def entry(hw, seed, index):
    """a roidb entry of an hw frame with N_BOXES cars (boxes in frame pixels, the right box 20 px to the left)"""
    H, W = hw
    rs = np.random.RandomState(seed)
    f = np.float32
    w, h = rs.uniform(60, 240, N_BOXES), rs.uniform(40, 150, N_BOXES)
    x1, y1 = rs.uniform(30, W - w - 1), rs.uniform(120, H - h - 1)
    bl = np.stack([x1, y1, x1 + w, y1 + h], 1).astype(f)
    br = bl.copy()
    br[:, [0, 2]] -= f(20)
    bm = np.stack([br[:, 0], bl[:, 1], bl[:, 2], bl[:, 3]], 1).astype(f)
    kp = np.full((N_BOXES, 6), -1, f)
    kp[np.arange(N_BOXES), rs.randint(0, 4, N_BOXES)] = rs.uniform(x1, x1 + w)
    kp[:, 4], kp[:, 5] = x1 + 0.1 * w, x1 + 0.9 * w
    do = np.stack([rs.uniform(1.4, 1.8, N_BOXES), rs.uniform(1.4, 1.7, N_BOXES), rs.uniform(3.4, 4.6, N_BOXES),
                   rs.uniform(-3.1, 3.1, N_BOXES)], 1).astype(f)
    return dict(boxes_left=bl, boxes_right=br, boxes_merge=bm, dim_orien=do, kpts=kp,
                kpts_right=np.where(kp >= 0, kp - f(20), kp).astype(f), gt_classes=np.ones(N_BOXES, np.int32),
                flipped=bool(index % 2), height=H, width=W, index=index)


def frames(e):
    rs = np.random.RandomState(1000 + e["index"])
    H, W = e["height"], e["width"]
    base = rs.randint(0, 256, (H // 8 + 2, W // 8 + 2, 3)).astype(np.float32)
    im = np.clip(np.kron(base, np.ones((8, 8, 1), np.float32))[:H, :W] + rs.randn(H, W, 3) * 6, 0, 255)
    left = im.astype(np.uint8)
    return left, np.roll(left, -20, axis=1)


def timed(fn, steps, warmup, ev):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(steps):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / steps


def run(args):
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
    dev = torch.device("cuda", torch.cuda.current_device())
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group("nccl")
    B = args.pairs_per_gpu
    sd = make_state_dict(3)
    tr = train.Trainer(StereoRCNNEngine(sd, dev, precision="fp16"), sd, grad_scale=2.0 ** 12, world=world,
                       dist=dist, seed=5)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    batch = [entry(FRAME, 10 * rank + b, 10 * rank + b) for b in range(B)]
    inp = train.StepInputs(FRAME, 600.0 / min(FRAME), dev, batch=B)
    inp.load(batch, [frames(e) for e in batch])
    with torch.no_grad():
        tr.step_from_frames(inp)                     # creates the workspaces
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        if world == 1:
            step = GraphRunner(lambda: tr.step_from_frames(inp), [], warmup=0)
        else:
            step = lambda: tr.step_from_frames(inp)  # noqa: E731
        step_ms = timed(step, args.steps, args.warmup, ev)
        peak_mb = torch.cuda.max_memory_allocated() / 2 ** 20
        ar_ms = timed(tr.grads.all_reduce, args.steps, args.warmup, ev) if world > 1 else None
    step_ms = max_over_ranks(step_ms, dev, world, dist)
    if world > 1:
        ar_ms = max_over_ranks(ar_ms, dev, world, dist)
        peaks = torch.zeros(world, dtype=torch.float64, device=dev)
        peaks[rank] = peak_mb
        dist.all_reduce(peaks)
        peaks = peaks.tolist()
    else:
        peaks = [peak_mb]
    skipped = int(tr.skipped.item())
    fit_peak = None
    blob = list(inp.im_left.shape[2:])
    if args.fit_shapes and world == 1:
        del step, inp                                # the fit below holds buffers and graphs of its own
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        shapes = KITTI_SHAPES[:args.fit_shapes]
        db = [entry(hw, 100 + i, 100 + i) for i, hw in enumerate(s for s in shapes for _ in range(2 * B))]
        train.fit(tr, db, frames, epochs=1, log=lambda s: None, batch_size=B)
        torch.cuda.synchronize()
        fit_peak = {"shapes": [list(s) for s in shapes], "steps": len(db) // B,
                    "peak_allocated_mb": round(torch.cuda.max_memory_allocated() / 2 ** 20, 1)}
    if rank != 0:
        if dist is not None:
            dist.destroy_process_group()
        return
    try:
        pl = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                             "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        pl = None
    print(json.dumps({
        "metric": "train_global_pairs_per_s", "value": round(world * B * 1e3 / step_ms, 2), "unit": "pairs/s",
        "higher_is_better": True, "world": world, "pairs_per_gpu": B, "frame": list(FRAME),
        "blob": blob, "gt_boxes_per_image": N_BOXES, "steps": args.steps,
        "warmup": args.warmup, "step_mode": "graph" if world == 1 else "eager", "ms_per_step": round(step_ms, 3),
        "allreduce_ms": None if ar_ms is None else round(ar_ms, 3), "buckets": tr.grads.describe(),
        "peak_allocated_mb_per_rank": [round(p, 1) for p in peaks], "fit": fit_peak, "skipped": skipped,
        "gpu": torch.cuda.get_device_name(dev), "power_limit_w": pl}))
    if dist is not None:
        dist.destroy_process_group()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs-per-gpu", type=int, default=2)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--fit-shapes", type=int, default=0)
    run(ap.parse_args())


if __name__ == "__main__":
    main()
