#!/usr/bin/env python
"""The training step from camera frames (train.Trainer.step_from_frames) on one benchmark-size stereo pair; one JSON
line.

    python tools/train_input_bench.py --steps K --warmup W

The setup is tools/train_step_bench.py's (weights synth.make_state_dict(3), 512 sampled RoIs with dropout,
FIXED_BLOCKS = 1, grad_scale 2^12), fed from 375x1242 uint8 frames at scale 1.6 -> 600x1987 and a 12-row roidb entry.
Reports ms per step_from_frames eager and replayed from a CUDA graph next to ms per step on the same prepared data,
each new kernel alone over many launches with the bytes it must move computed from shapes and its achieved GB/s, the
cost of the path it replaces (four torch.randint refills and two sb_prep_image calls per step), and the card's name and
power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from stereo_rcnn_b200 import ops, train  # noqa: E402
from stereo_rcnn_b200.engine import GraphRunner, StereoRCNNEngine  # noqa: E402
from stereo_rcnn_b200.synth import make_state_dict  # noqa: E402

H, W, SCALE = 375, 1242, 1.6


def frame(seed):
    rs = np.random.RandomState(seed)
    base = rs.randint(0, 256, (H // 8 + 2, W // 8 + 2, 3)).astype(np.float32)
    return np.clip(np.kron(base, np.ones((8, 8, 1), np.float32))[:H, :W] + rs.randn(H, W, 3) * 6, 0, 255).astype(np.uint8)


def entry(n=12, seed=7):
    rs = np.random.RandomState(seed)
    f = np.float32
    w, h = rs.uniform(0.08 * W, 0.3 * W, n), rs.uniform(0.1 * H, 0.4 * H, n)
    x1, y1 = rs.uniform(40, W - w - 1), rs.uniform(0, H - h - 1)
    bl = np.stack([x1, y1, x1 + w, y1 + h], 1).astype(f)
    br = bl.copy()
    br[:, [0, 2]] -= f(30)
    kp = np.full((n, 6), -1, f)
    kp[np.arange(n), rs.randint(0, 4, n)] = rs.uniform(x1, x1 + w)
    kp[:, 4], kp[:, 5] = rs.uniform(x1, x1 + 0.3 * w), rs.uniform(x1 + 0.7 * w, x1 + w)
    do = np.stack([rs.uniform(1.3, 1.8, n), rs.uniform(1.4, 1.9, n), rs.uniform(3.2, 4.6, n), rs.uniform(-3, 3, n)], 1)
    return dict(boxes_left=bl, boxes_right=br, boxes_merge=np.stack([br[:, 0], bl[:, 1], bl[:, 2], bl[:, 3]], 1),
                dim_orien=do.astype(f), kpts=kp, gt_classes=np.ones(n, np.int32), flipped=True)


def timed(fn, steps, warmup):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
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
    dev = torch.device("cuda")
    sd = make_state_dict(3)
    tr = train.Trainer(StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, fixed_blocks=1, grad_scale=2.0 ** 12, seed=5)
    inp = train.StepInputs((H, W), SCALE, dev)
    inp.load(entry(), frame(1), frame(2))
    inp.ready()
    step_args = [inp.im_left, inp.im_right, *inp.gt[:5], inp.keys, inp.words, inp.rpn_keys]
    with torch.no_grad():
        frames_eager = timed(lambda: tr.step_from_frames(inp), args.steps, args.warmup)
        step_eager = timed(lambda: tr.step(*step_args, dropout_words=inp.dropout_words), args.steps, args.warmup)
        r_frames = GraphRunner(lambda: tr.step_from_frames(inp), [], warmup=1)
        frames_graph = timed(r_frames, args.steps, args.warmup)
        r_step = GraphRunner(lambda *x: tr.step(*x, dropout_words=inp.dropout_words), step_args, warmup=1)
        step_graph = timed(r_step, args.steps, args.warmup)
        many = max(args.steps * 10, 200)
        pair_ms = timed(lambda: ops.prep_stereo_pair(inp.left_u8, inp.right_u8, SCALE, inp.flip, True,
                                                     out=(inp.im_left, inp.im_right)), many, 10)

        def fills():
            for sid, t in enumerate(inp.word_tensors):
                train.fill_random_words(t, tr.seed, tr.step_count, sid)
        words_ms = timed(fills, many, 10)
        gt_ms = timed(lambda: train.train_gt(inp.rows, inp.n_rows, inp.shuffle_words, SCALE, inp.im_left.shape[3],
                                             out=inp.gt), many, 10)

        def replaced():
            for t in inp.word_tensors[1:]:
                t.copy_(train.random_words(t.shape, dev))
            ops.prep_image(inp.left_u8[0], SCALE, True, out=inp.im_left[0])
            ops.prep_image(inp.right_u8[0], SCALE, True, out=inp.im_right[0])
        replaced_ms = timed(replaced, many, 10)
        skipped, steps_taken = int(tr.skipped.item()), int(tr.step_count.item())
    n_words = sum(t.numel() for t in inp.word_tensors)
    pair_bytes = 2 * H * W * 3 + 2 * inp.im_left.numel() * 4
    gbs = lambda nbytes, ms: round(nbytes / (ms * 1e-3) / 1e9, 1)
    try:
        pl = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                             "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        pl = None
    print(json.dumps({
        "metric": "step_from_frames_ms_per_pair", "value": round(frames_eager, 3), "unit": "ms/pair",
        "higher_is_better": False, "steps": args.steps, "warmup": args.warmup, "frame": [H, W],
        "image": list(inp.im_left.shape[2:]), "gpu": torch.cuda.get_device_name(dev), "power_limit_w": pl,
        "step_from_frames_ms_eager": round(frames_eager, 3), "step_from_frames_ms_graph": round(frames_graph, 3),
        "step_ms_eager": round(step_eager, 3), "step_ms_graph": round(step_graph, 3),
        "prep_stereo_pair_ms": round(pair_ms, 4), "random_words_ms": round(words_ms, 4), "train_gt_ms": round(gt_ms, 4),
        "bytes_mb": {"prep_stereo_pair": round(pair_bytes / 1e6, 1), "random_words": round(4 * n_words / 1e6, 1)},
        "achieved_gb_s": {"prep_stereo_pair": gbs(pair_bytes, pair_ms), "random_words": gbs(4 * n_words, words_ms)},
        "new_kernels_share_of_graph_step": round((pair_ms + words_ms + gt_ms) / frames_graph, 5),
        "replaced_randint_and_prep_image_ms": round(replaced_ms, 4), "n_words": n_words,
        "skipped": skipped, "steps_taken": steps_taken}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    run(ap.parse_args())


if __name__ == "__main__":
    main()
