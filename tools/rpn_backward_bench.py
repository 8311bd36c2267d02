#!/usr/bin/env python
"""Backward of the stereo RPN (engine.rpn_backward) and the whole RPN-loss gradient step (train.rpn_gradients) on one
benchmark-size stereo pair; one JSON line.

    python tools/rpn_backward_bench.py --steps K --warmup W [--fixed-blocks 1]

The pair is bench.py's synthetic 600x1987 KITTI-shape pair, the weights synth.make_state_dict(3), the ground truth
synth.synth_train_gt.  Reports ms per pair (CUDA events) of rpn_backward and of rpn_gradients (forward, anchor targets,
loss, RPN and trunk + FPN backward), the kernel time of rpn_backward split into dgrad / wgrad / packing (one
torch.profiler pass) with algorithmic TFLOP/s, and the memory the RPN keeps for its backward.
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
from stereo_rcnn_b200.engine import StereoRCNNEngine  # noqa: E402
from stereo_rcnn_b200.synth import make_state_dict, synth_pair, synth_train_gt  # noqa: E402

H_NET, W_NET = 600, 1987


def rpn_backward_flops(saved):
    """algorithmic FLOPs of rpn_backward: the fused head (24 live rows of 1024) and RPN_Conv (3x3, 256 -> 512, both
    images), each with a data and a weight gradient of 2 x the forward MACs"""
    px = sum(h * w for h, w in saved.shapes) * saved.B
    head = px * 1024 * 24
    conv = 2 * px * 256 * 512 * 9
    return 2.0 * (head + conv), 2.0 * (head + conv)


def run(args):
    dev = torch.device("cuda")
    eng = StereoRCNNEngine(make_state_dict(3), "cuda", precision="fp16")
    left, right = synth_pair(H_NET, W_NET, seed=3, shift=48)     # bench.py's pair of rank 0
    iml = torch.from_numpy(left[None]).to(dev).contiguous()
    imr = torch.from_numpy(right[None]).to(dev).contiguous()
    gt = [torch.from_numpy(t).to(dev) for t in synth_train_gt(1, 30, H_NET, W_NET, 7)[:3]]
    fb = args.fixed_blocks
    with torch.no_grad():
        im = torch.cat((iml, imr), 0)
        feats, saved_t = eng.trunk_fpn(im, save_for_backward=True)
        eng.rpn(feats, 1)                                           # warm the forward
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        _, bbox, shapes, saved, score = eng.rpn(feats, 1, save_for_backward=True)
        torch.cuda.synchronize()
        saved_mb = sum(c.numel() * c.element_size() for c in saved.cats) / 2 ** 20
        rpn_live_mb = (torch.cuda.memory_allocated() - base) / 2 ** 20
        A = score.shape[1]
        keys = train.random_words((1, A), dev, torch.Generator(device=dev).manual_seed(5))
        anchors = train.generate_anchors(shapes, dev)
        targets = train.anchor_targets(anchors, *gt, (H_NET, W_NET), keys)
        _, d_cls, d_box = train.rpn_loss(score, bbox, *targets)
        grads, _ = eng.rpn_backward(saved, d_cls, d_box)
        for _ in range(args.warmup):
            eng.rpn_backward(saved, d_cls, d_box, grads=grads)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        held = torch.cuda.memory_allocated()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(args.steps):
            eng.rpn_backward(saved, d_cls, d_box, grads=grads)
        ev[1].record()
        torch.cuda.synchronize()
        bwd_ms = ev[0].elapsed_time(ev[1]) / args.steps
        bwd_peak_mb = (torch.cuda.max_memory_allocated() - held) / 2 ** 20
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.rpn_backward(saved, d_cls, d_box, grads=grads)
            torch.cuda.synchronize()
        dg_flops, wg_flops = rpn_backward_flops(saved)
        del feats, saved_t, saved, score, bbox, d_cls, d_box, targets
        torch.cuda.empty_cache()
        # the whole step, gradients written into one set of buffers
        out = train.rpn_gradients(eng, iml, imr, *gt, keys, fixed_blocks=fb, grad_scale=2.0 ** 14)[1]
        for _ in range(args.warmup):
            train.rpn_gradients(eng, iml, imr, *gt, keys, fixed_blocks=fb, grads=out, grad_scale=2.0 ** 14)
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(args.steps):
            train.rpn_gradients(eng, iml, imr, *gt, keys, fixed_blocks=fb, grads=out, grad_scale=2.0 ** 14)
        ev[1].record()
        torch.cuda.synchronize()
        step_ms = ev[0].elapsed_time(ev[1]) / args.steps
    cat = {"dgrad": 0.0, "wgrad": 0.0, "packing": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        n = e.key
        if "conv_tc_kernel" in n:
            cat["dgrad"] += t
        elif "wgrad" in n or "colsum" in n:
            cat["wgrad"] += t
        elif "rpn_head_grad" in n or "fill" in n:
            cat["packing"] += t
    tf = lambda f, us: round(f / (us * 1e-6) / 1e12, 1) if us > 0 else None
    try:
        pl = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                             "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        pl = None
    print(json.dumps({
        "metric": "rpn_backward_ms_per_pair", "value": round(bwd_ms, 3), "unit": "ms/pair", "higher_is_better": False,
        "steps": args.steps, "warmup": args.warmup, "image": [H_NET, W_NET], "gpu": torch.cuda.get_device_name(dev),
        "power_limit_w": pl, "kernel_ms": {k: round(v / 1e3, 3) for k, v in cat.items()},
        "tflops": {"dgrad": tf(dg_flops, cat["dgrad"]), "wgrad": tf(wg_flops, cat["wgrad"])},
        "gflop": {"dgrad": round(dg_flops / 1e9, 1), "wgrad": round(wg_flops / 1e9, 1)},
        "rpn_gradients_ms_per_pair": round(step_ms, 3), "fixed_blocks": fb, "n_grads": len(out),
        "rpn_saved_cat_mb": round(saved_mb, 1), "rpn_saved_live_mb": round(rpn_live_mb, 1),
        "rpn_backward_peak_mb": round(bwd_peak_mb, 1)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--fixed-blocks", type=int, default=1, choices=[0, 1, 2, 3],
                    help="cfg.RESNET.FIXED_BLOCKS: layers 1..k are frozen")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
