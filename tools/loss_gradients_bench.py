#!/usr/bin/env python
"""Backward of the pyramid RoIAlign (engine.roi_align_backward) and the whole six-term training-loss gradient step
(train.loss_gradients) on one benchmark-size stereo pair; one JSON line.

    python tools/loss_gradients_bench.py --steps K --warmup W

The pair is bench.py's synthetic 600x1987 KITTI-shape pair, the weights synth.make_state_dict(3), the ground truth
synth.synth_train_gt, 512 sampled RoIs (the reference's TRAIN batch) with RCNN_top's dropout on, FIXED_BLOCKS = 1.
Reports ms per pair (CUDA events) of roi_align_backward and of loss_gradients, the roi_align_backward kernels split
(one torch.profiler pass), its traffic computed from shapes (lattice taps, fixed-point atomics, bytes), the peak memory
of the step, and the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from stereo_rcnn_b200 import ops, train  # noqa: E402
from stereo_rcnn_b200.engine import StereoRCNNEngine  # noqa: E402
from stereo_rcnn_b200.synth import make_state_dict, synth_pair, synth_train_gt  # noqa: E402

H_NET, W_NET = 600, 1987


def roi_backward_traffic(R, levels, C=256):
    """what roi_align_backward must move for R RoIs of each of its three sources (box L, box R, keypoints), from shapes:
    lattice taps, 64-bit atomics (4 corners x C per tap, an upper bound: zero taps and zero products skip theirs),
    bytes of pooled gradient read, accumulator bytes zeroed, and the final pass (read the accumulators and dP, write
    dP)"""
    taps = R * (8 * 8) * 2 + R * 15 * 15
    elems = sum(n * h * w for n, h, w in levels) * C
    return {"lattice_taps": taps, "atomics": taps * 4 * C,
            "d_pooled_read_mb": round(4 * (R * 49 * 512 + R * 196 * 256) / 1e6, 1),
            "acc_zero_mb": round(8 * elems / 1e6, 1), "finish_mb": round((8 + 4 + 4) * elems / 1e6, 1)}


def run(args):
    dev = torch.device("cuda")
    eng = StereoRCNNEngine(make_state_dict(3), "cuda", precision="fp16")
    left, right = synth_pair(H_NET, W_NET, seed=3, shift=48)     # bench.py's pair of rank 0
    iml = torch.from_numpy(left[None]).to(dev).contiguous()
    imr = torch.from_numpy(right[None]).to(dev).contiguous()
    gt = [torch.from_numpy(t).to(dev) for t in synth_train_gt(1, 30, H_NET, W_NET, 7)[:5]]
    gen = torch.Generator(device=dev).manual_seed(5)
    shapes = [[-(-H_NET // s), -(-W_NET // s)] for s in (4, 8, 16, 32, 64)]
    rpn_keys = train.random_words((1, 3 * sum(h * w for h, w in shapes)), dev, gen)
    keys = train.random_words((1, 2000 + 30), dev, gen)
    words = train.random_words((1, 512), dev, gen)
    dw = train.random_words((2, 512, 2048), dev, gen)
    gs = 2.0 ** 12
    with torch.no_grad():
        feats = eng.trunk_fpn(torch.cat((iml, imr), 0))
        cp, bb, shp = eng.rpn(feats, 1)
        rl, rr = ops.proposal_layer(cp, bb, train._im_info(1, H_NET, W_NET, dev), "TRAIN", shp)
        tgt = train.proposal_targets(rl, rr, gt[0], gt[1], gt[3], gt[4], keys, words)
        out, saved = eng.heads(feats, 1, tgt["rois_left"].view(-1, 5), tgt["rois_right"].view(-1, 5), float(H_NET),
                               save_for_backward=True, dropout_words=dw)
        _, g = train.rcnn_loss(out["cls_score"], out["bbox_pred"], out["dim_orien_pred"], out["kpts_pred"],
                               out["left_border_pred"], out["right_border_pred"], tgt)
        _, dpool = eng.heads_backward(saved, *g, grad_scale=gs)
        levels = [(2, feats[k].shape[1], feats[k].shape[2]) for k in ("p2", "p3", "p4", "p5")]
        dp = {k: torch.zeros_like(feats[k]) for k in ("p2", "p3", "p4", "p5")}
        for _ in range(args.warmup):
            eng.roi_align_backward(saved, dpool, dp)
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(args.steps):
            eng.roi_align_backward(saved, dpool, dp)
        ev[1].record()
        torch.cuda.synchronize()
        roi_ms = ev[0].elapsed_time(ev[1]) / args.steps
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.roi_align_backward(saved, dpool, dp)
            torch.cuda.synchronize()
        R = saved.R
        del feats, saved, out, g, dpool, dp
        torch.cuda.empty_cache()
        res = train.loss_gradients(eng, iml, imr, *gt, keys, words, rpn_keys, dropout_words=dw, grad_scale=gs)
        for _ in range(args.warmup):
            train.loss_gradients(eng, iml, imr, *gt, keys, words, rpn_keys, dropout_words=dw, grads=res[1],
                                 grad_scale=gs)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        ev[0].record()
        for _ in range(args.steps):
            train.loss_gradients(eng, iml, imr, *gt, keys, words, rpn_keys, dropout_words=dw, grads=res[1],
                                 grad_scale=gs)
        ev[1].record()
        torch.cuda.synchronize()
        step_ms = ev[0].elapsed_time(ev[1]) / args.steps
        peak_mb = torch.cuda.max_memory_allocated() / 2 ** 20
        found_inf = int(eng.found_inf.item())
    kern = {}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        for k in ("pyramid_grad_absmax", "roi_align_pyramid_bwd", "pyramid_grad_finish", "Memset"):
            if k in e.key:
                kern[k] = round(kern.get(k, 0.0) + t / 1e3, 3)
    try:
        pl = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                             "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        pl = None
    print(json.dumps({
        "metric": "roi_align_backward_ms_per_pair", "value": round(roi_ms, 3), "unit": "ms/pair",
        "higher_is_better": False, "steps": args.steps, "warmup": args.warmup, "image": [H_NET, W_NET], "rois": R,
        "gpu": torch.cuda.get_device_name(dev), "power_limit_w": pl, "kernel_ms": kern,
        "traffic": roi_backward_traffic(R, levels), "loss_gradients_ms_per_pair": round(step_ms, 3),
        "n_grads": len(res[1]), "peak_memory_mb": round(peak_mb, 1), "found_inf": found_inf}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    run(ap.parse_args())


if __name__ == "__main__":
    main()
