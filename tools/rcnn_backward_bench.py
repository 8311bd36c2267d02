#!/usr/bin/env python
"""Backward of the R-CNN heads (engine.heads_backward) and the whole R-CNN-loss gradient step of the heads
(train.rcnn_head_gradients) on one benchmark-size stereo pair; one JSON line.

    python tools/rcnn_backward_bench.py --steps K --warmup W

The pair is bench.py's synthetic 600x1987 KITTI-shape pair, the weights synth.make_state_dict(3), the ground truth
synth.synth_train_gt, 512 sampled RoIs (the reference's TRAIN batch) with RCNN_top's dropout on.  Reports ms per pair
(CUDA events) of heads_backward and of rcnn_head_gradients (frozen forward, proposal and target layers, heads with saved
tensors, loss, heads backward), the kernel time of heads_backward split into dgrad / wgrad / tail (one torch.profiler
pass) with algorithmic TFLOP/s computed from shapes, and the bytes HeadsSaved keeps and the backward's peak memory.
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


def heads_backward_flops(R):
    """algorithmic FLOPs (2 per MAC) of the tensor-core part of heads_backward, data and weight gradients: RCNN_top.0
    (25088 -> 2048), RCNN_top.3 (2048 -> 2048), the deconv as a 1x1 conv 256 -> 1024 on 14x14, and the six 3x3 convs
    256 -> 256 on 14x14; the first keypoint conv's data gradient is the pooled_kpts gradient"""
    top0, top3 = R * 25088 * 2048, R * 2048 * 2048
    deconv = R * 196 * 256 * 1024
    conv3 = R * 196 * 256 * 256 * 9
    dgrad = top0 + top3 + deconv + 6 * conv3
    wgrad = top0 + top3 + deconv + 6 * conv3
    return 2.0 * dgrad, 2.0 * wgrad


def run(args):
    dev = torch.device("cuda")
    eng = StereoRCNNEngine(make_state_dict(3), "cuda", precision="fp16")
    left, right = synth_pair(H_NET, W_NET, seed=3, shift=48)     # bench.py's pair of rank 0
    iml = torch.from_numpy(left[None]).to(dev).contiguous()
    imr = torch.from_numpy(right[None]).to(dev).contiguous()
    gt = [torch.from_numpy(t).to(dev) for t in synth_train_gt(1, 30, H_NET, W_NET, 7)[:5]]
    gen = torch.Generator(device=dev).manual_seed(5)
    keys = train.random_words((1, 2000 + 30), dev, gen)
    words = train.random_words((1, 512), dev, gen)
    dw = train.random_words((2, 512, 2048), dev, gen)
    with torch.no_grad():
        feats = eng.trunk_fpn(torch.cat((iml, imr), 0))
        cp, bb, shapes = eng.rpn(feats, 1)
        rl, rr = ops.proposal_layer(cp, bb, train._im_info(1, H_NET, W_NET, dev), "TRAIN", shapes)
        tgt = train.proposal_targets(rl, rr, gt[0], gt[1], gt[3], gt[4], keys, words)
        rois_l, rois_r = tgt["rois_left"].view(-1, 5), tgt["rois_right"].view(-1, 5)
        eng.heads(feats, 1, rois_l, rois_r, float(H_NET), save_for_backward=True, dropout_words=dw)   # warm
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        out, saved = eng.heads(feats, 1, rois_l, rois_r, float(H_NET), save_for_backward=True, dropout_words=dw)
        torch.cuda.synchronize()
        kept = [saved.pooled_box, saved.pooled_kpts, saved.top0, saved.fc7, saved.up] + list(saved.kpts)
        saved_mb = sum(t.numel() * t.element_size() for t in kept) / 2 ** 20
        heads_live_mb = (torch.cuda.memory_allocated() - base) / 2 ** 20
        R = saved.R
        _, g = train.rcnn_loss(out["cls_score"], out["bbox_pred"], out["dim_orien_pred"], out["kpts_pred"],
                               out["left_border_pred"], out["right_border_pred"], tgt)
        grads, _ = eng.heads_backward(saved, *g)
        for _ in range(args.warmup):
            eng.heads_backward(saved, *g, grads=grads)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        held = torch.cuda.memory_allocated()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(args.steps):
            eng.heads_backward(saved, *g, grads=grads)
        ev[1].record()
        torch.cuda.synchronize()
        bwd_ms = ev[0].elapsed_time(ev[1]) / args.steps
        bwd_peak_mb = (torch.cuda.max_memory_allocated() - held) / 2 ** 20
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.heads_backward(saved, *g, grads=grads)
            torch.cuda.synchronize()
        dg_flops, wg_flops = heads_backward_flops(R)
        del feats, saved, out, g
        torch.cuda.empty_cache()
        res = train.rcnn_head_gradients(eng, iml, imr, *gt, keys, words, dropout_words=dw)
        for _ in range(args.warmup):
            train.rcnn_head_gradients(eng, iml, imr, *gt, keys, words, dropout_words=dw, grads=res[1])
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(args.steps):
            train.rcnn_head_gradients(eng, iml, imr, *gt, keys, words, dropout_words=dw, grads=res[1])
        ev[1].record()
        torch.cuda.synchronize()
        step_ms = ev[0].elapsed_time(ev[1]) / args.steps
    cat = {"dgrad": 0.0, "wgrad": 0.0, "tail": 0.0, "other": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        n = e.key
        if "conv_tc_kernel" in n:
            cat["dgrad"] += t
        elif "wgrad" in n or "colsum_final" in n:
            cat["wgrad"] += t
        elif "box_tail" in n or "kpts_tail" in n:
            cat["tail"] += t
        elif "kernel" in n or "Kernel" in n:
            cat["other"] += t          # permutes, fills
    tf = lambda f, us: round(f / (us * 1e-6) / 1e12, 1) if us > 0 else None
    try:
        pl = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                             "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        pl = None
    print(json.dumps({
        "metric": "heads_backward_ms_per_pair", "value": round(bwd_ms, 3), "unit": "ms/pair", "higher_is_better": False,
        "steps": args.steps, "warmup": args.warmup, "image": [H_NET, W_NET], "rois": R,
        "gpu": torch.cuda.get_device_name(dev), "power_limit_w": pl,
        "kernel_ms": {k: round(v / 1e3, 3) for k, v in cat.items()},
        "tflops": {"dgrad": tf(dg_flops, cat["dgrad"]), "wgrad": tf(wg_flops, cat["wgrad"])},
        "gflop": {"dgrad": round(dg_flops / 1e9, 1), "wgrad": round(wg_flops / 1e9, 1)},
        "rcnn_head_gradients_ms_per_pair": round(step_ms, 3), "n_grads": len(res[1]),
        "heads_saved_mb": round(saved_mb, 1), "heads_live_mb": round(heads_live_mb, 1),
        "heads_backward_peak_mb": round(bwd_peak_mb, 1)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    run(ap.parse_args())


if __name__ == "__main__":
    main()
