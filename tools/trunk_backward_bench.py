#!/usr/bin/env python
"""Backward of the trunk + FPN (engine.trunk_fpn_backward) on one benchmark-size stereo pair; one JSON line.

    python tools/trunk_backward_bench.py --steps K --warmup W [--fixed-blocks 1]

The pair is bench.py's synthetic 600x1987 KITTI-shape pair (left + right batched), the weights synth.make_state_dict(3)
and the FPN gradients seeded random ~1e-3.  Reports ms per pair (CUDA events), kernel time and algorithmic TFLOP/s
split into dgrad / wgrad / memory kernels (one torch.profiler pass), and the memory of the saved forward.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from stereo_rcnn_b200.engine import LAYERS, StereoRCNNEngine  # noqa: E402
from stereo_rcnn_b200.synth import make_state_dict, synth_pair  # noqa: E402

H_NET, W_NET = 600, 1987


def trunk_backward_flops(eng, saved, fixed_blocks):
    """algorithmic FLOPs of trunk_fpn_backward from the saved shapes: wgrad = 2 x the forward MACs of every trainable
    conv, dgrad = 2 x the forward MACs of every conv whose input gradient is formed"""
    def macs(key, x):       # x: the conv's saved input [N,H,W,Cin] (stride-1 convs: output pixels = input pixels)
        pc = eng.p[key]
        return x.shape[0] * x.shape[1] * x.shape[2] * pc.Cin * pc.Cout * pc.kh * pc.kw
    wg = dg = 0
    for smooth, lat, t, c in (("RCNN_smooth3", "RCNN_latlayer3", "t2", "c2"), ("RCNN_smooth2", "RCNN_latlayer2", "t3", "c3"),
                              ("RCNN_smooth1", "RCNN_latlayer1", "t4", "c4")):
        wg += macs(smooth, saved[t]) + macs(lat, saved[c])
        dg += macs(smooth, saved[t])
        li = {"c2": 1, "c3": 2, "c4": 3}[c]
        if li > fixed_blocks:
            dg += macs(lat, saved[c])
    wg += macs("RCNN_toplayer", saved["c5"])
    dg += macs("RCNN_toplayer", saved["c5"])
    for li in range(fixed_blocks, 4):
        for bi in range(LAYERS[li]):
            p = "RCNN_layer%d.0.%d" % (li + 1, bi)
            r = saved[p]
            m = macs(p + ".conv1", r["xin"]) + macs(p + ".conv2", r["o1"]) + macs(p + ".conv3", r["o2"])
            m += macs(p + ".downsample.0", r["xin"]) if bi == 0 else 0
            wg += m
            dg += macs(p + ".conv2", r["o1"]) + macs(p + ".conv3", r["o2"])
            if bi > 0 or li > fixed_blocks:
                dg += macs(p + ".conv1", r["xin"]) + (macs(p + ".downsample.0", r["xin"]) if bi == 0 else 0)
    return 2.0 * dg, 2.0 * wg


def run(args):
    """trunk_fpn_backward of one 600x1987 pair (left + right batched), timed by CUDA events; per-category kernel time
    (dgrad = conv_tc_kernel, wgrad = the wgrad GEMM + its reductions, memory = the FPN level combine and fills) from
    one torch.profiler pass."""
    fixed_blocks = args.fixed_blocks
    dev = torch.device("cuda")
    eng = StereoRCNNEngine(make_state_dict(3), "cuda", precision="fp16")
    left, right = synth_pair(H_NET, W_NET, seed=3, shift=48)     # bench.py's pair of rank 0
    im = torch.from_numpy(np.concatenate([left[None], right[None]], 0)).to(dev).contiguous()
    with torch.no_grad():
        eng.trunk_fpn(im)                       # warm the forward (attributes, workspaces)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        feats, saved = eng.trunk_fpn(im, save_for_backward=True)
        torch.cuda.synchronize()
        saved_peak = torch.cuda.max_memory_allocated() - base
        saved_live = torch.cuda.memory_allocated() - base
        g = torch.Generator(device="cpu").manual_seed(7)
        d = {k: (torch.randn(feats[k].shape, generator=g) * 1e-3).to(dev) for k in ("p2", "p3", "p4", "p5", "p6")}
        grads = eng.trunk_fpn_backward(saved, d, fixed_blocks=fixed_blocks)
        for _ in range(args.warmup):
            eng.trunk_fpn_backward(saved, d, fixed_blocks=fixed_blocks, grads=grads)
        torch.cuda.synchronize()
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(args.steps):
            eng.trunk_fpn_backward(saved, d, fixed_blocks=fixed_blocks, grads=grads)
        ev[1].record()
        torch.cuda.synchronize()
        ms = ev[0].elapsed_time(ev[1]) / args.steps
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            eng.trunk_fpn_backward(saved, d, fixed_blocks=fixed_blocks, grads=grads)
            torch.cuda.synchronize()
    cat = {"dgrad": 0.0, "wgrad": 0.0, "memory": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        n = e.key
        if "conv_tc_kernel" in n:
            cat["dgrad"] += t
        elif "wgrad" in n or "colsum" in n:
            cat["wgrad"] += t
        elif "fpn_grad_combine" in n or "fill" in n:
            cat["memory"] += t
    dg_flops, wg_flops = trunk_backward_flops(eng, saved, fixed_blocks)
    tf = lambda f, us: round(f / (us * 1e-6) / 1e12, 1) if us > 0 else None
    name = torch.cuda.get_device_name(dev)
    try:
        pl = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                             "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=10).stdout.strip()
    except Exception:
        pl = None
    out = {"metric": "trunk_fpn_backward_ms_per_pair", "value": round(ms, 3), "unit": "ms/pair",
           "higher_is_better": False, "steps": args.steps, "warmup": args.warmup, "fixed_blocks": fixed_blocks,
           "image": [H_NET, W_NET], "n_grads": len(grads), "gpu": name, "power_limit_w": pl,
           "kernel_ms": {k: round(v / 1e3, 3) for k, v in cat.items()},
           "tflops": {"dgrad": tf(dg_flops, cat["dgrad"]), "wgrad": tf(wg_flops, cat["wgrad"])},
           "gflop": {"dgrad": round(dg_flops / 1e9, 1), "wgrad": round(wg_flops / 1e9, 1)},
           "memory_gbs": None, "saved_forward_peak_mb": round(saved_peak / 2 ** 20, 1),
           "saved_forward_live_mb": round(saved_live / 2 ** 20, 1)}
    # memory kernels: bytes of the level combines (read dP + dT, write fp32 + fp16) over their time
    mb = 0
    for lvl in (2, 3, 4, 5):
        n = feats["p%d" % lvl].numel()
        fine = feats["p%d" % (lvl - 1)].numel() if lvl > 2 else 0
        mb += n * (4 + 4 + 2) + fine * 4
    out["memory_gbs"] = round(mb / (cat["memory"] * 1e-6) / 1e9, 1) if cat["memory"] > 0 else None
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--fixed-blocks", type=int, default=1, choices=[0, 1, 2, 3],
                    help="cfg.RESNET.FIXED_BLOCKS: layers 1..k are frozen")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
