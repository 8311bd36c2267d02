#!/usr/bin/env python
"""The whole training step (train.Trainer.step: loss_gradients, clip_gradient, sb_sgd_step, sb_pack_weights) on one
benchmark-size stereo pair; one JSON line.

    python tools/train_step_bench.py --steps K --warmup W [--loss-scale {static,dynamic,ab}]

The setup is tools/loss_gradients_bench.py's: bench.py's synthetic 600x1987 KITTI-shape pair, the weights
synth.make_state_dict(3), the ground truth synth.synth_train_gt, 512 sampled RoIs with RCNN_top's dropout on,
FIXED_BLOCKS = 1, grad_scale 2^12.  Reports ms per step (CUDA events) eager and replayed from a CUDA graph, the step
split by kernel family (one torch.profiler pass in a run of its own), the bytes each new kernel must move computed from
shapes and its achieved GB/s, the peak memory, the skip count, and the card's name and power limit read in the same
run.

--loss-scale dynamic runs the same with grad_scale=train.DynamicLossScale(init_scale=2^12) (the scale read on the
device, updated after every step); --loss-scale ab builds one static and one dynamic trainer and alternates them,
eager and replayed, over --rounds rounds of --steps steps each, so both see the same clocks and neighbours, and times
the launches only the dynamic step adds (sb_loss_scale_update and the two sb_fill_reciprocal) alone.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from stereo_rcnn_b200 import train  # noqa: E402
from stereo_rcnn_b200.engine import GraphRunner, StereoRCNNEngine  # noqa: E402
from stereo_rcnn_b200.synth import make_state_dict, synth_pair, synth_train_gt  # noqa: E402

H_NET, W_NET = 600, 1987


def traffic(tr):
    """bytes each optimizer-side kernel must move, from shapes: SGD reads p, g, m and writes p, m (fp32); the pack
    reads each master once per target and writes every derived copy; clip reads g twice (norm, scale) and writes it
    once"""
    n_all = sum(v.numel() for v in tr.masters.grads)
    n_model = n_all - tr.uncert.numel()
    pack_w = pack_r = 0
    for name in tr.names:
        for t in tr.engine._refresh_tg[name]:
            n = 1
            for s in t.shape:
                n *= int(s)
            pack_r += 4 * n
            pack_w += n * t.dst.element_size() + (2 * n if t.dst16 is not None else 0)
    return {"sgd": 20 * n_all, "pack": pack_r + pack_w, "pack_write": pack_w, "clip": 12 * n_model}


def loss_scale_arg(kind):
    return train.DynamicLossScale(init_scale=2.0 ** 12) if kind == "dynamic" else 2.0 ** 12


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                               "--format=csv,noheader,nounits"], capture_output=True, text=True,
                              timeout=10).stdout.strip()
    except Exception:
        return None


def inputs(dev):
    left, right = synth_pair(H_NET, W_NET, seed=3, shift=48)
    iml = torch.from_numpy(left[None]).to(dev).contiguous()
    imr = torch.from_numpy(right[None]).to(dev).contiguous()
    gt = [torch.from_numpy(t).to(dev) for t in synth_train_gt(1, 30, H_NET, W_NET, 7)[:5]]
    gen = torch.Generator(device=dev).manual_seed(5)
    shapes = [[-(-H_NET // s), -(-W_NET // s)] for s in (4, 8, 16, 32, 64)]
    rpn_keys = train.random_words((1, 3 * sum(h * w for h, w in shapes)), dev, gen)
    keys = train.random_words((1, 2000 + 30), dev, gen)
    words = train.random_words((1, 512), dev, gen)
    dw = train.random_words((2, 512, 2048), dev, gen)
    return [iml, imr, *gt, keys, words, rpn_keys], dw


def timed(fn, n):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(n):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / n


def run_ab(args):
    """static and dynamic trainers alternated in one process: ms per step eager and replayed, per round"""
    from stereo_rcnn_b200 import ops
    dev = torch.device("cuda")
    sd = make_state_dict(3)
    step_args, dw = inputs(dev)
    trs = {k: train.Trainer(StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, fixed_blocks=1,
                            grad_scale=loss_scale_arg(k)) for k in ("static", "dynamic")}
    res = {k: {"eager": [], "graph": []} for k in trs}
    with torch.no_grad():
        runners = {k: GraphRunner(lambda *x, tr=tr: tr.step(*x, dropout_words=dw), step_args,
                                  warmup=max(args.warmup, 1)) for k, tr in trs.items()}
        for k in trs:
            for _ in range(args.warmup):
                runners[k]()
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for k, tr in trs.items():
                res[k]["eager"].append(timed(lambda: tr.step(*step_args, dropout_words=dw), args.steps))
            for k in trs:
                res[k]["graph"].append(timed(runners[k], args.steps))
        state = {k: (int(t.skipped.item()), float(t.loss_scale) if t.dynamic else t.grad_scale)
                 for k, t in trs.items()}
        # the launches only a dynamic step adds, alone over many launches
        tr = trs["dynamic"]
        u256 = torch.empty(256, dtype=torch.float32, device=dev)
        u2048 = torch.empty(2048, dtype=torch.float32, device=dev)
        added = {"sb_loss_scale_update": lambda: train.loss_scale_update(tr.engine.found_inf, tr.loss_scale,
                                                                         tr.growth_tracker),
                 "sb_fill_reciprocal_x2": lambda: (ops.fill_reciprocal_(u256, tr.loss_scale),
                                                   ops.fill_reciprocal_(u2048, tr.loss_scale))}
        # launched from the host one by one (bound by the host's launch rate), and replayed from a graph of 100
        # (the device time, as inside a replayed step)
        per = 100
        added_ms = {}
        for name, fn in added.items():
            host_ms = timed(fn, 20 * args.steps)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for _ in range(per):
                    fn()
            g.replay()
            graph_ms = timed(g.replay, args.steps) / per
            added_ms[name] = {"host_loop": round(host_ms, 4), "graph": round(graph_ms, 4)}
    med = {k: {m: round(statistics.median(v), 3) for m, v in r.items()} for k, r in res.items()}
    print(json.dumps({
        "metric": "train_step_ms_dynamic_minus_static", "unit": "ms/pair", "higher_is_better": False,
        "value": round(med["dynamic"]["graph"] - med["static"]["graph"], 3),
        "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "image": [H_NET, W_NET], "fixed_blocks": 1,
        "gpu": torch.cuda.get_device_name(dev), "power_limit_w": power_limit(),
        "median_ms": med, "rounds_ms": {k: {m: [round(x, 3) for x in v] for m, v in r.items()} for k, r in res.items()},
        "added_launches_ms": added_ms,
        "skipped_and_scale": state}))


def run(args):
    dev = torch.device("cuda")
    sd = make_state_dict(3)
    eng = StereoRCNNEngine(sd, "cuda", precision="fp16")
    step_args, dw = inputs(dev)
    tr = train.Trainer(eng, sd, fixed_blocks=1, grad_scale=loss_scale_arg(args.loss_scale))
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    with torch.no_grad():
        for _ in range(args.warmup):
            tr.step(*step_args, dropout_words=dw)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        ev[0].record()
        for _ in range(args.steps):
            tr.step(*step_args, dropout_words=dw)
        ev[1].record()
        torch.cuda.synchronize()
        eager_ms = ev[0].elapsed_time(ev[1]) / args.steps
        peak_mb = torch.cuda.max_memory_allocated() / 2 ** 20
        runner = GraphRunner(lambda *x: tr.step(*x, dropout_words=dw), step_args, warmup=max(args.warmup, 1))
        for _ in range(args.warmup):
            runner()
        torch.cuda.synchronize()
        ev[0].record()
        for _ in range(args.steps):
            runner()
        ev[1].record()
        torch.cuda.synchronize()
        graph_ms = ev[0].elapsed_time(ev[1]) / args.steps
        # each new kernel alone, over many launches (the step's own tensors)
        ev[0].record()
        for _ in range(args.steps):
            tr._sgd(tr.lr, tr.momentum, eng.found_inf, tr.skipped)
        ev[1].record()
        torch.cuda.synchronize()
        sgd_ms = ev[0].elapsed_time(ev[1]) / args.steps
        ev[0].record()
        for _ in range(args.steps):
            eng.refresh_weights(tr.params)
        ev[1].record()
        torch.cuda.synchronize()
        pack_ms = ev[0].elapsed_time(ev[1]) / args.steps
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            tr.step(*step_args, dropout_words=dw)
            torch.cuda.synchronize()
        skipped = int(tr.skipped.item())
    fam = {"sgd_step_kernel": "sb_sgd_step", "pack_weights_kernel": "sb_pack_weights",
           "clip_": "clip_gradient"}
    kern = {"sb_sgd_step": 0.0, "sb_pack_weights": 0.0, "clip_gradient": 0.0, "loss_gradients": 0.0}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = e.cuda_time_total
        if t <= 0:
            continue
        key = next((v for k, v in fam.items() if k in e.key), "loss_gradients")
        kern[key] += t / 1e3
    kern = {k: round(v, 3) for k, v in kern.items()}
    by = traffic(tr)
    gbs = lambda nbytes, ms: round(nbytes / (ms * 1e-3) / 1e9, 1) if ms > 0 else None
    pl = power_limit()
    opt_ms = kern["sb_sgd_step"] + kern["sb_pack_weights"] + kern["clip_gradient"]
    print(json.dumps({
        "metric": "train_step_ms_per_pair", "value": round(eager_ms, 3), "unit": "ms/pair", "higher_is_better": False,
        "steps": args.steps, "warmup": args.warmup, "image": [H_NET, W_NET], "fixed_blocks": 1, "grad_scale": 2 ** 12,
        **({"loss_scale": "dynamic", "final_loss_scale": float(tr.loss_scale)} if tr.dynamic else {}),
        "gpu": torch.cuda.get_device_name(dev), "power_limit_w": pl,
        "step_ms_eager": round(eager_ms, 3), "step_ms_graph": round(graph_ms, 3),
        "profile_ms": kern, "optimizer_share_of_step": round(opt_ms / max(sum(kern.values()), 1e-9), 4),
        "sgd_ms": round(sgd_ms, 3), "pack_ms": round(pack_ms, 3),
        "bytes_mb": {k: round(v / 1e6, 1) for k, v in by.items()},
        "achieved_gb_s": {"sgd": gbs(by["sgd"], sgd_ms), "pack": gbs(by["pack"], pack_ms),
                          "clip": gbs(by["clip"], kern["clip_gradient"])},
        "n_tensors": len(tr.names) + 1, "n_params": sum(v.numel() for v in tr.masters.grads),
        "pack_targets": sum(len(eng._refresh_tg[n]) for n in tr.names),
        "peak_memory_mb": round(peak_mb, 1), "skipped": skipped}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--loss-scale", choices=("static", "dynamic", "ab"), default="static")
    ap.add_argument("--rounds", type=int, default=5, help="--loss-scale ab: alternations of the two trainers")
    args = ap.parse_args()
    (run_ab if args.loss_scale == "ab" else run)(args)


if __name__ == "__main__":
    main()
