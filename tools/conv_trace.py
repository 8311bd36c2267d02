"""In-graph phase trace of every tensor-core conv launch of one forward (sb_conv_trace).

ncu serialises kernels and flushes caches, so it cannot show how the launches of a CUDA-graph replay overlap
(PDL prologues, the left/right chains on two streams).  The conv kernel can stamp %globaltimer / clock64 per
CTA at: entry, after griddepcontrol.wait, first operand stage landed, last MMA issued, first tile's epilogue
done, CTA exit, and which schedule the CTA's two consumer warpgroups ran (cooperative or ping-pong); the host
records which epilogue each launch ran (from registers, or stored by TMA through the per-warpgroup rings).  This tool
captures the forward into a graph with tracing on, replays it, and prints per launch: start / end relative to the
step, the span, and the median per-CTA phase durations.

    python tools/conv_trace.py [--out gpurun_out/conv_trace.json] [--segment trunk|all]
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
from stereo_rcnn_b200 import engine, lib, ops  # noqa: E402
from stereo_rcnn_b200.synth import make_state_dict, synth_pair  # noqa: E402

WORDS, CTAS = 16, 304


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/conv_trace.json")
    ap.add_argument("--segment", default="all")
    ap.add_argument("--max-launches", type=int, default=400)
    ap.add_argument("--throughput", action="store_true", help="the throughput schedule: one batched chain, no stream forks")
    a = ap.parse_args()
    L = lib.load()
    H, W = 600, 1987
    left, right = synth_pair(H, W, 3, 48)
    im = torch.cat((torch.from_numpy(left)[None], torch.from_numpy(right)[None]), 0).cuda().contiguous()
    info = torch.tensor([[H, W, 1.6]], device="cuda")
    eng = engine.StereoRCNNEngine(make_state_dict(3), "cuda", forks=not a.throughput)

    def fwd():
        feats = eng.trunk_fpn(im)
        if a.segment == "trunk":
            return feats
        cls_prob, bbox, shapes = eng.rpn(feats, 1)
        rl, rr = ops.proposal_layer(cls_prob, bbox, info, "TEST", shapes)
        return eng.heads(feats, 1, rl.view(-1, 5), rr.view(-1, 5), float(H))

    for _ in range(2):
        fwd()
    torch.cuda.synchronize()
    nbytes = L.sb_conv_trace_bytes(a.max_launches)
    buf = torch.zeros(nbytes // 8, dtype=torch.int64, device="cuda")
    assert L.sb_conv_trace(buf.data_ptr(), a.max_launches) == 0
    r = engine.GraphRunner(fwd, [], warmup=0)
    n = L.sb_conv_trace_count()
    infos, epis = [], []
    for i in range(n):
        v = (ctypes.c_int * 12)()
        L.sb_conv_trace_info(i, v)
        infos.append(list(v))
        epis.append(L.sb_conv_trace_epilogue(i))
    L.sb_conv_trace(None, 0)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device="cuda")
    for _ in range(3):
        ops.l2_flush(flush)
        buf.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        r()
        e.record()
        torch.cuda.synchronize()
    step_ms = s.elapsed_time(e)
    t = buf.cpu().numpy().reshape(a.max_launches, CTAS, WORDS)[:n]
    rows = []
    t_step0 = None
    for i in range(n):
        cin, cout, kh, M, BN, tiles, kblocks, res, up, variant, _max_ctas, N = infos[i]
        live = t[i, :, 0] != 0
        c = t[i, live]
        if c.shape[0] == 0:
            continue
        t0, t1, t2, t3, t4, t5 = (c[:, k].astype(np.float64) for k in range(6))
        k0, k1, k2, k3, k4, k5 = (c[:, 8 + k].astype(np.float64) for k in range(6))
        if t_step0 is None:
            t_step0 = t0.min()
        rows.append(dict(
            id=i, cin=cin, cout=cout, k=kh, M=M, N=N, BN=BN, tiles=tiles, kblocks=kblocks, res=res, up=up, variant=variant,
            ctas=int(c.shape[0]),
            start_us=(t0.min() - t_step0) / 1e3, first_work_us=(t1.min() - t_step0) / 1e3,
            end_us=(t5.max() - t_step0) / 1e3,
            span_us=(t5.max() - t0.min()) / 1e3, work_span_us=(t5.max() - t1.min()) / 1e3,
            wait_us=float(np.median(t1 - t0)) / 1e3,
            fill_cyc=float(np.median(k2 - k1)), mma_cyc=float(np.median(k3 - k2)),
            epi1_cyc=float(np.median(k4 - k2)), tail_cyc=float(np.median(k5 - k3)),
            cta_cyc=float(np.median(k5 - k1)), cta_cyc_max=float((k5 - k1).max()),
            start_skew_us=float(t1.max() - t1.min()) / 1e3, pingpong=int(c[0, 7]),
            epilogue="tma" if epis[i] == 1 else "reg"))
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(dict(step_ms=step_ms, launches=rows), f)
    print("graph step %.3f ms, %d traced conv launches" % (step_ms, len(rows)))
    print(" id  cin cout k      M  BN tiles ctas pp epi | start   work0     end |  span  wspan  wait | fill   mma  epi1  tail   cta ctamax (cycles) skew_us")
    for x in rows:
        print("%3d %4d %4d %d %6d %3d %5d %4d %2d %3s | %6.1f %6.1f %6.1f | %5.1f %5.1f %5.1f | %5.0f %5.0f %5.0f %5.0f %6.0f %6.0f  %5.1f" % (
            x["id"], x["cin"], x["cout"], x["k"], x["M"], x["BN"], x["tiles"], x["ctas"], x["pingpong"], x["epilogue"],
            x["start_us"], x["first_work_us"], x["end_us"], x["span_us"], x["work_span_us"], x["wait_us"],
            x["fill_cyc"], x["mma_cyc"], x["epi1_cyc"], x["tail_cyc"], x["cta_cyc"], x["cta_cyc_max"], x["start_skew_us"]))


    # SM time by class: sum over launches of (median CTA busy time x CTAs) / SMs, in us of a full GPU
    cls = {}
    clk_mhz = 1980.0
    n_sms = float(torch.cuda.get_device_properties(0).multi_processor_count)
    for x in rows:
        key = ("%dx%d" % (x["k"], x["k"])) + ("+res" if x["res"] else "") + ("+up" if x["up"] else "") + \
              (" f16" if x["variant"] & 1 else " tf32") + (" dgrad" if x["variant"] & 2 else "") + \
              (" small-M" if x["M"] < 30000 else "")
        c = cls.setdefault(key, [0, 0.0, 0.0, 0.0, 0.0])
        c[0] += 1
        c[1] += x["cta_cyc"] * x["ctas"] / n_sms / clk_mhz
        c[2] += x["fill_cyc"] * x["ctas"] / n_sms / clk_mhz
        c[3] += x["mma_cyc"] * x["ctas"] / n_sms / clk_mhz
        c[4] += x["tail_cyc"] * x["ctas"] / n_sms / clk_mhz
    print("\nSM time by class (us of a full GPU at %.0f MHz): launches, total, of which fill / mma / tail" % clk_mhz)
    for k_, c in sorted(cls.items(), key=lambda kv: -kv[1][1]):
        print("%-28s %3d  %7.1f   %6.1f %7.1f %6.1f" % (k_, c[0], c[1], c[2], c[3], c[4]))
    print("all convs: %.1f us" % sum(c[1] for c in cls.values()))


if __name__ == "__main__":
    main()
