"""The forward 3x3 convolutions of one 600x1987 pair on 8x16 patches (sb_conv2d_tc) against flat 128-pixel rows
(sb_conv2d_tc_rows).

    python tools/conv_rows_bench.py            # MMA rows issued per launch under both tilings (no GPU needed)
    python tools/conv_rows_bench.py --time     # and the CUDA-event time of every launch through both entry points

The count comes from the descriptors one forward of the throughput schedule records (with a GPU), or from the same
shapes listed here (without one; tile widths for 132 SMs).  A patch tile issues 128 MMA rows even where it runs past
the right or bottom edge of its map; a flat tile only past the last pixel of the launch.

--time re-launches each recorded fp16 3x3 descriptor back to back through one entry point, then the other, per class
of identical shapes (the same alternation for every repeat, best of --reps), and prints the card's name, power limit
and SM clocks beside the numbers."""
import argparse
import collections
import ctypes
import os
import subprocess
import sys

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))

H_NET, W_NET, SCALE = 600, 1987, 1.6
BM, TW, TH = 128, 16, 8
Shape = collections.namedtuple("Shape", "N H W Cin Cout")


def pick_block_n(cout, m_tiles, sms):
    """conv_tc.cu pick_block_n"""
    if cout <= 32:
        return 32
    if cout <= 64:
        return 64
    if cout < 256:
        return 128
    t128, t256 = m_tiles * -(-cout // 128), m_tiles * -(-cout // 256)
    return 256 if -(-t256 // sms) * 1024 <= -(-t128 // sms) * 512 else 128


def tiling(s, rows, sms):
    """-> (m-tiles, BLOCK_N, n-tiles) of a 3x3 launch"""
    mt = -(-(s.N * s.H * s.W) // BM) if rows else s.N * -(-s.H // TH) * -(-s.W // TW)
    bn = pick_block_n(s.Cout, mt, sms)
    return mt, bn, -(-s.Cout // bn)


def listed_shapes():
    """the fp16 3x3 launches of one pair's forward in the throughput schedule (the engine's order)"""
    hw = [(150, 497), (75, 249), (38, 125), (19, 63), (10, 32)]     # P2..P6 (C2..C5 and P5[::2, ::2])
    out = []
    for (h, w), (blocks, c) in zip(hw, ((3, 64), (4, 128), (23, 256), (3, 512))):
        out += [("layer conv2 %d" % c, Shape(2, h, w, c, c))] * blocks
    for i, (h, w) in ((1, hw[2]), (2, hw[1]), (3, hw[0])):
        out.append(("smooth%d" % i, Shape(2, h, w, 256, 256)))
    for lv, (h, w) in enumerate(hw):
        out.append(("rpn_conv P%d" % (lv + 2), Shape(2, h, w, 256, 512)))
    out += [("kpts", Shape(300, 14, 14, 256, 256))] * 6
    return out


def label(s):
    return "[%d,%d,%d] %d->%d" % (s.N, s.H, s.W, s.Cin, s.Cout)


def record_forward():
    """(shape, descriptor, tensors kept alive) of every fp16 3x3 conv of one forward, as bench.py's pipeline runs it"""
    import torch
    from stereo_rcnn_b200 import pipeline
    from stereo_rcnn_b200.synth import make_state_dict, synth_pair
    dev = torch.device("cuda", 0)
    left, right = synth_pair(H_NET, W_NET, seed=3, shift=48)
    iml, imr = torch.from_numpy(left)[None].to(dev), torch.from_numpy(right)[None].to(dev)
    pipe = pipeline.StereoPipeline(make_state_dict(3), dev, throughput=True, scale=SCALE)
    eng = pipe.eng
    eng.record = []
    eng.forward(iml, imr, pipe.im_info(1, H_NET, W_NET))
    torch.cuda.synchronize()
    rec, eng.record = eng.record, None
    return [(Shape(d.N, d.H, d.W, d.Cin, d.Cout), d, keep) for d, impl, keep in rec
            if impl == "tc" and d.kh == 3 and d.in_dtype == 1 and not d.residual and not d.up_src]


def count(shapes, sms):
    print("MMA rows issued per launch (x n-tiles x BLOCK_N x 9 Cin = MACs issued), %d SMs" % sms)
    print("%-34s %9s | %6s %4s %8s | %6s %4s %8s" % ("launch", "useful", "patch", "BN", "GMAC", "rows", "BN", "GMAC"))
    tot = [0.0, 0.0, 0.0]
    for name, s in shapes:
        k = 9 * s.Cin
        useful = s.N * s.H * s.W * s.Cout * k / 1e9
        line = "%-34s %9.2f" % (name + " " + label(s), useful)
        tot[0] += useful
        for i, rows in enumerate((False, True)):
            mt, bn, nt = tiling(s, rows, sms)
            g = mt * BM * nt * bn * k / 1e9
            tot[1 + i] += g
            line += " | %6d %4d %8.2f" % (mt, bn, g)
        print(line)
    print("%d launches: %.1f GMAC useful, %.1f issued on patches (%.1f %% padding), %.1f on flat rows (%.1f %%)" % (
        len(shapes), tot[0], tot[1], 100 * (tot[1] / tot[0] - 1), tot[2], 100 * (tot[2] / tot[0] - 1)))


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=10).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = "nvidia-smi unavailable"
    return out


def time_launches(rec, reps):
    import torch
    from stereo_rcnn_b200 import lib
    L = lib.load()
    st = lib.stream_ptr()
    entries = (("patch", L.sb_conv2d_tc), ("rows", L.sb_conv2d_tc_rows))
    classes = collections.OrderedDict()
    for s, d, _keep in rec:
        classes.setdefault(s, []).append(d)

    def seq_ms(fn, descs):
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for d in descs:
            assert fn(ctypes.byref(d), st) == 0
        ev[1].record()
        torch.cuda.synchronize()
        return ev[0].elapsed_time(ev[1])

    for descs in classes.values():          # warm-up: module load, tensor-map encoder, attributes
        for _n, fn in entries:
            seq_ms(fn, descs)
    print("\n%s" % card())
    print("CUDA events, back-to-back launches of each class, best of %d (patch and rows alternated)" % reps)
    print("%-26s %3s | %9s %9s | %9s %9s | %6s" % ("class", "n", "patch ms", "per launch", "rows ms", "per launch",
                                                   "gain"))
    tot = {"patch": 0.0, "rows": 0.0}
    for s, descs in classes.items():
        best = {n: None for n, _ in entries}
        for _ in range(reps):
            for n, fn in entries:
                t = seq_ms(fn, descs)
                best[n] = t if best[n] is None else min(best[n], t)
        for n in tot:
            tot[n] += best[n]
        print("%-26s %3d | %9.3f %9.3f | %9.3f %9.3f | %5.1f%%" % (
            label(s), len(descs), best["patch"], best["patch"] / len(descs), best["rows"], best["rows"] / len(descs),
            100 * (1 - best["rows"] / best["patch"])))
    print("%-26s %3d | %9.3f %9s | %9.3f %9s | %5.1f%%" % ("all fp16 3x3", len(rec), tot["patch"], "", tot["rows"], "",
                                                            100 * (1 - tot["rows"] / tot["patch"])))
    print("%s (after timing)" % card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--time", action="store_true", help="time both entry points on the GPU")
    ap.add_argument("--reps", type=int, default=7)
    a = ap.parse_args()
    try:
        import torch
        gpu = torch.cuda.is_available()
    except ImportError:
        gpu = False
    if a.time and not gpu:
        sys.exit("--time needs a GPU")
    if gpu:
        rec = record_forward()
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        shapes = [("", s) for s, _d, _k in rec]
        print("shapes recorded from one forward (%d fp16 3x3 launches)" % len(rec))
    else:
        rec, sms, shapes = None, 132, listed_shapes()
        print("shapes as listed in this tool (no GPU: nothing recorded)")
    count(shapes, sms)
    if a.time:
        time_launches(rec, a.reps)


if __name__ == "__main__":
    main()
