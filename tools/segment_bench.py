"""Time the forward in CUDA-graph segments (trunk+FPN / RPN / proposals / heads / tail) on the GPU box."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(__file__), ".."))
from stereo_rcnn_b200 import engine, ops  # noqa: E402
from stereo_rcnn_b200.synth import DEMO_P2, DEMO_P3, gen_rois, make_state_dict, synth_pair  # noqa: E402


def timed_graph(fn, reps=10):
    r = engine.GraphRunner(fn, [])
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device="cuda")
    ts = []
    for _ in range(reps):
        ops.l2_flush(flush)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        r()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    return float(np.median(ts)), r.outputs


def main():
    H, W = 600, 1987
    left, right = synth_pair(H, W, 3, 48)
    iml, imr = torch.from_numpy(left)[None].cuda(), torch.from_numpy(right)[None].cuda()
    im = torch.cat((iml, imr), 0).contiguous()
    info = torch.tensor([[H, W, 1.6]], device="cuda")
    eng = engine.StereoRCNNEngine(make_state_dict(3), "cuda")
    b, k, p = (torch.from_numpy(x).cuda() for x in gen_rois(32, seed=3))
    c4 = ops.calib_vec(DEMO_P2, DEMO_P3)

    def stem():
        return ops.stem_conv_tc(im, eng.stem_w16, *eng.stem[1:])

    def trunk_only():
        c0 = stem()
        c1 = ops.maxpool3x3s2_ceil(c0)
        x32, x16 = None, c1
        outs = []
        for li, nb in enumerate(engine.LAYERS):
            for bi in range(nb):
                x32, x16 = eng._bottleneck16(x32, x16, "RCNN_layer%d.0.%d" % (li + 1, bi),
                                             engine.STRIDES[li] if bi == 0 else 1, bi == 0)
            outs.append((x32, x16))
        return outs
    t_layers = []
    t, _ = timed_graph(stem)
    print("stem (fused gather+GEMM)  %7.3f ms" % t)
    t_tr, _ = timed_graph(trunk_only)
    print("stem + layers 1-4         %7.3f ms" % t_tr)
    t_tf, feats = timed_graph(lambda: eng.trunk_fpn(im))
    print("trunk + FPN               %7.3f ms  (FPN %.3f)" % (t_tf, t_tf - t_tr))
    t_rpn, (cls_prob, bbox, shapes) = timed_graph(lambda: eng.rpn(feats, 1))
    print("RPN convs + head epilogue %7.3f ms" % t_rpn)
    t_pr, (rl, rr) = timed_graph(lambda: ops.proposal_layer(cls_prob, bbox, info, "TEST", shapes))
    print("proposal layer            %7.3f ms" % t_pr)
    t_hd, h = timed_graph(lambda: eng.heads(feats, 1, rl.view(-1, 5), rr.view(-1, 5), float(H)))
    print("RoIAlign + heads          %7.3f ms" % t_hd)

    def tail():
        pbl, pbr, dimo, pk = ops.test_decode(rl[0], rr[0], h["bbox_pred"], h["dim_orien_pred"], h["kpts_prob"],
                                             h["left_border_prob"], h["right_border_prob"], info[0])
        return ops.class_nms(h["cls_prob"], pbl, 1, 0.05, 0.3)
    t_tl, _ = timed_graph(tail)
    print("decode + class NMS        %7.3f ms" % t_tl)
    t_da, _ = timed_graph(lambda: ops.dense_align(c4, float(np.float32(1.6)), iml, imr, b, k, p))
    print("dense_align (D=32)        %7.3f ms" % t_da)
    print("sum                       %7.3f ms" % (t_tf + t_rpn + t_pr + t_hd + t_tl + t_da))
    for li in range(4):
        def one_layer(li=li):
            x32, x16 = (None, feats["c1_16"]) if li == 0 else (feats["c%d" % (li + 1)], feats["c%d_16" % (li + 1)])
            for bi in range(engine.LAYERS[li]):
                x32, x16 = eng._bottleneck16(x32, x16, "RCNN_layer%d.0.%d" % (li + 1, bi),
                                             engine.STRIDES[li] if bi == 0 else 1, bi == 0)
            return x32, x16
        t, _ = timed_graph(one_layer)
        print("  layer%d (%2d blocks)        %7.3f ms" % (li + 1, engine.LAYERS[li], t))


if __name__ == "__main__":
    main()
