"""The public end-to-end call of the hot path: stereo pair(s) in -> detection records + refined disparities out.

This is what test_net.py:120-330 does per image around the network -- forward (stereo_rcnn.py:141-324), the
test-time decode (test_net.py:138-212), the per-class NMS (test_net.py:233-259), and `align_parallel`
(dense_align.py:240-300) on the solver's poses -- as one stream-ordered launch sequence of libstereo_b200 kernels
with no host synchronisation, so that it can be captured into a CUDA graph and replayed.

* `StereoPipeline.step`   : one pass over a batch of B pairs (B = 1 is the reference's test configuration).
* `GraphSlot`             : one in-flight unit of work -- its own stream, fixed input buffers, private kernel
                            workspaces (ops.WorkspaceOwner) and the CUDA graph of one step.  Several slots may
                            replay concurrently; they share nothing but the (read-only) weights.
"""
import numpy as np
import torch

from . import engine, ops, parallel

N_CLASSES = 2


class StereoPipeline(object):
    def __init__(self, state_dict, device, throughput=False, scale=1.6, precision=None):
        """throughput=True: the schedule for several pairs in flight -- no intra-pair stream forks (left/right
        chains, RPN levels, box head): they shorten one pair's latency but cost SM time that other pairs can use"""
        self.dev = torch.device(device)
        self.eng = engine.StereoRCNNEngine(state_dict, device, precision=precision, forks=not throughput)
        self.scale = float(np.float32(scale))
        self._info = {}
        self.side = torch.cuda.Stream(device=self.dev)

    def im_info(self, B, H, W):
        key = (B, H, W)
        if key not in self._info:
            self._info[key] = torch.tensor([[H, W, self.scale]] * B, dtype=torch.float32, device=self.dev)
        return self._info[key]

    def step(self, iml, imr, calib4, rois3d, record=None):
        """iml/imr [B,3,H,W] fp32 (BGR - means, network scale); rois3d = per image (box_left [D,4], keypoints [D,5],
        poses [D,7]) in original-image units (a single tuple is accepted for B = 1) ->
        (record [B,300,33], keep [B,300] int32, nkeep [B] int32, status [B][D], best_dis [B][D])"""
        B, _, H, W = iml.shape
        if B == 1 and len(rois3d) == 3 and torch.is_tensor(rois3d[0]):
            rois3d = [rois3d]
        info = self.im_info(B, H, W)
        side_out = []

        def fork_dense_align():
            # dense_align depends only on the input pair and the poses: a parallel branch of the CUDA graph, forked
            # where the main branch runs its small proposal kernels and most SMs are idle
            main = torch.cuda.current_stream()
            self.side.wait_stream(main)
            with torch.cuda.stream(self.side):
                for b in range(B):
                    side_out.append(ops.dense_align(calib4, self.scale, iml[b], imr[b], *rois3d[b]))
        o = self.eng.forward(iml, imr, info, before_proposals=fork_dense_align)
        R = o["rois_left"].shape[1]
        if record is None:
            record = torch.empty(B, R, parallel.REC_COLS, dtype=torch.float32, device=self.dev)
        keep = torch.empty(B, R, dtype=torch.int32, device=self.dev)
        nkeep = torch.empty(B, dtype=torch.int32, device=self.dev)
        for b in range(B):
            sl = slice(b * R, (b + 1) * R)
            pbl, _pbr, _do, _pk, _ = ops.test_decode_record(
                o["rois_left"][b], o["rois_right"][b], o["cls_prob"][b], o["bbox_pred"][b], o["dim_orien_pred"][b],
                o["kpts_prob"][sl], o["left_border_prob"][sl], o["right_border_prob"][sl], info[b],
                n_classes=N_CLASSES, record=record[b])
            ops.class_nms(o["cls_prob"][b], pbl, 1, 0.05, 0.3, keep=keep[b], num=nkeep[b:b + 1])
        torch.cuda.current_stream().wait_stream(self.side)
        st = [s for s, _d in side_out]
        dis = [d for _s, d in side_out]
        return record, keep, nkeep, st, dis


    def step_with_solver(self, iml, imr, p2, p3, im_hw_orig, cls=1, eval_thresh=0.05, cap=None):
        """One pair (B = 1) end to end as test_net.py:120-330 runs it, with the solver stage on the device:
        forward -> decode (+ record) -> per-class NMS -> infer_boundary + border fix-up ->
        solve_x_y_z_theta_from_kpt -> dense_align on the solved poses -> solve_x_y_theta_from_kpt.
        No host synchronisation: detection counts stay on the device (graph-capturable).
        -> dict(record [300,33], keep, nkeep, n_solved [1], boxes_all, poses_all, status, best_dis, final [cap,13])"""
        assert iml.shape[0] == 1
        _, _, H, W = iml.shape
        info = self.im_info(1, H, W)
        o = self.eng.forward(iml, imr, info)
        R = o["rois_left"].shape[1]
        pbl, pbr, do, pk, rec = ops.test_decode_record(
            o["rois_left"][0], o["rois_right"][0], o["cls_prob"][0], o["bbox_pred"][0], o["dim_orien_pred"][0],
            o["kpts_prob"], o["left_border_prob"], o["right_border_prob"], info[0], n_classes=N_CLASSES)
        keep, nkeep = ops.class_nms(o["cls_prob"][0], pbl, cls, eval_thresh, 0.3)
        inferred = ops.infer_boundary(pbl, keep, nkeep, im_hw_orig[1], col_offset=4 * cls)
        boxes_all, kpts_all, poses_all, src, n = ops.box_solve(
            o["cls_prob"][0], pbl, pbr, do, pk, keep, nkeep, im_hw_orig, p2, p3, cls=cls, eval_thresh=eval_thresh,
            inferred=inferred, cap=cap or R)
        calib4 = ops.calib_vec(p2, p3)
        st, dis = ops.dense_align_n(calib4, self.scale, iml[0], imr[0], boxes_all, kpts_all, poses_all, n)
        final = ops.box_rectify(boxes_all, kpts_all, poses_all, st, dis, n, im_hw_orig, p2, p3)
        return dict(record=rec, keep=keep, nkeep=nkeep, n_solved=n, boxes_all=boxes_all, kpts_all=kpts_all,
                    poses_all=poses_all, src_index=src, status=st, best_dis=dis, final=final)


class GraphSlot(object):
    """One in-flight step: fixed device inputs, private workspaces, own stream, CUDA graph of `pipe.step`.

    `pipe` may be shared between slots (weights are read-only); everything a step WRITES -- activations (graph-private
    allocations), kernel workspaces (this slot's WorkspaceOwner) and results -- belongs to the slot."""

    def __init__(self, pipe, iml, imr, calib4, rois3d, own_stream=True, use_graph=True):
        self.pipe = pipe
        dev = pipe.dev
        self.stream = torch.cuda.Stream(device=dev) if own_stream else torch.cuda.current_stream()
        self.iml, self.imr = iml.clone(), imr.clone()
        self.calib4, self.rois3d = calib4, rois3d
        self.ws = ops.WorkspaceOwner()
        self.runner = None
        self.outputs = None
        if use_graph:
            # the launches of one step are captured once into a CUDA graph (no tracing compiler: the graph is the
            # literal launch sequence of our kernels) and replayed; inputs live in fixed device buffers
            with ops.workspace_owner(self.ws):
                self.runner = engine.GraphRunner(lambda a, c: pipe.step(a, c, calib4, rois3d), [self.iml, self.imr])
            self.outputs = self.runner.outputs

    def run(self):
        if self.runner is not None:
            return self.runner()
        with ops.workspace_owner(self.ws):
            self.outputs = self.pipe.step(self.iml, self.imr, self.calib4, self.rois3d)
        return self.outputs

    def load(self, iml, imr, non_blocking=True):
        """stage a new pair into the slot's fixed inputs (stream-ordered on the current stream)"""
        self.iml.copy_(iml, non_blocking=non_blocking)
        self.imr.copy_(imr, non_blocking=non_blocking)
