"""The public end-to-end call of the hot path: stereo pair(s) in -> detection records + refined disparities out.

This is what test_net.py:120-330 does per image around the network -- forward (stereo_rcnn.py:141-324), the
test-time decode (test_net.py:138-212), the per-class NMS (test_net.py:233-259), and `align_parallel`
(dense_align.py:240-300) on the solver's poses -- as one stream-ordered launch sequence of libstereo_b200 kernels
with no host synchronisation, so that it can be captured into a CUDA graph and replayed.

* `StereoPipeline.step`   : one pass over a batch of B pairs (B = 1 is the reference's test configuration).
* `GraphSlot`             : one in-flight unit of work -- its own stream, fixed input buffers, private kernel
                            workspaces (ops.WorkspaceOwner) and the CUDA graph of one step.  Several slots may
                            replay concurrently; they share nothing but the (read-only) weights.
* `StereoPipeline.step_from_frames` + `EvalInputs` : one image of a test split from its uint8 frames and its
                            calibration, both in static device buffers, so that one captured graph per frame shape
                            serves every image of the split.
* `evaluate`              : test_net.py:118-335 over a split -- the KITTI result files, one per image, and with
                            `labels` their Car AP (kitti_eval).
"""
import glob
import os
import time

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

    def im_info(self, B, H, W, scale=None):
        """[B, 3] fp32 (H, W, scale) on the device, cached: two frame shapes can give one blob shape at two scales"""
        scale = self.scale if scale is None else float(np.float32(scale))
        key = (B, H, W, scale)
        if key not in self._info:
            self._info[key] = torch.tensor([[H, W, scale]] * B, dtype=torch.float32, device=self.dev)
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


    def step_with_solver(self, iml, imr, p2, p3, im_hw_orig, cls=1, eval_thresh=0.05, cap=None, scale=None):
        """One pair (B = 1) end to end as test_net.py:120-330 runs it, with the solver stage on the device:
        forward -> decode (+ record) -> per-class NMS -> infer_boundary + border fix-up ->
        solve_x_y_z_theta_from_kpt -> dense_align on the solved poses -> solve_x_y_theta_from_kpt.
        No host synchronisation: detection counts stay on the device (graph-capturable).
        p2, p3: host 3x4 matrices, or p2 a device calibration [24] (ops.device_calib) and p3 None -- read when the
        kernels run, so a captured call serves any calibration written there.  scale: im_scale of the blobs (default
        the pipeline's), rounded to fp32 as im_info holds it.
        -> dict(record [300,33], keep, nkeep, n_solved [1], boxes_all, poses_all, status, best_dis, final [cap,13])"""
        assert iml.shape[0] == 1
        _, _, H, W = iml.shape
        scale = self.scale if scale is None else float(np.float32(scale))
        info = self.im_info(1, H, W, scale)
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
        calib4 = p2 if torch.is_tensor(p2) else ops.calib_vec(p2, p3)
        st, dis = ops.dense_align_n(calib4, scale, iml[0], imr[0], boxes_all, kpts_all, poses_all, n)
        final = ops.box_rectify(boxes_all, kpts_all, poses_all, st, dis, n, im_hw_orig, p2, p3)
        return dict(record=rec, keep=keep, nkeep=nkeep, n_solved=n, boxes_all=boxes_all, kpts_all=kpts_all,
                    poses_all=poses_all, src_index=src, status=st, best_dis=dis, final=final)

    def step_from_frames(self, inp, cls=1, eval_thresh=0.05, cap=None):
        """One test image from the buffers of an EvalInputs: sb_prep_stereo_pair (flip 0) makes the two blobs, then
        step_with_solver on them with the device calibration and the scale of the frame shape.  Returns what
        step_with_solver returns.  Outside a stream capture the current stream first waits for inp.load's copies and
        afterwards marks the buffers as consumed; a captured call holds the kernels only, and whoever replays it calls
        inp.ready() before and inp.release() after."""
        capturing = torch.cuda.is_current_stream_capturing()
        if not capturing:
            inp.ready()
        ops.prep_stereo_pair(inp.left_u8, inp.right_u8, inp.scale, inp.flip, rgb_input=inp.rgb_input,
                             out=(inp.im_left[0], inp.im_right[0]))
        out = self.step_with_solver(inp.im_left, inp.im_right, inp.calib, None, inp.frame_hw, cls=cls,
                                    eval_thresh=eval_thresh, cap=cap, scale=inp.scale)
        if not capturing:
            inp.release()
        return out


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


class EvalInputs(object):
    """The static buffers of one in-flight step_from_frames at one frame shape: the uint8 frame pair, the device
    calibration [24] (P2 then P3), a flip flag fixed at 0 and the two blobs.  load() fills the frames and the
    calibration from pinned host memory on a copy stream of its own.  frame_hw: (H, W) of the camera frames; scale:
    im_scale of the blobs (target size / shorter side, blob.py:51), unrounded as prep_im_for_blob takes it; rgb_input:
    the frames are RGB, as image decoders give them, not BGR."""

    def __init__(self, frame_hw, scale, device, rgb_input=True):
        H, W = int(frame_hw[0]), int(frame_hw[1])
        self.frame_hw, self.scale, self.rgb_input, self.device = (H, W), float(scale), bool(rgb_input), device
        host = {"left_u8": torch.empty(H, W, 3, dtype=torch.uint8), "right_u8": torch.empty(H, W, 3, dtype=torch.uint8),
                "calib": torch.zeros(24, dtype=torch.float64)}
        self._host = {k: v.pin_memory() for k, v in host.items()}
        self._dev = {k: torch.zeros_like(v, device=device) for k, v in host.items()}
        self.left_u8, self.right_u8, self.calib = self._dev["left_u8"], self._dev["right_u8"], self._dev["calib"]
        self.flip = torch.zeros(1, dtype=torch.int32, device=device)
        Ho, Wo = ops.prep_image_size(H, W, self.scale)
        self.im_left = torch.zeros(1, 3, Ho, Wo, dtype=torch.float32, device=device)
        self.im_right = torch.zeros(1, 3, Ho, Wo, dtype=torch.float32, device=device)
        self._copy_stream = torch.cuda.Stream(device)
        self._copied, self._consumed = torch.cuda.Event(), torch.cuda.Event()
        torch.cuda.current_stream(device).synchronize()        # the zero fills above precede any other stream's use

    def load(self, left, right, calib):
        """fill the inputs from two uint8 [H,W,3] frames (numpy arrays or tensors) and a calibration (what
        ops.read_calibration returns, or 24 numbers: P2 then P3): a host copy into pinned memory, then non_blocking
        copies on the copy stream, which first waits until the step that last read these buffers has finished.  The
        host waits only for the previous load's copies out of the pinned buffers."""
        self._copied.synchronize()
        h = self._host
        h["left_u8"].copy_(torch.as_tensor(left))
        h["right_u8"].copy_(torch.as_tensor(right))
        if hasattr(calib, "p2"):
            calib = np.concatenate([np.asarray(calib.p2, np.float64).reshape(12), np.asarray(calib.p3, np.float64).reshape(12)])
        h["calib"].copy_(torch.as_tensor(np.asarray(calib, np.float64).reshape(24)))
        self._copy_stream.wait_event(self._consumed)
        with torch.cuda.stream(self._copy_stream):
            for k, v in h.items():
                self._dev[k].copy_(v, non_blocking=True)
            self._copied.record(self._copy_stream)

    def ready(self):
        """the current stream waits for the copies of the last load()"""
        torch.cuda.current_stream().wait_event(self._copied)

    def release(self):
        """the work enqueued so far on the current stream is the last reader of the loaded inputs"""
        self._consumed.record(torch.cuda.current_stream())


def frame_scale(frame_hw, target_size=600):
    """im_scale of a frame shape (blob.py:51): the unrounded double that prep_im_for_blob takes; im_info and
    dense_align use it rounded to fp32"""
    return float(target_size) / float(min(int(frame_hw[0]), int(frame_hw[1])))


class _EvalSlot(object):
    """one (frame shape, slot) of evaluate: inputs, workspaces, stream, graph, pinned results and their event"""

    def __init__(self, pipe, frame_hw, target_size, rgb_input):
        self.inp = EvalInputs(frame_hw, frame_scale(frame_hw, target_size), pipe.dev, rgb_input=rgb_input)
        self.ws = ops.WorkspaceOwner()
        self.stream = torch.cuda.Stream(device=pipe.dev)
        self.runner = None
        self.final_h = self.n_h = None
        self.done = torch.cuda.Event()

    def step(self, pipe):
        """step_from_frames, then its final rows and n_solved copied to this slot's pinned host buffers"""
        out = pipe.step_from_frames(self.inp)
        if self.final_h is None:
            self.final_h = torch.zeros(out["final"].shape, dtype=out["final"].dtype).pin_memory()
            self.n_h = torch.zeros(1, dtype=torch.int32).pin_memory()
        self.final_h.copy_(out["final"], non_blocking=True)
        self.n_h.copy_(out["n_solved"], non_blocking=True)
        return out


def evaluate(pipe, entries, frames, calib, result_dir, inflight=1, use_graph=True, target_size=600, rgb_input=True,
             name=None, log=print, empty_files=False, labels=None):
    """The test loop of test_net.py:118-335 over a split: per entry the frames and the calibration, forward, decode,
    per-class NMS, infer_boundary, solve_x_y_z_theta_from_kpt, align_parallel, solve_x_y_theta_from_kpt (all in
    StereoPipeline.step_from_frames), then write_detection_results' lines (kitti_utils.py:440-460) in
    result_dir/data/<name>.txt -- the files a KITTI evaluation tool reads.

    frames(entry) -> (left, right) uint8 [H,W,3] arrays (RGB unless rgb_input is False); calib(entry) -> what
    ops.read_calibration returns; name(entry) -> the file stem (default entry["image_id"]).  The scale of a frame shape
    is target_size / its shorter side (blob.py:51).

    Each (frame shape, slot) has its own EvalInputs, workspaces, stream and -- with use_graph -- one CUDA graph,
    captured after a first eager step; the graph also copies `final` and `n_solved` to the slot's pinned host
    buffers.  Entries go round-robin over `inflight` slots; the next entry's frames are read and copied while the
    current step runs, and a slot's results are read after its event, `inflight` entries late, so the steady state
    has no device-wide synchronise.  With use_graph the pipeline must be built with throughput=True (one chain per
    step, no stream forks inside it; the slots supply the concurrency), which is checked before any work.

    Files are written in entry order.  As in the reference, an image without a detection gets no file; with
    empty_files every evaluated image gets one (evaluation tools read one file per image of the split).  Where the
    reference deletes its result directory, this refuses to start when result_dir/data already holds .txt files.

    labels(entry) -> the image's KITTI label file (a path or its text): when given, the lines written for each image
    are scored against it (kitti_eval.KittiEval, on the device, after the loop), images without a detection included,
    and summary["ap"] holds KittiEval.result() -- the Car AP of exactly the files written.
    -> dict(images, lines, files, graphs, write_s: host seconds spent formatting and writing the files[, ap])"""
    data_dir = os.path.join(result_dir, "data")
    if glob.glob(os.path.join(data_dir, "*.txt")):
        raise FileExistsError("%s already holds result files; evaluate writes into an empty directory" % data_dir)
    if inflight < 1:
        raise ValueError("inflight must be >= 1")
    if use_graph and pipe.eng.forks:
        raise ValueError("evaluate captures its graphs from a pipeline built with throughput=True")
    os.makedirs(data_dir, exist_ok=True)
    name = name or (lambda e: e["image_id"])
    states = {}
    pending = [None] * inflight                  # per slot: (entry index, _EvalSlot, t_cam2_cam0_x, file stem)
    summary = dict(images=0, lines=0, files=0, graphs=0, write_s=0.0)
    scorer = None
    if labels is not None:
        from .kitti_eval import KittiEval
        scorer = KittiEval(pipe.dev)

    def load(k):
        left, right = frames(entries[k])
        hw = (int(left.shape[0]), int(left.shape[1]))
        key = (hw, k % inflight)
        if key not in states:
            states[key] = _EvalSlot(pipe, hw, target_size, rgb_input)
        st = states[key]
        c = calib(entries[k])
        st.inp.load(left, right, c)
        return st, c.t_cam2_cam0_x

    def launch(st):
        with torch.cuda.stream(st.stream), torch.no_grad(), ops.workspace_owner(st.ws):
            if not use_graph or st.runner is None:
                st.step(pipe)                    # eager; the first step on a slot also creates its workspaces
                if use_graph:
                    from .engine import GraphRunner
                    st.runner = GraphRunner(lambda: st.step(pipe), [], warmup=0)
                    summary["graphs"] += 1
            else:
                st.inp.ready()
                st.runner()
                st.inp.release()
            st.done.record(st.stream)

    def finish(p):
        k, st, t_x, stem = p
        st.done.synchronize()
        t0 = time.perf_counter()
        n = int(st.n_h[0])
        lines = ops.kitti_result_lines(st.final_h[:n], t_x)
        if lines or empty_files:
            with open(os.path.join(data_dir, stem + ".txt"), "w") as f:
                f.write("".join(lines))
            summary["files"] += 1
        summary["write_s"] += time.perf_counter() - t0
        if scorer is not None:
            scorer.add(labels(entries[k]), "".join(lines))
        summary["images"] += 1
        summary["lines"] += len(lines)

    n = len(entries)
    nxt = load(0) if n else None
    for k in range(n):
        st, t_x = nxt
        if pending[k % inflight] is not None:    # entry k - inflight: read before this slot's buffers are reused
            finish(pending[k % inflight])
        launch(st)
        pending[k % inflight] = (k, st, t_x, str(name(entries[k])))
        if k + 1 < n:
            nxt = load(k + 1)                    # host reads + H2D of the next entry overlap this step
    for j in range(inflight):                    # the last ones, in entry order
        p = pending[(n + j) % inflight]
        if p is not None:
            finish(p)
    log("evaluate: %d images, %d lines in %d files, %d graphs" % (summary["images"], summary["lines"],
                                                                 summary["files"], summary["graphs"]))
    if scorer is not None and n:
        summary["ap"] = scorer.result()
        log("evaluate: Car AP|R11 (easy, moderate, hard) 2D %s, AOS %s, BEV %s, 3D %s at IoU 0.7" % tuple(
            "/".join("%.2f" % v for v in summary["ap"][m][0.7][:, 0]) for m in ("bbox", "aos", "bev", "3d")))
    return summary
