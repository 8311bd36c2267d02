"""Torch-tensor front end of the C ABI (device memory + current stream only).

Every function launches hand-written sm_90a kernels from libstereo_b200.so on
torch's current stream; nothing here computes on the host and nothing falls back.
"""
import collections
import contextlib
import ctypes
import threading

import numpy as np
import torch

from . import lib as _l
from .lib import ConvDesc, ProposalCfg, check, ptr, stream_ptr

# constants of lib/model/utils/config.py that the hot path reads (SURVEY section 5)
CFG = dict(
    ANCHOR_RATIOS=[0.5, 1, 2], FPN_ANCHOR_SCALES=[32, 64, 128, 256, 512],
    FPN_FEAT_STRIDES=[4, 8, 16, 32, 64],
    TEST=dict(RPN_PRE_NMS_TOP_N=6000, RPN_POST_NMS_TOP_N=300, RPN_NMS_THRESH=0.7, NMS=0.3),
    TRAIN=dict(RPN_PRE_NMS_TOP_N=12000, RPN_POST_NMS_TOP_N=2000, RPN_NMS_THRESH=0.7),
    POOLING_SIZE=7, KPTS_GRID=28,
)

class WorkspaceOwner(object):
    """Scratch buffers of ONE in-flight unit of work (a pipeline slot, a CUDA graph, a test).

    Kernel workspaces hold live state between the launches of one call sequence (select histograms, NMS masks,
    partial costs), so two sequences that may overlap on the device -- e.g. two CUDA graphs replayed on different
    streams -- must not share them: each owns a WorkspaceOwner and issues its launches inside
    ``with ops.workspace_owner(owner):``.  Buffers are grow-only and a replaced buffer is RETIRED, never freed: a
    CUDA graph captured earlier has its address baked in."""

    def __init__(self):
        self.bufs, self.retired = {}, []

    def get(self, nbytes, device, tag):
        key = (str(device), tag)
        w = self.bufs.get(key)
        if w is None or w.numel() < nbytes:
            if w is not None:
                self.retired.append(w)
            w = torch.empty(int(nbytes) + 256, dtype=torch.uint8, device=device)
            self.bufs[key] = w
        return w


_default_owner = WorkspaceOwner()
_tls = threading.local()


@contextlib.contextmanager
def workspace_owner(owner):
    """route every ops.workspace() request of the enclosed launches to `owner`'s private buffers"""
    prev = getattr(_tls, "owner", None)
    _tls.owner = owner
    try:
        yield owner
    finally:
        _tls.owner = prev


def workspace(nbytes, device, tag="default"):
    """grow-only byte workspace per (owner, device, tag); avoids cudaMalloc in steady state.  Without an enclosing
    workspace_owner() the process-wide default owner is used: fine for strictly stream-ordered callers only."""
    owner = getattr(_tls, "owner", None) or _default_owner
    return owner.get(nbytes, device, tag)


def _f32c(t):
    assert t.dtype == torch.float32
    return t if t.is_contiguous() else t.contiguous()


# ------------------------------------------------------------------ NMS ----
def nms_into(keep, dets, num_out, thresh):
    """caller-allocated outputs, as nms.nms_cuda(keep, dets, num_out, thresh) (nms_gpu.py:8-10)"""
    L = _l.load()
    n = dets.shape[0]
    assert dets.dim() == 2 and dets.shape[1] == 5 and keep.dtype == torch.int32 and num_out.dtype == torch.int32
    dets = _f32c(dets)
    nb = L.sb_nms_workspace_bytes(n)
    ws = workspace(nb, dets.device, "nms")
    check(L.sb_nms(ptr(dets), n, float(thresh), ptr(keep), ptr(num_out), ptr(ws), nb, stream_ptr()), "sb_nms")
    return 1


def nms(dets, thresh):
    """-> int32 [K,1] indices kept (ascending), like nms_gpu (lib/model/nms/nms_gpu.py:7-12)"""
    n = dets.shape[0]
    keep = torch.zeros(n, 1, dtype=torch.int32, device=dets.device)
    num_out = torch.zeros(1, dtype=torch.int32, device=dets.device)
    if n == 0:
        return keep
    nms_into(keep, dets, num_out, thresh)
    return keep[:int(num_out[0])]


def nms_mask(dets, thresh):
    L = _l.load()
    n = dets.shape[0]
    cb = (n + 63) // 64
    mask = torch.zeros(n, cb, dtype=torch.int64, device=dets.device)
    check(L.sb_nms_mask(ptr(_f32c(dets)), n, float(thresh), ptr(mask), stream_ptr()), "sb_nms_mask")
    return mask


# -------------------------------------------------------------- RoIAlign ----
def roi_align_forward(ah, aw, scale, features, rois, output):
    """roi_align.roi_align_forward_cuda(ah, aw, scale, features, rois, output) (functions/roi_align.py:24-27)"""
    L = _l.load()
    if rois.dim() != 2 or rois.shape[1] != 5:
        return 0                                   # roi_align_cuda.c:19-22
    N, C, H, W = features.shape
    check(L.sb_roi_align_forward(ptr(_f32c(features)), N, C, H, W, ptr(_f32c(rois)), rois.shape[0],
                                 int(ah), int(aw), float(scale), ptr(output), stream_ptr()), "sb_roi_align_forward")
    return 1


def roi_align_backward(ah, aw, scale, top_grad, rois, bottom_grad):
    L = _l.load()
    if rois.dim() != 2 or rois.shape[1] != 5:
        return 0
    N, C, H, W = bottom_grad.shape
    check(L.sb_roi_align_backward(ptr(_f32c(top_grad)), N, C, H, W, ptr(_f32c(rois)), rois.shape[0],
                                  int(ah), int(aw), float(scale), ptr(bottom_grad), stream_ptr()),
          "sb_roi_align_backward")
    return 1


def roi_align_backward_det(ah, aw, scale, top_grad, rois, bottom_grad):
    """deterministic RoIAlign backward (fixed-point accumulation): overwrites bottom_grad [N,C,H,W]"""
    L = _l.load()
    N, C, H, W = bottom_grad.shape
    nbytes = L.sb_roi_align_backward_det_workspace(N, C, H, W)
    ws = workspace(nbytes, bottom_grad.device, "roi_bwd_det")
    check(L.sb_roi_align_backward_det(ptr(_f32c(top_grad)), N, C, H, W, ptr(_f32c(rois)), rois.shape[0], int(ah),
                                      int(aw), float(scale), ptr(bottom_grad), ptr(ws), nbytes, stream_ptr()),
          "sb_roi_align_backward_det")
    return 1


def roi_align_pyramid_nhwc(feats, im_h, rois, pooled, out=None, out_coff=0, round_tf32=False, half=False):
    """feats: 4 NHWC fp32 tensors (P2..P5); rois [R,5]; -> out [R,pooled,pooled,out_ld] NHWC (fp32, fp32 rounded
    to TF32, or fp16 when half=True)"""
    L = _l.load()
    assert len(feats) == 4
    C = feats[0].shape[3]
    for f in feats:       # the kernel reads each level as dense [N, H, W, C] fp32 rows on the RoIs' device
        assert f.dim() == 4 and f.dtype == torch.float32 and f.is_contiguous() and f.shape[3] == C, \
            "pyramid levels must be contiguous fp32 NHWC tensors with the same C"
        assert f.device == rois.device, "pyramid levels must be on the RoIs' device"
    R = rois.shape[0]
    if out is None:
        out = torch.empty(R, pooled, pooled, C, dtype=torch.float16 if half else torch.float32, device=rois.device)
    if half:
        assert out.dtype == torch.float16
        round_tf32 = 2
    fp = (ctypes.c_void_p * 4)(*[f.data_ptr() for f in feats])
    hs = (ctypes.c_int * 4)(*[f.shape[1] for f in feats])
    ws_ = (ctypes.c_int * 4)(*[f.shape[2] for f in feats])
    check(L.sb_roi_align_pyramid_nhwc(fp, hs, ws_, C, float(im_h), ptr(_f32c(rois)), R, pooled, ptr(out),
                                      out.shape[3], out_coff, int(round_tf32), stream_ptr()),
          "sb_roi_align_pyramid_nhwc")
    return out


def roi_align_pyramid_backward(d_feats, im_h, sources, nonfinite=None):
    """backward of roi_align_pyramid_nhwc: adds the gradient of every source into d_feats, 4 NHWC fp32 tensors
    [N,h,w,C] (P2..P5), in place.  sources: up to 4 tuples (grad [R,P,P,ld] fp32, rois [R,5], coff, batch_offset):
    channels coff..coff+C of grad are the gradient of a forward call on the levels' images batch_offset + rois[:,0].
    Deterministic (64-bit fixed point, one exponent for the call); nonfinite: int32 [1] device flag set to 1 on a
    non-finite gradient or result, never cleared.  -> d_feats"""
    L = _l.load()
    assert len(d_feats) == 4 and 1 <= len(sources)
    N, C = d_feats[0].shape[0], d_feats[0].shape[3]
    dev = d_feats[0].device
    for f in d_feats:     # the kernel adds into each level as dense [N, H, W, C] fp32 rows on the RoIs' device
        assert f.dim() == 4 and f.dtype == torch.float32 and f.is_contiguous() and f.shape[3] == C and \
            f.shape[0] == N, "level gradients must be contiguous fp32 NHWC tensors with the same N and C"
        assert f.device == dev
    src = (_l.RoiGradSource * len(sources))()
    keep = []           # contiguous copies must outlive the loop: the call reads them after it
    for s, (g, rois, coff, boff) in zip(src, sources):
        assert g.dim() == 4 and g.shape[1] == g.shape[2] and g.shape[0] == rois.shape[0]
        assert g.device == rois.device == dev, "gradients and level gradients must be on the RoIs' device"
        g, rois = _f32c(g), _f32c(rois)
        keep += [g, rois]
        s.grad, s.rois = g.data_ptr(), rois.data_ptr()
        s.R, s.pooled, s.ld, s.coff, s.batch_offset = g.shape[0], g.shape[1], g.shape[3], int(coff), int(boff)
    fp = (ctypes.c_void_p * 4)(*[f.data_ptr() for f in d_feats])
    hs = (ctypes.c_int * 4)(*[f.shape[1] for f in d_feats])
    ws_ = (ctypes.c_int * 4)(*[f.shape[2] for f in d_feats])
    nb = L.sb_roi_align_pyramid_backward_workspace(hs, ws_, N, C)
    ws = workspace(nb, dev, "roi_pyramid_bwd")
    check(L.sb_roi_align_pyramid_backward(src, len(sources), fp, hs, ws_, N, C, float(im_h), ptr(nonfinite), ptr(ws),
                                          nb, stream_ptr()), "sb_roi_align_pyramid_backward")
    return d_feats


# -------------------------------------------------------- proposal layer ----
def make_proposal_cfg(cfg_key, feat_shapes, ratios=None, scales=None, strides=None, cfg=None):
    cfg = CFG if cfg is None else cfg
    pc = ProposalCfg()
    ratios = cfg["ANCHOR_RATIOS"] if ratios is None else ratios
    scales = cfg["FPN_ANCHOR_SCALES"] if scales is None else scales
    strides = cfg["FPN_FEAT_STRIDES"] if strides is None else strides
    pc.n_levels = len(feat_shapes)
    for i, (h, w) in enumerate(feat_shapes):
        pc.shapes[i][0], pc.shapes[i][1] = int(h), int(w)
        pc.anchor_scales[i], pc.feat_strides[i] = int(scales[i]), int(strides[i])
    pc.n_ratios = len(ratios)
    for i, r in enumerate(ratios):
        pc.ratios[i] = float(r)
    pc.pre_nms_top_n = int(cfg[cfg_key]["RPN_PRE_NMS_TOP_N"])
    pc.post_nms_top_n = int(cfg[cfg_key]["RPN_POST_NMS_TOP_N"])
    pc.nms_thresh = float(cfg[cfg_key]["RPN_NMS_THRESH"])
    return pc


def proposal_layer(cls_prob, bbox_pred_lr, im_info, cfg_key, feat_shapes, pc=None):
    """_ProposalLayer.forward (proposal_layer.py:42-145) -> rois_left, rois_right [B,N,5]"""
    L = _l.load()
    B, A = cls_prob.shape[:2]
    pc = make_proposal_cfg(cfg_key, feat_shapes) if pc is None else pc
    post = pc.post_nms_top_n
    dev = cls_prob.device
    rl = torch.empty(B, post, 5, dtype=torch.float32, device=dev)
    rr = torch.empty(B, post, 5, dtype=torch.float32, device=dev)
    nb = L.sb_proposal_workspace_bytes(B, A, pc.pre_nms_top_n)
    ws = workspace(nb, dev, "proposal")
    check(L.sb_proposal_layer(ptr(_f32c(cls_prob)), ptr(_f32c(bbox_pred_lr)), ptr(_f32c(im_info)), B, A,
                              ctypes.byref(pc), ptr(rl), ptr(rr), ptr(ws), nb, stream_ptr()), "sb_proposal_layer")
    return rl, rr


def rpn_head_epilogue(head, B, P):
    """raw fused head output [B*P, ld] -> cls_prob [B, 3P, 2], bbox_pred [B, 3P, 6]"""
    L = _l.load()
    dev = head.device
    cls_prob = torch.empty(B, 3 * P, 2, dtype=torch.float32, device=dev)
    bbox = torch.empty(B, 3 * P, 6, dtype=torch.float32, device=dev)
    check(L.sb_rpn_head_epilogue(ptr(head), B, P, head.shape[-1], ptr(cls_prob), ptr(bbox), stream_ptr()),
          "sb_rpn_head_epilogue")
    return cls_prob, bbox


# ----------------------------------------------------------- dense_align ----
def calib_vec(p2, p3):
    p2, p3 = np.asarray(p2, np.float64), np.asarray(p3, np.float64)
    return np.array([p2[0, 0], p2[0, 2], p2[1, 2], p2[0, 3] - p3[0, 3]], np.float64)


def dense_align(calib4, scale, im_left, im_right, box_left, keypoints, poses):
    """align_parallel (dense_align.py:240-300) -> solve_status [D], best_dis [D]"""
    L = _l.load()
    iml = _f32c(im_left).reshape(3, *im_left.shape[-2:])
    imr = _f32c(im_right).reshape(3, *im_right.shape[-2:])
    H, W = iml.shape[1:]
    D = box_left.shape[0]
    dev = iml.device
    status = torch.zeros(D, dtype=torch.float32, device=dev)
    best = torch.zeros(D, dtype=torch.float32, device=dev)
    if D == 0:
        return status, best
    nb = L.sb_dense_align_workspace_bytes(H, W, D)
    ws = workspace(nb, dev, "dense_align")
    c4 = (ctypes.c_double * 4)(*[float(v) for v in calib4])
    check(L.sb_dense_align(ptr(iml), ptr(imr), H, W, c4, float(scale), ptr(_f32c(box_left)),
                           ptr(_f32c(keypoints)), ptr(_f32c(poses)), D, ptr(status), ptr(best), ptr(ws), nb,
                           stream_ptr()), "sb_dense_align")
    return status, best


def device_calib(p2, p3, device):
    """the device calibration of the *_devcalib entry points: P2 then P3, row-major, fp64 [24] on `device`"""
    c = np.concatenate([np.asarray(p2, np.float64).reshape(12), np.asarray(p3, np.float64).reshape(12)])
    return torch.from_numpy(c).to(device)


def _devcalib(c):
    """c if it is a device calibration (a CUDA fp64 tensor [24]), else None"""
    if not torch.is_tensor(c):
        return None
    assert c.is_cuda and c.dtype == torch.float64 and c.numel() == 24 and c.is_contiguous(), \
        "a device calibration is a contiguous CUDA fp64 tensor [24] (P2 then P3, row-major)"
    return c


def dense_align_n(calib4, scale, im_left, im_right, boxes_all, keypoints, poses_all, n_dev):
    """align_parallel on device-resident solver outputs: boxes_all [cap,>=4], keypoints [cap,5], poses_all [cap,>=7],
    n_dev int32 [1] (how many rows are live) -> status [cap], best_dis [cap]; rows >= n are left at zero.
    calib4: calib_vec(p2, p3) on the host, or a device calibration [24] (device_calib), read when the kernels run"""
    L = _l.load()
    iml = _f32c(im_left).reshape(3, *im_left.shape[-2:])
    imr = _f32c(im_right).reshape(3, *im_right.shape[-2:])
    H, W = iml.shape[1:]
    cap = boxes_all.shape[0]
    dev = iml.device
    status = torch.zeros(cap, dtype=torch.float32, device=dev)
    best = torch.zeros(cap, dtype=torch.float32, device=dev)
    nb = L.sb_dense_align_workspace_bytes(H, W, cap)
    ws = workspace(nb, dev, "dense_align")
    dc = _devcalib(calib4)
    if dc is not None:
        check(L.sb_dense_align_n_devcalib(ptr(iml), ptr(imr), H, W, ptr(dc), float(scale), ptr(_f32c(boxes_all)),
                                          boxes_all.shape[1], ptr(_f32c(keypoints)), ptr(_f32c(poses_all)),
                                          poses_all.shape[1], cap, ptr(n_dev), ptr(status), ptr(best), ptr(ws), nb,
                                          stream_ptr()), "sb_dense_align_n_devcalib")
        return status, best
    c4 = (ctypes.c_double * 4)(*[float(v) for v in calib4])
    check(L.sb_dense_align_n(ptr(iml), ptr(imr), H, W, c4, float(scale), ptr(_f32c(boxes_all)), boxes_all.shape[1],
                             ptr(_f32c(keypoints)), ptr(_f32c(poses_all)), poses_all.shape[1], cap, ptr(n_dev),
                             ptr(status), ptr(best), ptr(ws), nb, stream_ptr()), "sb_dense_align_n")
    return status, best


# ------------------------------------------------------------ box solver ----
def _p34(p):
    return (ctypes.c_double * 12)(*[float(v) for v in np.asarray(p, np.float64).reshape(-1)])


def infer_boundary(boxes, keep, num, im_w, col_offset=0):
    """kitti_utils.infer_boundary (kitti_utils.py:398-437) over boxes[keep[:num]] -> left_right [R,2] (kept order)"""
    L = _l.load()
    R = boxes.shape[0]
    out = torch.zeros(R, 2, dtype=torch.float32, device=boxes.device)
    check(L.sb_infer_boundary(ptr(_f32c(boxes)), boxes.shape[1], int(col_offset), ptr(keep), ptr(num), int(im_w),
                              ptr(out), stream_ptr()), "sb_infer_boundary")
    return out


def box_solve(scores, boxes_left, boxes_right, dim_orien, kpts, keep, num, im_hw, p2, p3, cls=1, eval_thresh=0.05,
              inferred=None, cap=None):
    """test_net.py:263-303 on the device: border fix-up + solve_x_y_z_theta_from_kpt per kept detection, solved ones
    appended in order -> boxes_all [cap,5], kpts_all [cap,5], poses_all [cap,8], src_index [cap], n [1] (device).
    p2, p3: host 3x4 matrices, or p2 a device calibration [24] (device_calib) and p3 None"""
    L = _l.load()
    R, nc = scores.shape
    cap = R if cap is None else int(cap)
    dev = scores.device
    boxes_all = torch.zeros(cap, 5, dtype=torch.float32, device=dev)
    kpts_all = torch.zeros(cap, 5, dtype=torch.float32, device=dev)
    poses_all = torch.zeros(cap, 8, dtype=torch.float32, device=dev)
    src = torch.zeros(cap, dtype=torch.int32, device=dev)
    n = torch.zeros(1, dtype=torch.int32, device=dev)
    dc = _devcalib(p2)
    if dc is not None:
        assert p3 is None, "with a device calibration p3 is None"
        check(L.sb_box_solve_devcalib(ptr(_f32c(scores)), ptr(_f32c(boxes_left)), ptr(_f32c(boxes_right)),
                                      ptr(_f32c(dim_orien)), ptr(_f32c(kpts)), ptr(keep), ptr(num), ptr(inferred), nc,
                                      int(cls), int(im_hw[0]), int(im_hw[1]), ptr(dc), float(eval_thresh), cap,
                                      ptr(boxes_all), ptr(kpts_all), ptr(poses_all), ptr(src), ptr(n), stream_ptr()),
              "sb_box_solve_devcalib")
        return boxes_all, kpts_all, poses_all, src, n
    check(L.sb_box_solve(ptr(_f32c(scores)), ptr(_f32c(boxes_left)), ptr(_f32c(boxes_right)), ptr(_f32c(dim_orien)),
                         ptr(_f32c(kpts)), ptr(keep), ptr(num), ptr(inferred), nc, int(cls), int(im_hw[0]),
                         int(im_hw[1]), _p34(p2), _p34(p3), float(eval_thresh), cap, ptr(boxes_all), ptr(kpts_all),
                         ptr(poses_all), ptr(src), ptr(n), stream_ptr()), "sb_box_solve")
    return boxes_all, kpts_all, poses_all, src, n


def box_rectify(boxes_all, kpts_all, poses_all, succ, best_dis, n, im_hw, p2, p3):
    """test_net.py:311-325: solve_x_y_theta_from_kpt with the aligned disparity -> final [cap,13] float64
    (valid, score, box_left 4, x, y, z, w, h, l, theta).  p2, p3 as in box_solve"""
    L = _l.load()
    cap = boxes_all.shape[0]
    out = torch.zeros(cap, 13, dtype=torch.float64, device=boxes_all.device)
    dc = _devcalib(p2)
    if dc is not None:
        assert p3 is None, "with a device calibration p3 is None"
        check(L.sb_box_rectify_devcalib(ptr(boxes_all), ptr(kpts_all), ptr(poses_all), ptr(succ), ptr(best_dis), ptr(n),
                                        cap, int(im_hw[0]), int(im_hw[1]), ptr(dc), ptr(out), stream_ptr()),
              "sb_box_rectify_devcalib")
        return out
    check(L.sb_box_rectify(ptr(boxes_all), ptr(kpts_all), ptr(poses_all), ptr(succ), ptr(best_dis), ptr(n), cap,
                           int(im_hw[0]), int(im_hw[1]), _p34(p2), _p34(p3), ptr(out), stream_ptr()), "sb_box_rectify")
    return out


Calibration = collections.namedtuple("Calibration", "p0 p1 p2 p3 t_cam2_cam0_x")


def read_calibration(path_or_text):
    """kitti_utils.read_obj_calibration (kitti_utils.py:97-159) for what the test loop reads: a KITTI calib/*.txt, given
    as a path or as its text (anything with a line break) -> Calibration(p0, p1, p2, p3 [3,4] float64,
    t_cam2_cam0_x), t_cam2_cam0_x = (p2[0,3] - p0[0,3]) / p2[0,0] (what write_detection_results subtracts from x).
    Host side: parsing text is not device work."""
    text = path_or_text
    if "\n" not in text:
        with open(path_or_text) as f:
            text = f.read()
    lines = text.splitlines()
    mats = []
    for i in range(4):
        tok = lines[i].split() if i < len(lines) else []
        if len(tok) != 13 or tok[0] != "P%d:" % i:
            raise ValueError("calibration line %d is not 'P%d:' followed by 12 numbers: %r"
                             % (i + 1, i, lines[i] if i < len(lines) else ""))
        mats.append(np.array([float(v) for v in tok[1:]], np.float64).reshape(3, 4))
    t = (mats[2][0, 3] - mats[0][0, 3]) / mats[2][0, 0]
    return Calibration(*mats, t_cam2_cam0_x=float(t))


def kitti_result_lines(final, t_cam2_cam0_x):
    """kitti_utils.write_detection_results' text (kitti_utils.py:440-460) for the valid rows of box_rectify's output
    (host side: formatting text is not device work)"""
    import math
    lines = []
    for r in final.detach().cpu().numpy():
        if r[0] <= 0:
            continue
        score, box, pos, dim, orien = r[1], r[2:6], r[6:9], r[9:12], r[12]
        alpha = orien - math.pi / 2 + math.atan2(-pos[0], pos[2])
        s = "Car -1 -1 "
        s += "%f %f %f %f %f " % (alpha, box[0], box[1], box[2], box[3])
        s += "%f %f %f %f %f %f %f %f \n" % (dim[1], dim[0], dim[2], pos[0] - t_cam2_cam0_x, pos[1], pos[2], orien - 1.57, score)
        lines.append(s)
    return lines


# ------------------------------------------------------------- layer ops ----
def conv_desc(x, wgt, out, Cin, Cout, kh, kw, stride, pad, Ho, Wo, scale=None, shift=None, residual=None,
              up_src=None, relu=False, out_coff=0, out_strides=None, out_mode=0, res_biased=False,
              in_biased=False, out16=None, max_ctas=0, in_ld=None):
    """x: NHWC [N,H,W,in_ld]; wgt packed [Cout,kh,kw,Cin]; out: any tensor addressed through out_strides
    = (n, h, w) strides in floats (default: dense NHWC of out.shape[-1] channels).  in_ld: pixel stride of x in
    elements (default x.shape[3]; a channel slice of a wider tensor passes the wider tensor's)."""
    d = ConvDesc()
    N, H, W = x.shape[0], x.shape[1], x.shape[2]
    d.in_, d.wgt = x.data_ptr(), wgt.data_ptr()
    d.out = out.data_ptr() if out is not None else None
    d.out16 = out16.data_ptr() if out16 is not None else None
    d.in_dtype = 1 if x.dtype == torch.float16 else 0
    d.max_ctas = int(max_ctas)
    assert wgt.dtype == x.dtype, "weights and activations of a conv share one operand type"
    d.scale = scale.data_ptr() if scale is not None else None
    d.shift = shift.data_ptr() if shift is not None else None
    d.residual = residual.data_ptr() if residual is not None else None
    d.up_src = up_src.data_ptr() if up_src is not None else None
    d.N, d.H, d.W, d.Cin, d.Cout, d.kh, d.kw = N, H, W, Cin, Cout, kh, kw
    d.stride, d.pad, d.Ho, d.Wo = stride, pad, Ho, Wo
    d.in_ld = x.shape[3] if in_ld is None else int(in_ld)
    d.res_ld = _flat_rows_ld(residual) if residual is not None else 0
    d.UH, d.UW = (up_src.shape[1], up_src.shape[2]) if up_src is not None else (0, 0)
    d.relu = 1 if relu else 0
    d.out_coff = out_coff
    d.out_mode, d.res_biased, d.in_biased = int(out_mode), int(bool(res_biased)), int(bool(in_biased))
    if out_strides is None:
        ld = (out if out is not None else out16).shape[-1]
        out_strides = (Ho * Wo * ld, Wo * ld, ld)
    d.out_n_stride, d.out_h_stride, d.out_w_stride = [int(s) for s in out_strides]
    return d


def _flat_rows_ld(t):
    """row pitch (elements) of an NHWC tensor whose pixels are evenly spaced rows: element (n, h, w, c) at
    (n*H*W + h*W + w) * ld + c -- the only residual layout the kernels address"""
    N, H, W, C = t.shape
    pixels = {0: H * W, 1: W, 2: 1}                  # pixels per step along n, h, w
    dims = [i for i in (2, 1, 0) if t.shape[i] > 1]  # the stride of a size-1 dimension is arbitrary
    ld = t.stride(dims[0]) // pixels[dims[0]] if dims else C
    assert (C == 1 or t.stride(3) == 1) and ld >= C, "residual channels must be contiguous"
    assert all(t.stride(i) == pixels[i] * ld for i in dims), "residual pixels must be rows of one pitch"
    return ld


def conv2d(desc, impl="auto"):
    """impl "auto": the tensor-core kernel when it takes the descriptor, else the exact-fp32 SIMT kernel, which
    has no fp16 mode -- an fp16 descriptor the tensor-core kernel rejects raises"""
    L = _l.load()
    if impl == "auto":
        impl = "tc" if L.sb_conv2d_tc_supported(ctypes.byref(desc)) else "simt"
        if impl == "simt" and (desc.in_dtype != 0 or desc.out16):
            raise _l.SbError("sb_conv2d_tc_supported rejects this fp16 descriptor and sb_conv2d_simt has no "
                             "fp16 mode")
    if impl == "tc":
        check(L.sb_conv2d_tc(ctypes.byref(desc), stream_ptr()), "sb_conv2d_tc")
    else:
        check(L.sb_conv2d_simt(ctypes.byref(desc), stream_ptr()), "sb_conv2d_simt")
    return impl


def conv2d_rows(desc):
    """fp16 3x3 / pad 1 / stride 1 conv without residual or upsample source on flat 128-pixel tiles (TMA im2col):
    bit-identical to conv2d(desc, "tc") with fewer MMA rows past the map edges; anything else raises"""
    L = _l.load()
    check(L.sb_conv2d_tc_rows(ctypes.byref(desc), stream_ptr()), "sb_conv2d_tc_rows")


def conv2d_dgrad(desc, mask16=None):
    """data gradient through the tensor-core conv (desc built on transposed weights, see sb_conv2d_tc_dgrad);
    mask16: fp16 tensor with the output's layout whose ReLU mask (> 0) is applied after the residual add"""
    L = _l.load()
    check(L.sb_conv2d_tc_dgrad(ctypes.byref(desc), ptr(mask16), stream_ptr()), "sb_conv2d_tc_dgrad")


def device_scale(grad_scale):
    """True when grad_scale is a loss scale that lives on the device (fp32 [1] CUDA tensor, read by the _devscale entry
    points), False for a host float"""
    if not torch.is_tensor(grad_scale):
        return False
    assert grad_scale.dtype == torch.float32 and grad_scale.is_cuda and grad_scale.numel() == 1 and \
        grad_scale.is_contiguous(), "a device grad_scale is an fp32 [1] CUDA tensor"
    return True


def conv_wgrad(dy16, x16, k, dw, scale=None, grad_scale=1.0, dy32=None, db=None, nonfinite=None):
    """weight (and bias) gradient of a k x k (pad k // 2) stride-1 conv: dy16 [N,H,W,Cout], x16 [N,H,W,Cin] fp16 NHWC
    -> dw [Cout,Cin,k,k] = scale[co] / grad_scale * sum dy x, db [Cout] = sum dy32 / grad_scale (fp32, written in
    place); nonfinite: int32 [1] device flag set to 1 on a non-finite result.  grad_scale: a host float, or an fp32 [1]
    CUDA tensor read on the device (sb_conv_wgrad_devscale)"""
    L = _l.load()
    N, H, W, Cout = dy16.shape
    Cin = x16.shape[3]
    assert dy16.dtype == torch.float16 and x16.dtype == torch.float16 and tuple(x16.shape[:3]) == (N, H, W)
    assert tuple(dw.shape) == (Cout, Cin, k, k) and dw.dtype == torch.float32
    nb = L.sb_conv_wgrad_workspace(N, H, W, Cin, Cout, k)
    ws = workspace(nb, dy16.device, "wgrad")
    if device_scale(grad_scale):
        check(L.sb_conv_wgrad_devscale(ptr(dy16), ptr(x16), N, H, W, Cin, Cout, k, ptr(scale), ptr(grad_scale),
                                       ptr(dw), ptr(dy32), ptr(db), ptr(nonfinite), ptr(ws), nb, stream_ptr()),
              "sb_conv_wgrad_devscale")
    else:
        check(L.sb_conv_wgrad(ptr(dy16), ptr(x16), N, H, W, Cin, Cout, k, ptr(scale), float(1.0 / grad_scale),
                              ptr(dw), ptr(dy32), ptr(db), ptr(nonfinite), ptr(ws), nb, stream_ptr()), "sb_conv_wgrad")
    return dw, db


def _vptr(t):
    """device pointer of a CUDA tensor that may be a strided view (None -> NULL)"""
    if t is None:
        return ctypes.c_void_p(0)
    assert t.is_cuda
    return ctypes.c_void_p(t.data_ptr())


def conv_wgrad_acc(dy16, x16, k, dw, db=None, dy32=None, scale=None, grad_scale=1.0, accumulate=False, rows=None,
                   split=None, dw_hi=None, db_hi=None, nonfinite=None):
    """conv_wgrad on NHWC views whose pixels are rows of one pitch (dy16 may be a channel slice of a wider tensor),
    optionally added to dw / db (accumulate=True).  Rows [0, split) of dW / db go to dw / db, rows [split, rows) to
    dw_hi / db_hi, rows past `rows` are dropped (defaults: rows = split = Cout).  grad_scale as in conv_wgrad."""
    L = _l.load()
    N, H, W, Cout = dy16.shape
    Cin = x16.shape[3]
    assert dy16.dtype == torch.float16 and x16.dtype == torch.float16 and tuple(x16.shape[:3]) == (N, H, W)
    rows = Cout if rows is None else int(rows)
    split = rows if split is None else int(split)
    kk = Cin * k * k
    assert dw.dtype == torch.float32 and dw.is_contiguous() and dw.numel() == split * kk
    assert dw_hi is None or (dw_hi.dtype == torch.float32 and dw_hi.is_contiguous() and
                             dw_hi.numel() == (rows - split) * kk)
    for b, n in ((db, split), (db_hi, rows - split)):
        assert b is None or (b.dtype == torch.float32 and b.is_contiguous() and b.numel() == n)
    assert dy32 is None or (dy32.dtype == torch.float32 and tuple(dy32.shape) == (N, H, W, Cout))
    nb = L.sb_conv_wgrad_acc_workspace(N, H, W, Cin, Cout, k)
    ws = workspace(nb, dy16.device, "wgrad")
    dev = device_scale(grad_scale)
    fn, name = (L.sb_conv_wgrad_acc_devscale, "sb_conv_wgrad_acc_devscale") if dev else \
        (L.sb_conv_wgrad_acc, "sb_conv_wgrad_acc")
    check(fn(_vptr(dy16), _flat_rows_ld(dy16), _vptr(x16), _flat_rows_ld(x16), N, H, W, Cin, Cout, k, ptr(scale),
             ptr(grad_scale) if dev else float(1.0 / grad_scale), _vptr(dy32),
             _flat_rows_ld(dy32) if dy32 is not None else 0, int(bool(accumulate)), rows, split, ptr(dw), ptr(db),
             ptr(dw_hi), ptr(db_hi), ptr(nonfinite), ptr(ws), nb, stream_ptr()), name)
    return dw, db


def rpn_head_scores(head, B, P):
    """raw fused head output [B, P, ld] -> the loss's raw class scores rpn_cls_score [B, 3P, 2]"""
    L = _l.load()
    score = torch.empty(B, 3 * P, 2, dtype=torch.float32, device=head.device)
    check(L.sb_rpn_head_scores(ptr(head), B, P, head.shape[-1], ptr(score), stream_ptr()), "sb_rpn_head_scores")
    return score


def rpn_head_grad(d_cls_score, d_bbox_pred, B, P, grad_scale=1.0, f32=True):
    """d rpn_cls_score [B,3P,2], d rpn_bbox_pred [B,3P,6] -> (dhead16 [B,P,64] fp16, dhead32 [B,P,64] fp32 or None):
    grad_scale * d in the fused head's rows 0..23, zero in 24..63 (grad_scale as in conv_wgrad)"""
    L = _l.load()
    assert tuple(d_cls_score.shape) == (B, 3 * P, 2) and tuple(d_bbox_pred.shape) == (B, 3 * P, 6)
    dev = d_cls_score.device
    dh16 = torch.empty(B, P, 64, dtype=torch.float16, device=dev)
    dh32 = torch.empty(B, P, 64, dtype=torch.float32, device=dev) if f32 else None
    if device_scale(grad_scale):
        check(L.sb_rpn_head_grad_devscale(ptr(_f32c(d_cls_score)), ptr(_f32c(d_bbox_pred)), B, P, ptr(grad_scale),
                                          ptr(dh16), ptr(dh32), stream_ptr()), "sb_rpn_head_grad_devscale")
    else:
        check(L.sb_rpn_head_grad(ptr(_f32c(d_cls_score)), ptr(_f32c(d_bbox_pred)), B, P, float(grad_scale), ptr(dh16),
                                 ptr(dh32), stream_ptr()), "sb_rpn_head_grad")
    return dh16, dh32


def fpn_grad_combine(dp=None, dt=None, dp6=None, scale=1.0, shape=None, out=None, out16=None, f32=True, f16=True):
    """gradient of one FPN level (NHWC fp32): scale * dp + up^T(dt) + scatter2(scale * dp6), where up^T is the
    transpose of the align_corners bilinear upsample from this level to dt's size and scatter2 the backward of
    P6 = P5[::2, ::2].  shape = (N, H, W, C) when dp is None.  scale: a host float or an fp32 [1] CUDA tensor read on
    the device (sb_fpn_grad_combine_devscale).  Returns (fp32, fp16) as requested."""
    L = _l.load()
    N, H, W, C = dp.shape if dp is not None else shape
    dev = next(t.device for t in (dp, dt, dp6) if t is not None)
    if out is None and f32:
        out = torch.empty(N, H, W, C, dtype=torch.float32, device=dev)
    if out16 is None and f16:
        out16 = torch.empty(N, H, W, C, dtype=torch.float16, device=dev)
    TH, TW = (dt.shape[1], dt.shape[2]) if dt is not None else (0, 0)
    H6, W6 = (dp6.shape[1], dp6.shape[2]) if dp6 is not None else (0, 0)
    for t in (dp, dt, dp6):
        assert t is None or (t.dtype == torch.float32 and t.shape[0] == N and t.shape[3] == C)
    if device_scale(scale):
        check(L.sb_fpn_grad_combine_devscale(ptr(dp), ptr(dt), N, H, W, TH, TW, C, ptr(dp6), H6, W6, ptr(scale),
                                             ptr(out), ptr(out16), stream_ptr()), "sb_fpn_grad_combine_devscale")
    else:
        check(L.sb_fpn_grad_combine(ptr(dp), ptr(dt), N, H, W, TH, TW, C, ptr(dp6), H6, W6, float(scale), ptr(out),
                                    ptr(out16), stream_ptr()), "sb_fpn_grad_combine")
    return out, out16


def upsample_transpose(dt, H, W):
    """transpose of the align_corners bilinear upsample [N,H,W,C] -> [N,TH,TW,C] applied to dt (NHWC fp32)"""
    return fpn_grad_combine(dt=dt, shape=(dt.shape[0], H, W, dt.shape[3]), f16=False)[0]


def fill_(t, v=0.0):
    """t[...] = v for a contiguous 4-byte-element CUDA tensor (sb_fill)"""
    L = _l.load()
    assert t.element_size() == 4
    check(L.sb_fill(ptr(t), t.numel(), float(v), stream_ptr()), "sb_fill")
    return t


def fill_reciprocal_(t, v):
    """t[...] = 1 / v for a contiguous fp32 CUDA tensor t and v an fp32 [1] CUDA tensor, read on the device
    (sb_fill_reciprocal)"""
    L = _l.load()
    assert t.dtype == torch.float32 and device_scale(v)
    check(L.sb_fill_reciprocal(ptr(t), t.numel(), ptr(v), stream_ptr()), "sb_fill_reciprocal")
    return t


def stem_conv(im_nchw, wgt, scale, shift, out_mode=0):
    L = _l.load()
    N, _, H, W = im_nchw.shape
    Ho, Wo = (H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1
    out = torch.empty(N, Ho, Wo, 64, dtype=torch.float32, device=im_nchw.device)
    check(L.sb_stem_conv(ptr(_f32c(im_nchw)), N, H, W, ptr(wgt), ptr(scale), ptr(shift), ptr(out), int(out_mode),
                         stream_ptr()), "sb_stem_conv")
    return out


def stem_im2col(im_nchw):
    """-> [N, Ho, Wo, 160] patch matrix of the 7x7/2 stem (147 taps zero-padded to 160)"""
    L = _l.load()
    N, _, H, W = im_nchw.shape
    Ho, Wo = (H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1
    out = torch.empty(N, Ho, Wo, 160, dtype=torch.float32, device=im_nchw.device)
    check(L.sb_stem_im2col(ptr(_f32c(im_nchw)), N, H, W, ptr(out), stream_ptr()), "sb_stem_im2col")
    return out


def stem_conv_tc(im_nchw, w16, scale, shift):
    """stem conv7x7/2 + frozen BN + ReLU as an implicit tensor-core GEMM (patch gather inside the kernel)
    -> fp16 NHWC [N, Ho, Wo, 64]; w16: fp16 [64,192], tap (ci, r, s) of output channel co at [co][ci*49 + r*7 + s],
    zero padded from 147 to three 64-wide K-steps (the engine's stem_w16)"""
    L = _l.load()
    N, _, H, W = im_nchw.shape
    Ho, Wo = (H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1
    out = torch.empty(N, Ho, Wo, 64, dtype=torch.float16, device=im_nchw.device)
    check(L.sb_stem_conv_tc(ptr(_f32c(im_nchw)), N, H, W, ptr(w16), ptr(scale), ptr(shift), ptr(out), stream_ptr()),
          "sb_stem_conv_tc")
    return out


def maxpool3x3s2_ceil(x):
    L = _l.load()
    N, H, W, C = x.shape

    def osz(v):
        o = (v - 3 + 1) // 2 + 1
        return o - 1 if (o - 1) * 2 >= v else o
    out = torch.empty(N, osz(H), osz(W), C, dtype=x.dtype, device=x.device)
    if x.dtype == torch.float16:
        check(L.sb_maxpool3x3s2_ceil16(ptr(x), N, H, W, C, ptr(out), stream_ptr()), "sb_maxpool3x3s2_ceil16")
    else:
        check(L.sb_maxpool3x3s2_ceil(ptr(x), N, H, W, C, ptr(out), stream_ptr()), "sb_maxpool3x3s2_ceil")
    return out


def subsample2(x):
    """x[:, ::2, ::2, :]; a pure copy, so fp16 tensors go through the same kernel viewed as C/2 fp32 lanes"""
    L = _l.load()
    N, H, W, C = x.shape
    out = torch.empty(N, (H - 1) // 2 + 1, (W - 1) // 2 + 1, C, dtype=x.dtype, device=x.device)
    cw = C // 2 if x.dtype == torch.float16 else C
    check(L.sb_subsample2(ptr(x), N, H, W, cw, ptr(out), stream_ptr()), "sb_subsample2")
    return out


def kpts_tail(x, w, b, want_pred_all=False):
    L = _l.load()
    R, G, _, C = x.shape
    dev = x.device
    kp = torch.empty(R, 4 * G, dtype=torch.float32, device=dev)
    lp = torch.empty(R, G, dtype=torch.float32, device=dev)
    rp = torch.empty(R, G, dtype=torch.float32, device=dev)
    ka = torch.empty(R, 6, G, dtype=torch.float32, device=dev)      # logits; also the staging between the 2 kernels
    check(L.sb_kpts_tail(ptr(x), 1 if x.dtype == torch.float16 else 0, R, G, C, ptr(w), ptr(b), ptr(kp), ptr(lp),
                         ptr(rp), ptr(ka), stream_ptr()),
          "sb_kpts_tail")
    return kp, lp, rp, ka


def box_tail(fc7, w_cls, b_cls, w_box, b_box, w_dim, b_dim, n_classes):
    L = _l.load()
    R, K = fc7.shape
    dev = fc7.device
    cls_prob = torch.empty(R, n_classes, dtype=torch.float32, device=dev)
    bbox = torch.empty(R, 6 * n_classes, dtype=torch.float32, device=dev)
    dim = torch.empty(R, 5 * n_classes, dtype=torch.float32, device=dev)
    check(L.sb_box_tail(ptr(fc7), R, K, n_classes, ptr(w_cls), ptr(b_cls), ptr(w_box), ptr(b_box), ptr(w_dim),
                        ptr(b_dim), ptr(cls_prob), ptr(bbox), ptr(dim), stream_ptr()), "sb_box_tail")
    return cls_prob, bbox, dim


def box_tail_scores(fc7, w_cls, b_cls, w_box, b_box, w_dim, b_dim, n_classes, out=None):
    """box_tail plus the raw class scores the loss reads -> cls_prob, bbox_pred, dim_orien, cls_score [R,nc]
    (out: the four tensors to write, else allocated)"""
    L = _l.load()
    R, K = fc7.shape
    dev = fc7.device
    if out is None:
        out = [torch.empty(R, n * n_classes, dtype=torch.float32, device=dev) for n in (1, 6, 5, 1)]
    cls_prob, bbox, dim, score = out
    for t, n in zip(out, (1, 6, 5, 1)):
        assert tuple(t.shape) == (R, n * n_classes) and t.dtype == torch.float32
    check(L.sb_box_tail_scores(ptr(fc7), R, K, n_classes, ptr(w_cls), ptr(b_cls), ptr(w_box), ptr(b_box), ptr(w_dim),
                               ptr(b_dim), ptr(cls_prob), ptr(bbox), ptr(dim), ptr(score), stream_ptr()),
          "sb_box_tail_scores")
    return cls_prob, bbox, dim, score


def kpts_logits(pred_all):
    """keypoint logits [R,6,G] -> kpts_pred [R,4G], left_border_pred [R,G], right_border_pred [R,G]"""
    L = _l.load()
    R, _, G = pred_all.shape
    dev = pred_all.device
    kp = torch.empty(R, 4 * G, dtype=torch.float32, device=dev)
    lb = torch.empty(R, G, dtype=torch.float32, device=dev)
    rb = torch.empty(R, G, dtype=torch.float32, device=dev)
    check(L.sb_kpts_logits(ptr(_f32c(pred_all)), R, G, ptr(kp), ptr(lb), ptr(rb), stream_ptr()), "sb_kpts_logits")
    return kp, lb, rb


def dropout_words_(x, words, p):
    """training-mode Dropout(p) in place on a contiguous fp16 / fp32 tensor: zero where the int32 word, read as uint32,
    is < p 2^32, x / (1 - p) elsewhere (one word per element)"""
    L = _l.load()
    assert x.dtype in (torch.float16, torch.float32) and words.dtype == torch.int32
    assert words.is_contiguous() and words.numel() == x.numel() and words.device == x.device
    check(L.sb_dropout_words(ptr(x), 1 if x.dtype == torch.float16 else 0, x.numel(), ptr(words), float(p),
                             stream_ptr()), "sb_dropout_words")
    return x


def box_tail_backward(d_cls, d_box, d_dim, fc7, w_cls, w_box, w_dim, grads, mask_scale=1.0, grad_scale=1.0,
                      nonfinite=None):
    """backward of the box tail's three linears: grads = (dw_cls, db_cls, dw_box, db_box, dw_dim, db_dim), written in
    place -> (dz16, dz32) [R,K], the gradient of RCNN_top.3's pre-activation times grad_scale (as in conv_wgrad)"""
    L = _l.load()
    R, K = fc7.shape
    nc = d_cls.shape[1]
    assert tuple(d_box.shape) == (R, 6 * nc) and tuple(d_dim.shape) == (R, 5 * nc) and d_cls.shape[0] == R
    for g, n in zip(grads, (nc * K, nc, 6 * nc * K, 6 * nc, 5 * nc * K, 5 * nc)):
        assert g.dtype == torch.float32 and g.is_contiguous() and g.numel() == n
    dz16 = torch.empty(R, K, dtype=torch.float16, device=fc7.device)
    dz32 = torch.empty(R, K, dtype=torch.float32, device=fc7.device)
    dev = device_scale(grad_scale)
    fn, name = (L.sb_box_tail_backward_devscale, "sb_box_tail_backward_devscale") if dev else \
        (L.sb_box_tail_backward, "sb_box_tail_backward")
    check(fn(ptr(_f32c(d_cls)), ptr(_f32c(d_box)), ptr(_f32c(d_dim)), ptr(_f32c(fc7)), R, K, nc, ptr(w_cls), ptr(w_box),
             ptr(w_dim), float(mask_scale), ptr(grad_scale) if dev else float(grad_scale), *[ptr(g) for g in grads],
             ptr(dz16), ptr(dz32), ptr(nonfinite), stream_ptr()), name)
    return dz16, dz32


def kpts_tail_backward(up16, w, d_kpts_pred, d_left, d_right, dw, db, db_up, grad_scale=1.0, nonfinite=None):
    """backward of the keypoint tail: up16 [R,G,G,C] the saved deconv output, w [6,C] kpts_class -> dw [6*C], db [6],
    db_up [C] written in place; returns dup16 [R,G/2,G/2,4C], the masked deconv-output gradient times grad_scale in
    the deconv's four (a, b) phases (grad_scale as in conv_wgrad)"""
    L = _l.load()
    R, G, _, C = up16.shape
    assert up16.dtype == torch.float16 and up16.is_contiguous()
    assert tuple(d_kpts_pred.shape) == (R, 4 * G) and tuple(d_left.shape) == (R, G) and tuple(d_right.shape) == (R, G)
    for g, n in ((dw, 6 * C), (db, 6), (db_up, C)):
        assert g.dtype == torch.float32 and g.is_contiguous() and g.numel() == n
    dup = torch.empty(R, G // 2, G // 2, 4 * C, dtype=torch.float16, device=up16.device)
    nb = L.sb_kpts_tail_backward_workspace(R, C)
    ws = workspace(nb, up16.device, "kpts_tail_bwd")
    dev = device_scale(grad_scale)
    fn, name = (L.sb_kpts_tail_backward_devscale, "sb_kpts_tail_backward_devscale") if dev else \
        (L.sb_kpts_tail_backward, "sb_kpts_tail_backward")
    check(fn(ptr(up16), R, G, C, ptr(w), ptr(_f32c(d_kpts_pred)), ptr(_f32c(d_left)), ptr(_f32c(d_right)),
             ptr(grad_scale) if dev else float(grad_scale), ptr(dup), ptr(dw), ptr(db), ptr(db_up), ptr(nonfinite),
             ptr(ws), nb, stream_ptr()), name)
    return dup


def permute3(src, dims, strides, dst):
    """dst[i0 s0 + i1 s1 + i2 s2] = src[i0, i1, i2] for src viewed as dims = (d0, d1, d2) (fp32, out of place)"""
    L = _l.load()
    assert src.dtype == torch.float32 and dst.dtype == torch.float32 and dst.is_contiguous()
    assert src.numel() == dst.numel() == dims[0] * dims[1] * dims[2]
    check(L.sb_permute3(ptr(_f32c(src)), *[int(d) for d in dims], *[int(s) for s in strides], ptr(dst), stream_ptr()),
          "sb_permute3")
    return dst


def test_decode(rois_left, rois_right, bbox_pred, dim_orien, kpts_prob, left_prob, right_prob, im_info,
                n_classes=2, grid=28):
    """test_net.py:138-212 -> pred_boxes_left [R,4nc], pred_boxes_right, dim_orien [R,5nc], pred_kpts [R,5]"""
    L = _l.load()
    R = rois_left.shape[0]
    dev = rois_left.device
    pbl = torch.empty(R, 4 * n_classes, dtype=torch.float32, device=dev)
    pbr = torch.empty(R, 4 * n_classes, dtype=torch.float32, device=dev)
    do = torch.empty(R, 5 * n_classes, dtype=torch.float32, device=dev)
    pk = torch.empty(R, 5, dtype=torch.float32, device=dev)
    check(L.sb_test_decode(ptr(_f32c(rois_left)), ptr(_f32c(rois_right)), ptr(_f32c(bbox_pred)),
                           ptr(_f32c(dim_orien)), ptr(_f32c(kpts_prob)), ptr(_f32c(left_prob)),
                           ptr(_f32c(right_prob)), ptr(_f32c(im_info)), R, n_classes, grid, ptr(pbl), ptr(pbr),
                           ptr(do), ptr(pk), stream_ptr()), "sb_test_decode")
    return pbl, pbr, do, pk


def test_decode_record(rois_left, rois_right, cls_prob, bbox_pred, dim_orien, kpts_prob, left_prob, right_prob,
                       im_info, n_classes=2, grid=28, record=None):
    """test_decode + the [R, 14nc+5] detection record of the image (what ranks all-gather), one launch"""
    L = _l.load()
    R = rois_left.shape[0]
    dev = rois_left.device
    pbl = torch.empty(R, 4 * n_classes, dtype=torch.float32, device=dev)
    pbr = torch.empty(R, 4 * n_classes, dtype=torch.float32, device=dev)
    do = torch.empty(R, 5 * n_classes, dtype=torch.float32, device=dev)
    pk = torch.empty(R, 5, dtype=torch.float32, device=dev)
    if record is None:
        record = torch.empty(R, 14 * n_classes + 5, dtype=torch.float32, device=dev)
    check(L.sb_test_decode_record(ptr(_f32c(rois_left)), ptr(_f32c(rois_right)), ptr(_f32c(cls_prob)),
                                  ptr(_f32c(bbox_pred)), ptr(_f32c(dim_orien)), ptr(_f32c(kpts_prob)),
                                  ptr(_f32c(left_prob)), ptr(_f32c(right_prob)), ptr(_f32c(im_info)), R, n_classes,
                                  grid, ptr(pbl), ptr(pbr), ptr(do), ptr(pk), ptr(record), record.shape[-1],
                                  stream_ptr()), "sb_test_decode_record")
    return pbl, pbr, do, pk, record


def class_nms(scores, boxes_left, cls, score_thresh=0.05, nms_thresh=0.3, keep=None, num=None):
    """test_net.py:233-259 on device -> (keep [R] int32 RoI indices in kept order, num [1] int32)"""
    L = _l.load()
    R, nc = scores.shape
    if keep is None:
        keep = torch.empty(R, dtype=torch.int32, device=scores.device)
    if num is None:
        num = torch.empty(1, dtype=torch.int32, device=scores.device)
    check(L.sb_class_nms(ptr(_f32c(scores)), ptr(_f32c(boxes_left)), R, nc, int(cls), float(score_thresh),
                         float(nms_thresh), ptr(keep), ptr(num), stream_ptr()), "sb_class_nms")
    return keep, num


def prep_image(img_u8, scale, rgb_input=False, out=None):
    """prep_im_for_blob (blob.py:44-64) on the device: uint8 [H,W,3] -> fp32 [3,Ho,Wo] (BGR - means, resized)"""
    L = _l.load()
    assert img_u8.dtype == torch.uint8 and img_u8.dim() == 3 and img_u8.shape[2] == 3
    H, W = img_u8.shape[:2]
    ho, wo = ctypes.c_int(), ctypes.c_int()
    check(L.sb_prep_image_size(H, W, float(scale), ctypes.byref(ho), ctypes.byref(wo)), "sb_prep_image_size")
    if out is None:
        out = torch.empty(3, ho.value, wo.value, dtype=torch.float32, device=img_u8.device)
    assert tuple(out.shape) == (3, ho.value, wo.value)
    check(L.sb_prep_image(ptr(img_u8.contiguous()), H, W, float(scale), 1 if rgb_input else 0, ptr(out), stream_ptr()),
          "sb_prep_image")
    return out


def prep_image_size(H, W, scale):
    """(Ho, Wo) of the blob prep_image makes of an [H, W] frame at `scale`"""
    ho, wo = ctypes.c_int(), ctypes.c_int()
    check(_l.load().sb_prep_image_size(int(H), int(W), float(scale), ctypes.byref(ho), ctypes.byref(wo)),
          "sb_prep_image_size")
    return ho.value, wo.value


def prep_stereo_pair(left_u8, right_u8, scale, flip, rgb_input=False, out=None):
    """_get_image_blob (minibatch.py:89-131) for one pair or a batch of pairs in one launch: uint8 frames [H,W,3]
    (one pair, flip int32 [1], blobs fp32 [3,Ho,Wo]) or [B,H,W,3] (B pairs, flip int32 [B], blobs [B,3,Ho,Wo]).
    flip: device tensor; where set the left blob of the pair is prep_image of the column-mirrored right frame and the
    right blob of the mirrored left frame (minibatch.py:116-119).  out: (left, right) to write"""
    L = _l.load()
    assert left_u8.dtype == torch.uint8 and left_u8.dim() in (3, 4) and left_u8.shape[-1] == 3
    assert right_u8.dtype == torch.uint8 and right_u8.shape == left_u8.shape and flip.dtype == torch.int32
    lead = tuple(left_u8.shape[:-3])
    B = lead[0] if lead else 1
    assert flip.numel() == B
    H, W = left_u8.shape[-3:-1]
    ho, wo = ctypes.c_int(), ctypes.c_int()
    check(L.sb_prep_image_size(H, W, float(scale), ctypes.byref(ho), ctypes.byref(wo)), "sb_prep_image_size")
    shape = lead + (3, ho.value, wo.value)
    if out is None:
        out = tuple(torch.empty(shape, dtype=torch.float32, device=left_u8.device) for _ in range(2))
    assert all(tuple(o.shape) == shape and o.dtype == torch.float32 for o in out)
    check(L.sb_prep_stereo_pairs(ptr(left_u8), ptr(right_u8), B, H, W, float(scale), 1 if rgb_input else 0, ptr(flip),
                                 ptr(out[0]), ptr(out[1]), stream_ptr()), "sb_prep_stereo_pairs")
    return out


def l2_flush(buf):
    L = _l.load()
    check(L.sb_fill(ptr(buf), buf.numel(), 0.0, stream_ptr()), "sb_fill")


def launch_count():
    return int(_l.load().sb_launch_count())


EXACT, ROUND_TF32, BIASED = 0, 1, 2          # sb_conv_desc.out_mode


def round_tf32_(w):
    """in-place round-to-nearest (ties away) of fp32 values to TF32 precision (weights, once at pack time)"""
    b = w.view(torch.int32)
    b.add_(0x1000).bitwise_and_(~0x1FFF)
    return w


def unbias(x):
    """exact fp32 view of a tensor stored pre-biased (out_mode 2); debugging / tests only"""
    return (x.view(torch.int32) - 0x1000).view(torch.float32)


# ------------------------------------------------------------- KITTI evaluation ----
KITTI_ROW, KITTI_T = 16, 41                       # SB_KITTI_ROW, SB_KITTI_MAX_THRESHOLDS


def kitti_overlaps(gt, gt_code, det, gt_off, det_off, pair_off, n_pairs):
    """sb_kitti_overlaps: rows fp64 [n,16], codes int32, CSR offsets int64 [n_images+1] (device), n_pairs =
    pair_off[-1] -> (ov_2d, ov_bev, ov_3d) fp64 [n_pairs], image k's pair (det j, gt i) at pair_off[k] + j * n_gt(k) + i"""
    L = _l.load()
    n_pairs = int(n_pairs)
    dev = gt_off.device
    out = torch.empty(3, max(n_pairs, 1), dtype=torch.float64, device=dev)
    check(L.sb_kitti_overlaps(ptr(gt), ptr(gt_code), ptr(det), ptr(gt_off), ptr(det_off), ptr(pair_off),
                              gt_off.numel() - 1, n_pairs, ptr(out[0]), ptr(out[1]), ptr(out[2]), stream_ptr()),
          "sb_kitti_overlaps")
    return out[0, :n_pairs], out[1, :n_pairs], out[2, :n_pairs]


KITTI_OUTPUTS = (("thresholds", torch.float64, KITTI_T), ("n_thresholds", torch.int32, 0), ("tp", torch.int64, KITTI_T),
                 ("fp", torch.int64, KITTI_T), ("fn", torch.int64, KITTI_T), ("sim", torch.float64, KITTI_T),
                 ("precision", torch.float64, KITTI_T), ("recall", torch.float64, KITTI_T),
                 ("aos", torch.float64, KITTI_T), ("ap", torch.float64, 4), ("n_gt", torch.int64, 0))


def kitti_eval(gt, gt_code, det, det_code, gt_off, det_off, pair_off, n_pairs, bars, out=None):
    """sb_kitti_eval over a packed split (see kitti_overlaps; n_pairs = pair_off[-1], known on the host) ->
    dict of the outputs, configuration c = (metric * len(bars) + bar) * 3 + difficulty.  out: a dict of the same
    tensors to write into (kitti_eval_outputs)"""
    L = _l.load()
    n_images = gt_off.numel() - 1
    ng, nd = gt_code.numel(), det_code.numel()
    dev = gt_off.device
    nb = L.sb_kitti_eval_workspace_bytes(n_images, ng, nd, int(n_pairs), len(bars))
    if nb == 0:
        raise ValueError("sb_kitti_eval refuses these sizes (%d images, %d bars)" % (n_images, len(bars)))
    ws = workspace(nb + 256, dev, "kitti_eval")
    base = (-ws.data_ptr()) % 256
    out = out or kitti_eval_outputs(len(bars), dev)
    b = (ctypes.c_double * len(bars))(*[float(v) for v in bars])
    check(L.sb_kitti_eval(ptr(gt), ptr(gt_code), ptr(det), ptr(det_code), ptr(gt_off), ptr(det_off), ptr(pair_off),
                          n_images, ng, nd, int(n_pairs), b, len(bars), ctypes.c_void_p(ws.data_ptr() + base), nb,
                          *[ptr(out[k]) for k, _t, _n in KITTI_OUTPUTS], stream_ptr()), "sb_kitti_eval")
    return out


KITTI_ANN_IN, KITTI_ANN_OUT, KITTI_ANN_CALIB, KITTI_DEPTH_COLS = 11, 30, 25, 1260  # the SB_KITTI_ANN_* constants


def kitti_annotations(rows, codes, obj_off, calib, image_hw, out=None):
    """sb_kitti_annotations over a packed split: rows fp64 [n,11], codes int32 [n], obj_off int64 [n_images+1], calib
    fp64 [n_images,25], image_hw int32 [n_images,2], all on the device -> (out fp32 [n,30], n_kept int32 [n_images],
    status int32 [n_images]); out: those three tensors to write into"""
    L = _l.load()
    n_images, n = obj_off.numel() - 1, codes.numel()
    dev = obj_off.device
    assert rows.dtype == torch.float64 and codes.dtype == torch.int32 and obj_off.dtype == torch.int64
    assert calib.dtype == torch.float64 and image_hw.dtype == torch.int32
    assert rows.numel() == n * KITTI_ANN_IN and calib.numel() == n_images * KITTI_ANN_CALIB
    assert image_hw.numel() == 2 * n_images
    nb = L.sb_kitti_annotations_workspace_bytes(n_images, n)
    if nb == 0:
        raise ValueError("sb_kitti_annotations refuses these sizes (%d images, %d rows)" % (n_images, n))
    ws = workspace(nb + 256, dev, "kitti_annotations")
    base = (-ws.data_ptr()) % 256
    if out is None:
        out = (torch.empty(max(n, 1), KITTI_ANN_OUT, dtype=torch.float32, device=dev)[:n],
               torch.empty(n_images, dtype=torch.int32, device=dev), torch.empty(n_images, dtype=torch.int32, device=dev))
    assert out[0].shape == (n, KITTI_ANN_OUT) and out[1].numel() == out[2].numel() == n_images
    check(L.sb_kitti_annotations(ptr(rows) if n else None, ptr(codes) if n else None, ptr(obj_off), ptr(calib),
                                 ptr(image_hw), n_images, n, ctypes.c_void_p(ws.data_ptr() + base), nb,
                                 ptr(out[0]) if n else None, ptr(out[1]), ptr(out[2]), stream_ptr()),
          "sb_kitti_annotations")
    return out


def kitti_eval_outputs(n_bars, device):
    """the output tensors of kitti_eval for n_bars bars: views into one device buffer (one D2H copies them all)"""
    C = 9 * n_bars
    sizes = [C * max(n, 1) for _k, _t, n in KITTI_OUTPUTS]
    buf = torch.zeros(sum(sizes), dtype=torch.float64, device=device)
    out, o = {}, 0
    for (k, t, n), s in zip(KITTI_OUTPUTS, sizes):
        v = buf[o:o + s].view(t)
        out[k] = v.view(C, n) if n else v[:C]
        o += s
    out["_buffer"] = buf
    return out
