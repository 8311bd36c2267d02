"""CPU oracle operators -- TEST INFRASTRUCTURE ONLY.

numpy / plain-C restatement of the reference's operators on the Stereo R-CNN
hot path.  Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s
``cpu_baseline`` / ``--impl reference`` legs may import this module; the
product path (``stereo_rcnn_b200``) never does.

Pinning status: NMS / RoIAlign are pinned against the reference's own CUDA
sources compiled unmodified (``oracle/_ref``, GPU tests); anchors, box
decode/clip, the proposal layer and ``dense_align`` are pinned against the
reference's own Python run in the build container through
``oracle/ref_shim.py`` (fixtures in ``tests/golden``).
"""
import ctypes
import os

import numpy as np

from . import build as _build

_lib = None


def lib():
    global _lib
    if _lib is None:
        so = _build.ORACLE_SO
        if not os.path.exists(so):
            so = _build.build_oracle()
        _lib = ctypes.CDLL(so)
        _lib.sb_expf.restype = ctypes.c_float
        _lib.sb_expf.argtypes = [ctypes.c_float]
        _lib.oracle_nms.restype = ctypes.c_int
    return _lib


def _p(a, t=ctypes.c_float):
    return a.ctypes.data_as(ctypes.POINTER(t))


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


# --------------------------------------------------------------------------
# constants the hot path reads from lib/model/utils/config.py
# --------------------------------------------------------------------------
CFG = dict(
    ANCHOR_RATIOS=[0.5, 1, 2],                 # config.py:210
    FPN_ANCHOR_SCALES=[32, 64, 128, 256, 512],  # config.py:216
    FPN_FEAT_STRIDES=[4, 8, 16, 32, 64],        # config.py:219
    FPN_ANCHOR_STRIDE=1,                        # config.py:222
    TEST=dict(RPN_PRE_NMS_TOP_N=6000, RPN_POST_NMS_TOP_N=300, RPN_NMS_THRESH=0.7, NMS=0.3),
    TRAIN=dict(RPN_PRE_NMS_TOP_N=12000, RPN_POST_NMS_TOP_N=2000, RPN_NMS_THRESH=0.7),
    POOLING_SIZE=7, KPTS_GRID=28,
    BBOX_NORMALIZE_MEANS=(0.0, 0.0, 0.0, 0.0), BBOX_NORMALIZE_STDS=(0.1, 0.1, 0.2, 0.2),
    DIM_NORMALIZE_MEANS=(1.6, 1.5, 4.0, 0.0, 0.0), DIM_NORMALIZE_STDS=(0.5, 0.5, 0.5, 0.5, 0.5),
    PIXEL_MEANS=np.array([[[102.9801, 115.9465, 122.7717]]]),
)


def sb_expf(x):
    x = _f32(x)
    y = np.empty_like(x)
    lib().sb_expf_array(_p(x), _p(y), ctypes.c_int(x.size))
    return y


# --------------------------------------------------------------------------
# anchors: lib/model/rpn/generate_anchors.py:112-173 (float64, level->y->x->ratio)
# --------------------------------------------------------------------------
def anchors_all_pyramids(feat_shapes, scales=None, ratios=None, strides=None):
    scales = CFG["FPN_ANCHOR_SCALES"] if scales is None else scales
    ratios = np.asarray(CFG["ANCHOR_RATIOS"] if ratios is None else ratios, dtype=np.float64)
    strides = CFG["FPN_FEAT_STRIDES"] if strides is None else strides
    out = []
    for (h, w), s, st in zip(feat_shapes, scales, strides):
        hs = float(s) / np.sqrt(ratios)           # heights
        ws = float(s) * np.sqrt(ratios)           # widths
        ys = np.arange(0, h, dtype=np.float64) * st
        xs = np.arange(0, w, dtype=np.float64) * st
        cy, cx, _ = np.meshgrid(ys, xs, np.zeros(len(ratios)), indexing="ij")
        bw = np.broadcast_to(ws, cx.shape)
        bh = np.broadcast_to(hs, cx.shape)
        a = np.stack([cx - 0.5 * bw, cy - 0.5 * bh, cx + 0.5 * bw, cy + 0.5 * bh], axis=-1)
        out.append(a.reshape(-1, 4))
    return np.concatenate(out, axis=0)            # float64, caller casts (.type_as(scores))


def decode_clip(boxes, deltas, im_h, im_w):
    """bbox_transform_inv + clip_boxes (bbox_transform.py:79-104,177-185)."""
    boxes, deltas = _f32(boxes), _f32(deltas)
    out = np.empty_like(boxes)
    lib().oracle_decode_clip(_p(boxes), _p(deltas), ctypes.c_int(boxes.shape[0]),
                             ctypes.c_float(im_h), ctypes.c_float(im_w), _p(out))
    return out


# --------------------------------------------------------------------------
# NMS: nms_cuda_kernel.cu:31-161
# --------------------------------------------------------------------------
def nms(dets, thresh):
    dets = _f32(dets)
    n = dets.shape[0]
    keep = np.empty(max(n, 1), dtype=np.int32)
    k = lib().oracle_nms(_p(dets), ctypes.c_int(n), ctypes.c_int(dets.shape[1]),
                         ctypes.c_float(thresh), _p(keep, ctypes.c_int))
    return keep[:k].copy()


def nms_mask(dets, thresh):
    dets = _f32(dets)
    n = dets.shape[0]
    cb = (n + 63) // 64
    mask = np.zeros((n, cb), dtype=np.uint64)
    lib().oracle_nms_mask(_p(dets), ctypes.c_int(n), ctypes.c_int(dets.shape[1]),
                          ctypes.c_float(thresh), _p(mask, ctypes.c_uint64))
    return mask


# --------------------------------------------------------------------------
# proposal layer: lib/model/rpn/proposal_layer.py:42-145 (Q7-Q11 of SURVEY)
# --------------------------------------------------------------------------
def stable_order_desc(scores):
    """total order the oracle pins: score descending as torch.sort(descending=True) ranks it (every NaN above +inf,
    -0.0 equal to +0.0), ties -- NaNs included -- by ascending index"""
    with np.errstate(invalid="ignore"):                    # signalling NaNs quieten on the cast
        s = np.asarray(scores, np.float64).reshape(-1)
    nan = np.isnan(s)
    return np.lexsort((-np.where(nan, 0.0, s), ~nan))     # last key first: NaNs, then -score (stable: index)


def proposal_layer(cls_prob, bbox_pred_lr, im_info, cfg_key, feat_shapes, return_debug=False, pre_nms_top_n=None,
                   post_nms_top_n=None, nms_thresh=None, scales=None, ratios=None, strides=None):
    """cls_prob [B,A,2], bbox_pred_lr [B,A,6], im_info [B,3] -> rois_left/right [B,N,5].  The keyword overrides
    replace CFG[cfg_key]'s RPN_PRE_NMS_TOP_N / RPN_POST_NMS_TOP_N / RPN_NMS_THRESH and the anchor pyramid's
    FPN_ANCHOR_SCALES / ANCHOR_RATIOS / FPN_FEAT_STRIDES."""
    cls_prob, bbox_pred_lr, im_info = _f32(cls_prob), _f32(bbox_pred_lr), _f32(im_info)
    cfg = CFG[cfg_key]
    pre_n = cfg["RPN_PRE_NMS_TOP_N"] if pre_nms_top_n is None else pre_nms_top_n
    post_n = cfg["RPN_POST_NMS_TOP_N"] if post_nms_top_n is None else post_nms_top_n
    thr = cfg["RPN_NMS_THRESH"] if nms_thresh is None else nms_thresh
    B, A = cls_prob.shape[:2]
    anchors = anchors_all_pyramids(feat_shapes, scales, ratios, strides).astype(np.float32)
    assert anchors.shape[0] == A
    out_l = np.zeros((B, post_n, 5), np.float32)
    out_r = np.zeros((B, post_n, 5), np.float32)
    dbg = []
    for b in range(B):
        scores = cls_prob[b, :, 1]
        d = bbox_pred_lr[b]
        dl = d[:, :4].copy()
        dr = d[:, :4].copy()
        dr[:, 0] = d[:, 4]
        dr[:, 2] = d[:, 5]
        order = stable_order_desc(scores)
        if 0 < pre_n < scores.size:
            order = order[:pre_n]
        # decode only the survivors: elementwise op, same values as decoding all then gathering
        pl = decode_clip(anchors[order], dl[order], im_info[b, 0], im_info[b, 1])
        pr = decode_clip(anchors[order], dr[order], im_info[b, 0], im_info[b, 1])
        sc = scores[order][:, None]
        kl = nms(np.concatenate([pl, sc], 1), thr)
        kr = nms(np.concatenate([pr, sc], 1), thr)
        keep = np.intersect1d(kl, kr)
        if post_n > 0:
            keep = keep[:post_n]
        n = keep.size
        out_l[b, :, 0] = b
        out_r[b, :, 0] = b
        out_l[b, :n, 1:] = pl[keep]
        out_r[b, :n, 1:] = pr[keep]
        dbg.append(dict(order=order, prop_l=pl, prop_r=pr, keep_l=kl, keep_r=kr, keep=keep))
    if return_debug:
        return out_l, out_r, dbg
    return out_l, out_r


# --------------------------------------------------------------------------
# RoIAlign: roi_align_kernel.cu:15-143, modules/roi_align.py:26-29
# --------------------------------------------------------------------------
def roi_align_forward(features, rois, ah, aw, scale):
    """features NCHW, rois r x 5, (ah, aw) = lattice size; -> r x C x ah x aw"""
    features, rois = _f32(features), _f32(rois)
    N, C, H, W = features.shape
    R = rois.shape[0]
    out = np.zeros((R, C, ah, aw), np.float32)
    lib().oracle_roi_align_forward(_p(features), N, C, H, W, _p(rois), R, ah, aw,
                                   ctypes.c_float(scale), _p(out))
    return out


def roi_align_backward(top, rois, feat_shape, ah, aw, scale):
    top, rois = _f32(top), _f32(rois)
    N, C, H, W = feat_shape
    R = rois.shape[0]
    bottom = np.zeros((N, C, H, W), np.float32)
    lib().oracle_roi_align_backward(_p(top), N, C, H, W, _p(rois), R, ah, aw,
                                    ctypes.c_float(scale), _p(bottom))
    return bottom


def avg_pool_2x2_s1(x):
    """avg_pool2d(kernel=2, stride=1) (modules/roi_align.py:29)"""
    return ((x[..., :-1, :-1] + x[..., :-1, 1:]) + (x[..., 1:, :-1] + x[..., 1:, 1:])) * np.float32(0.25)


def roi_align_avg(features, rois, ph, pw, scale):
    return avg_pool_2x2_s1(roi_align_forward(features, rois, ph + 1, pw + 1, scale))


def roi_levels(rois):
    """stereo_rcnn.py:113-119: round(ln(sqrt(h*w)/224)+4) clamped to [2,5] (natural log, fp32)"""
    rois = _f32(rois)
    h = rois[:, 4] - rois[:, 2] + np.float32(1)
    w = rois[:, 3] - rois[:, 1] + np.float32(1)
    lv = np.log(np.sqrt(h * w) / np.float32(224.0)).astype(np.float32)
    lv = np.round(lv + np.float32(4))      # torch.round == round-half-even == np.round
    return np.clip(lv, 2, 5).astype(np.int32)


def pyramid_roi_feat(feat_maps, rois, im_h, pooled):
    """PyramidRoI_Feat (stereo_rcnn.py:110-139).  feat_maps: list of NCHW arrays P2..P5."""
    rois = _f32(rois)
    lv = roi_levels(rois)
    C = feat_maps[0].shape[1]
    out = np.zeros((rois.shape[0], C, pooled, pooled), np.float32)
    for i, l in enumerate(range(2, 6)):
        idx = np.nonzero(lv == l)[0]
        if idx.size == 0:
            continue
        scale = np.float32(feat_maps[i].shape[2] / float(im_h))   # python float -> C float arg
        out[idx] = roi_align_avg(feat_maps[i], rois[idx], pooled, pooled, scale)
    return out


# --------------------------------------------------------------------------
# test-time decode: test_net.py:138-212
# --------------------------------------------------------------------------
def test_decode(rois_left, rois_right, cls_prob, bbox_pred, dim_orien_pred,
                kpts_prob, left_prob, right_prob, im_info, n_classes=2):
    """all inputs for one image (leading batch dim of 1 already stripped).

    returns scores [R,nc], pred_boxes_left [R,4nc], pred_boxes_right [R,4nc],
    dim_orien [R,5nc], pred_kpts [R,5]"""
    f = np.float32
    rl, rr = _f32(rois_left)[:, 1:5], _f32(rois_right)[:, 1:5]
    bp = _f32(bbox_pred)
    R = bp.shape[0]
    dl = np.zeros((R, 4 * n_classes), f)
    dr = np.zeros((R, 4 * n_classes), f)
    dl[:, 0::4], dl[:, 1::4], dl[:, 2::4], dl[:, 3::4] = bp[:, 0::6], bp[:, 1::6], bp[:, 2::6], bp[:, 3::6]
    dr[:, 0::4], dr[:, 1::4], dr[:, 2::4], dr[:, 3::4] = bp[:, 4::6], bp[:, 1::6], bp[:, 5::6], bp[:, 3::6]
    stds = np.asarray(CFG["BBOX_NORMALIZE_STDS"], f)
    means = np.asarray(CFG["BBOX_NORMALIZE_MEANS"], f)
    dl = (dl.reshape(-1, 4) * stds + means).reshape(R, -1)
    dr = (dr.reshape(-1, 4) * stds + means).reshape(R, -1)
    do = _f32(dim_orien_pred).reshape(-1, 5) * np.asarray(CFG["DIM_NORMALIZE_STDS"], f) \
        + np.asarray(CFG["DIM_NORMALIZE_MEANS"], f)
    do = do.reshape(R, -1)
    grid = CFG["KPTS_GRID"]
    kp = _f32(kpts_prob)
    kd = np.argmax(kp, 1)
    maxp = kp[np.arange(R), kd]
    ld = np.argmax(_f32(left_prob), 1)
    rd = np.argmax(_f32(right_prob), 1)
    im_h, im_w, sc = f(im_info[0]), f(im_info[1]), f(im_info[2])
    pbl = np.empty((R, 4 * n_classes), f)
    pbr = np.empty((R, 4 * n_classes), f)
    for j in range(n_classes):
        pbl[:, 4 * j:4 * j + 4] = decode_clip(rl, dl[:, 4 * j:4 * j + 4], im_h, im_w)
        pbr[:, 4 * j:4 * j + 4] = decode_clip(rr, dr[:, 4 * j:4 * j + 4], im_h, im_w)
    widths = rl[:, 2] - rl[:, 0] + f(1.0)
    kd_f = kd.astype(f)
    ktype = kd_f / f(grid)                       # bbox_transform.py:139 (float division)
    kdelta = np.fmod(kd_f, f(grid))
    pk = kdelta * widths / f(grid) + rl[:, 0]
    pleft = ld.astype(f) * widths / f(grid) + rl[:, 0]
    pright = rd.astype(f) * widths / f(grid) + rl[:, 0]
    pbl /= sc
    pbr /= sc
    pk, pleft, pright = pk / sc, pleft / sc, pright / sc
    pred_kpts = np.stack([pk, ktype, maxp, pleft, pright], 1).astype(f)
    return _f32(cls_prob), pbl, pbr, do.astype(f), pred_kpts


def per_class_nms(scores, boxes_left, j, thresh=0.05, nms_thresh=None):
    """test_net.py:233-259: threshold, sort desc (stable: index asc), nms; returns indices into RoIs"""
    nms_thresh = CFG["TEST"]["NMS"] if nms_thresh is None else nms_thresh
    inds = np.nonzero(scores[:, j] > np.float32(thresh))[0]
    if inds.size == 0:
        return inds
    cs = scores[inds, j]
    order = stable_order_desc(cs)
    dets = np.concatenate([boxes_left[inds][:, 4 * j:4 * j + 4], cs[:, None]], 1)[order]
    keep = nms(dets, nms_thresh)
    return inds[order][keep]


# --------------------------------------------------------------------------
# dense_align: dense_align.py:13-69,175-300 + box_3d.py
# --------------------------------------------------------------------------
def calib_vec(p2, p3):
    p2, p3 = np.asarray(p2, np.float64), np.asarray(p3, np.float64)
    return np.array([p2[0, 0], p2[0, 2], p2[1, 2], p2[0, 3] - p3[0, 3]], np.float64)


def dense_align(calib, scale, im_left, im_right, box_left, keypoints, poses, diagnostics=False):
    """calib: 4-vector from calib_vec; im_*: [1,3,H,W] or [3,H,W]; returns status[D], best_dis[D]"""
    iml = _f32(im_left).reshape(3, *np.shape(im_left)[-2:])
    imr = _f32(im_right).reshape(3, *np.shape(im_right)[-2:])
    H, W = iml.shape[1:]
    box_left, keypoints, poses = _f32(box_left), _f32(keypoints), _f32(poses)
    D = box_left.shape[0]
    status = np.zeros(D, np.float32)
    best = np.zeros(D, np.float32)
    calib = np.ascontiguousarray(calib, np.float64)
    null = ctypes.c_void_p(0)
    if diagnostics:
        npix = np.zeros(D, np.int32)
        cc = np.zeros((D, 50), np.float64)
        cf = np.zeros((D, 20), np.float64)
        idx = np.zeros((D, 2), np.int32)
        args = (_p(npix, ctypes.c_int), _p(cc, ctypes.c_double), _p(cf, ctypes.c_double),
                _p(idx, ctypes.c_int))
    else:
        args = (null, null, null, null)
    lib().oracle_dense_align(_p(iml), _p(imr), H, W, _p(calib, ctypes.c_double),
                             ctypes.c_double(float(scale)), _p(box_left), _p(keypoints),
                             _p(poses), D, _p(status), _p(best), *args)
    if diagnostics:
        return status, best, dict(npix=npix, cost_coarse=cc, cost_fine=cf, idx=idx)
    return status, best


def dense_sample(calib, scale, H, W, box_left, keypoints, poses, maxp=8192):
    box_left, keypoints, poses = _f32(box_left), _f32(keypoints), _f32(poses)
    D = box_left.shape[0]
    uvz = np.zeros((D, maxp, 3), np.float32)
    npix = np.zeros(D, np.int32)
    calib = np.ascontiguousarray(calib, np.float64)
    lib().oracle_dense_sample(H, W, _p(calib, ctypes.c_double), ctypes.c_double(float(scale)),
                              _p(box_left), _p(keypoints), _p(poses), D, maxp,
                              _p(uvz), _p(npix, ctypes.c_int))
    return uvz, npix


def upsample2x(im):
    im = _f32(im)
    C, H, W = im.shape[-3:]
    out = np.empty((C, 2 * H, 2 * W), np.float32)
    lib().oracle_upsample2x(_p(im), C, H, W, _p(out))
    return out


# --------------------------------------------------------------------------
# input pipeline (SURVEY 8f-3): prep_im_for_blob (lib/model/utils/blob.py:44-64) = BGR - PIXEL_MEANS (fp32), then
# cv2.resize(fx=fy=scale, INTER_LINEAR), then HWC -> CHW (demo.py:124-128, roibatchLoader.py:111-113).
# OpenCV (third-party, unpinned by the reference; 4.13 in this image) resizes float images separably: for each
# output column dx, x = (dx+0.5)/scale - 0.5 in fp64, sx = floor(x), weight = float(x - sx), clamped to the image; a
# horizontal pass a0*S[sx] + a1*S[sx+1] on the two source rows, then the vertical pass b0*row0 + b1*row1, in fp32.
# Pinned empirically against cv2.resize of this image (tests/golden/make_golden.py (8)): <= 2 ulp at any scale
# (cv2's SIMD path contracts some multiply-adds); computing the coordinate in fp32 instead is off by 1e-4 relative.
# --------------------------------------------------------------------------
PIXEL_MEANS = np.array([102.9801, 115.9465, 122.7717], np.float64)       # config.py:170 (BGR)


def _resize_axis(n_src, scale):
    n_dst = int(np.rint(n_src * scale))                 # cv::saturate_cast<int>(ssize * inv_scale) = cvRound
    inv = 1.0 / float(scale)
    x = (np.arange(n_dst, dtype=np.float64) + 0.5) * inv - 0.5
    s = np.floor(x).astype(np.int64)
    f = (x - s).astype(np.float32)
    lo = s < 0
    f[lo], s[lo] = 0.0, 0
    hi = s >= n_src - 1
    f[hi], s[hi] = 0.0, n_src - 1
    s1 = np.minimum(s + 1, n_src - 1)
    return n_dst, s, s1, (np.float32(1.0) - f).astype(np.float32), f


def prep_image(bgr_u8, scale):
    """[H,W,3] uint8 BGR -> [3, round(H*scale), round(W*scale)] fp32 network input (blob.py:44-64 + HWC->CHW)"""
    # `img.astype(np.float32); img -= pixel_means` (float64 means): computed in fp64, stored as fp32
    im = (bgr_u8.astype(np.float32).astype(np.float64) - PIXEL_MEANS).astype(np.float32)
    H, W = im.shape[:2]
    Ho, y0, y1, b0, b1 = _resize_axis(H, scale)
    Wo, x0, x1, a0, a1 = _resize_axis(W, scale)
    rows = (im[:, x0, :] * a0[None, :, None]).astype(np.float32) + (im[:, x1, :] * a1[None, :, None]).astype(np.float32)
    rows = rows.astype(np.float32)
    out = (rows[y0] * b0[:, None, None]).astype(np.float32) + (rows[y1] * b1[:, None, None]).astype(np.float32)
    return np.ascontiguousarray(out.astype(np.float32).transpose(2, 0, 1))
