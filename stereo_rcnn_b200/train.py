"""Train-time target layers and losses of the reference on the device (SURVEY A16 / 8f-4).

Host-side mirror of `_AnchorTargetLayer` (lib/model/rpn/anchor_target_layer.py:42-164), `_ProposalTargetLayer`
(lib/model/rpn/proposal_target_layer.py:36-333), the RPN / RCNN losses (stereo_rpn.py:114-140,
stereo_rcnn.py:201-311), the multi-task sum (trainval_net.py:214-219) and `clip_gradient` (net_utils.py:37-49) over
libstereo_b200's kernels (csrc/train_targets.cu, csrc/train_loss.cu).  No host synchronisation anywhere: counts,
sampled indices and losses stay on the device.  rpn_gradients composes them with the engine's forward and backward
passes into the gradients of the RPN loss for the trunk, the FPN and the RPN, rcnn_head_gradients into the gradients
of the R-CNN loss for the heads, and loss_gradients into the gradients of the whole six-term loss for every trainable
parameter.
"""
import ctypes

import numpy as np
import torch

from . import lib as _l
from .ops import check, ptr, stream_ptr, workspace, _f32c

CFG = dict(                                          # lib/model/utils/config.py:55-108,173
    RPN_NEGATIVE_OVERLAP=0.3, RPN_POSITIVE_OVERLAP=0.7, RPN_FG_FRACTION=0.5, RPN_BATCHSIZE=512,
    BATCH_SIZE=512, FG_FRACTION=0.25, FG_THRESH=0.5, BG_THRESH_HI=0.5, BG_THRESH_LO=0.0,
    BBOX_NORMALIZE_MEANS=(0.0, 0.0, 0.0, 0.0), BBOX_NORMALIZE_STDS=(0.1, 0.1, 0.2, 0.2),
    DIM_NORMALIZE_MEANS=(1.6, 1.5, 4.0, 0.0, 0.0), DIM_NORMALIZE_STDS=(0.5, 0.5, 0.5, 0.5, 0.5),
    KPTS_GRID=28,
)


def random_words(shape, device, generator=None):
    """uint32 random words for the samplers (stored as int32 bit patterns: torch has no uint32 arithmetic)"""
    return torch.randint(-2 ** 31, 2 ** 31, shape, dtype=torch.int32, device=device, generator=generator)


def _words(t):
    assert t.dtype == torch.int32 and t.is_contiguous()
    return t


def fill_random_words(out, seed, step, stream_id):
    """sb_random_words: fill the int32 tensor `out` with Philox4x32-10 words that are a pure function of (seed,
    *step, stream_id, index).  step: int64 [1] device tensor (a uint64 counter), read by the kernel, so a captured fill
    draws new words on every replay once sb_step_advance has run.  In place of the torch.randint of random_words."""
    assert out.dtype == torch.int32 and step.dtype == torch.int64 and step.numel() == 1
    check(_l.load().sb_random_words(int(seed) & (2 ** 64 - 1), ptr(step), int(stream_id), ptr(out), out.numel(),
                                    stream_ptr()), "sb_random_words")
    return out


def step_advance(step):
    """sb_step_advance: *step += 1 on the device (int64 [1])"""
    assert step.dtype == torch.int64 and step.numel() == 1
    check(_l.load().sb_step_advance(ptr(step), stream_ptr()), "sb_step_advance")
    return step


GT_ROW_FIELDS = (("boxes_left", 4), ("boxes_right", 4), ("boxes_merge", 4), ("dim_orien", 4), ("kpts", 6))
MAX_NUM_GT_BOXES = 30                                # config.py:283


def train_gt(rows, n_rows, words, im_scale, im_width, out=None):
    """The ground truth of a step on the device (sb_train_gt: minibatch.py:43-85 + roibatchLoader.py:72-107).
    rows: {"boxes_left" / "boxes_right" / "boxes_merge" [B,N,4], "dim_orien" [B,N,4], "kpts" [B,N,6] fp32,
    "gt_classes" [B,N] int32}, the roidb rows at a fixed capacity N; n_rows [B] int32 (device) rows in use;
    words [B,N] int32 random words that order the kept rows (in place of np.random.shuffle); im_scale, im_width: the
    scale and the width of the blob.  -> (gt_left, gt_right, gt_merge [B,30,5], gt_dim_orien [B,30,5],
    gt_kpts [B,30,6], num_boxes [B] int32), written into `out` when given"""
    L = _l.load()
    B, N = rows["gt_classes"].shape
    dev = words.device
    assert rows["gt_classes"].dtype == torch.int32 and n_rows.dtype == torch.int32 and n_rows.numel() == B
    assert all(rows[k].shape == (B, N, w) and rows[k].dtype == torch.float32 for k, w in GT_ROW_FIELDS)
    assert _words(words).shape == (B, N)
    if out is None:
        out = tuple(torch.empty(B, MAX_NUM_GT_BOXES, w, dtype=torch.float32, device=dev) for w in (5, 5, 5, 5, 6)) + \
            (torch.empty(B, dtype=torch.int32, device=dev),)
    assert [tuple(o.shape[1:]) for o in out[:5]] == [(30, 5)] * 4 + [(30, 6)] and out[5].dtype == torch.int32
    check(L.sb_train_gt(ptr(rows["boxes_left"]), ptr(rows["boxes_right"]), ptr(rows["boxes_merge"]),
                        ptr(rows["gt_classes"]), ptr(rows["dim_orien"]), ptr(rows["kpts"]), ptr(n_rows), ptr(words),
                        B, N, float(im_scale), int(im_width), *[ptr(o) for o in out], stream_ptr()), "sb_train_gt")
    return out


def _mirror_cols(a, cols_from, cols_to, width):
    out = a.astype(np.float32).copy()
    out[:, cols_to] = (np.float32(width) - a[:, cols_from].astype(np.float32)) - np.float32(1)
    return out


def append_flipped(roidb, widths):
    """imdb.append_flipped_images (imdb.py:117-176) in numpy, once at start-up: roidb + the flip of every entry.  The
    flip swaps the sides and mirrors the boxes (x1 = width - x2 - 1, x2 = width - x1 - 1), reflects theta (wrapped
    into [-pi, pi] first) and takes the keypoints from `kpts_right` in the order (3, 2, 1, 0, 5, 4), all in float32.
    The flipped entry keeps every other key of the entry and carries `kpts_right` (the mirror of `kpts`), so the
    flip of a flip gives the first entry's geometry back.  The frames are not touched: sb_prep_stereo_pair mirrors
    them on the device for an entry with `flipped` set."""
    import math
    pi, two_pi = np.float32(math.pi), np.float32(2.0 * math.pi)
    out = list(roidb)
    for e, w in zip(roidb, widths):
        f = dict(e)
        for dst, src in (("boxes_left", "boxes_right"), ("boxes_right", "boxes_left"), ("boxes_merge", "boxes_merge")):
            f[dst] = _mirror_cols(e[src], [2, 0], [0, 2], w)
            assert (f[dst][:, 2] >= f[dst][:, 0]).all()
        d = e["dim_orien"].astype(np.float32).copy()
        t = d[:, 3]
        t = np.where(t > pi, t - two_pi, t)
        t = np.where(t < -pi, t + two_pi, t)
        d[:, 3] = np.where(t >= 0, pi - t, -pi - t)
        f["dim_orien"] = d
        f["kpts"] = _mirror_cols(e["kpts_right"], [3, 2, 1, 0, 5, 4], list(range(6)), w)
        f["kpts_right"] = _mirror_cols(e["kpts"], [3, 2, 1, 0, 5, 4], list(range(6)), w)
        f["flipped"] = not e.get("flipped", False)
        out.append(f)
    return out


def generate_anchors(feat_shapes, device, ratios=None, scales=None, strides=None):
    """generate_anchors_all_pyramids (generate_anchors.py:157-173) on the device -> [A,4] fp32"""
    from .ops import make_proposal_cfg
    L = _l.load()
    pc = make_proposal_cfg("TRAIN", [list(map(int, s)) for s in feat_shapes], ratios=ratios, scales=scales, strides=strides)
    A = sum(int(h) * int(w) for h, w in feat_shapes) * pc.n_ratios
    out = torch.empty(A, 4, dtype=torch.float32, device=device)
    check(L.sb_generate_anchors(ctypes.byref(pc), A, ptr(out), stream_ptr()), "sb_generate_anchors")
    return out


def anchor_targets(anchors, gt_left, gt_right, gt_merge, im_info, keys, cfg=CFG):
    """_AnchorTargetLayer.forward: anchors [A,4] fp32, gt_* [B,K,5], im_info = (H, W, ...) of image 0 as Python
    numbers, keys [B,A] int32 words -> labels [B,A], targets_left [B,A,4], targets_right [B,A,4], inside_w [B,A],
    outside_w [B,A]"""
    L = _l.load()
    A = anchors.shape[0]
    B, K = gt_left.shape[:2]
    dev = anchors.device
    assert keys.shape == (B, A)
    labels = torch.empty(B, A, dtype=torch.float32, device=dev)
    tl = torch.empty(B, A, 4, dtype=torch.float32, device=dev)
    tr = torch.empty(B, A, 4, dtype=torch.float32, device=dev)
    iw = torch.empty(B, A, dtype=torch.float32, device=dev)
    ow = torch.empty(B, A, dtype=torch.float32, device=dev)
    nbytes = L.sb_anchor_targets_workspace(B, A)
    ws = workspace(nbytes, dev, "anchor_targets")
    num_fg = int(cfg["RPN_FG_FRACTION"] * cfg["RPN_BATCHSIZE"])
    check(L.sb_anchor_targets(ptr(_f32c(anchors)), A, ptr(_f32c(gt_left)), ptr(_f32c(gt_right)), ptr(_f32c(gt_merge)),
                              B, K, int(im_info[0]), int(im_info[1]), ptr(_words(keys)),
                              float(cfg["RPN_NEGATIVE_OVERLAP"]), float(cfg["RPN_POSITIVE_OVERLAP"]),
                              int(cfg["RPN_BATCHSIZE"]), num_fg, ptr(ws), nbytes, ptr(labels), ptr(tl), ptr(tr),
                              ptr(iw), ptr(ow), stream_ptr()), "sb_anchor_targets")
    return labels, tl, tr, iw, ow


def _pt_cfg(cfg):
    c = _l.ProposalTargetCfg()
    c.rois_per_image = int(cfg["BATCH_SIZE"])
    c.fg_rois_per_image = int(np.round(cfg["FG_FRACTION"] * cfg["BATCH_SIZE"]))
    c.fg_thresh, c.bg_thresh_hi, c.bg_thresh_lo = cfg["FG_THRESH"], cfg["BG_THRESH_HI"], cfg["BG_THRESH_LO"]
    c.bbox_means = (ctypes.c_float * 4)(*cfg["BBOX_NORMALIZE_MEANS"])
    c.bbox_stds = (ctypes.c_float * 4)(*cfg["BBOX_NORMALIZE_STDS"])
    c.dim_means = (ctypes.c_float * 5)(*cfg["DIM_NORMALIZE_MEANS"])
    c.dim_stds = (ctypes.c_float * 5)(*cfg["DIM_NORMALIZE_STDS"])
    c.kpts_grid = int(cfg["KPTS_GRID"])
    return c


def proposal_targets(rois_left, rois_right, gt_left, gt_right, gt_dim_orien, gt_kpts, keys, words, cfg=CFG):
    """_ProposalTargetLayer.forward: rois_* [B,R,5], gt_* [B,K,5], gt_dim_orien [B,K,5], gt_kpts [B,K,6],
    keys [B,R+K] / words [B,S] int32 random words -> dict like oracle.train_targets.proposal_target_layer
    (kpts_targets int32, plus status [B])"""
    L = _l.load()
    B, R = rois_left.shape[:2]
    K = gt_left.shape[1]
    S = int(cfg["BATCH_SIZE"])
    dev = rois_left.device
    assert keys.shape == (B, R + K) and words.shape == (B, S)
    f = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
    o = dict(rois_left=f(B, S, 5), rois_right=f(B, S, 5), labels=f(B, S), bbox_targets_left=f(B, S, 4),
             bbox_targets_right=f(B, S, 4), dim_orien_targets=f(B, S, 5),
             kpts_targets=torch.empty(B, S, 3, dtype=torch.int32, device=dev), kpts_weight=f(B, S, 3),
             inside_w=f(B, S, 4), outside_w=f(B, S, 4),
             keep_inds=torch.empty(B, S, dtype=torch.int32, device=dev),
             status=torch.empty(B, dtype=torch.int32, device=dev))
    c = _pt_cfg(cfg)
    check(L.sb_proposal_targets(ptr(_f32c(rois_left)), ptr(_f32c(rois_right)), B, R, ptr(_f32c(gt_left)),
                                ptr(_f32c(gt_right)), ptr(_f32c(gt_dim_orien)), ptr(_f32c(gt_kpts)), K,
                                ptr(_words(keys)), ptr(_words(words)), ctypes.byref(c), ptr(o["rois_left"]),
                                ptr(o["rois_right"]), ptr(o["labels"]), ptr(o["bbox_targets_left"]),
                                ptr(o["bbox_targets_right"]), ptr(o["dim_orien_targets"]), ptr(o["kpts_targets"]),
                                ptr(o["kpts_weight"]), ptr(o["inside_w"]), ptr(o["outside_w"]), ptr(o["keep_inds"]),
                                ptr(o["status"]), stream_ptr()), "sb_proposal_targets")
    return o


def rpn_loss(rpn_cls_score, rpn_bbox_pred, labels, targets_left, targets_right, inside_w, outside_w, uncert=None,
             grads=True):
    """stereo_rpn.py:114-140: rpn_cls_score [B,A,2], rpn_bbox_pred [B,A,6] -> losses [2] (cls, box) and, with grads,
    d loss / d rpn_cls_score, d loss / d rpn_bbox_pred (times exp(-uncert[0..1]) if uncert is given)"""
    L = _l.load()
    B, A = labels.shape
    dev = labels.device
    losses = torch.empty(2, dtype=torch.float32, device=dev)
    d_cls = torch.empty_like(rpn_cls_score) if grads else None
    d_box = torch.empty_like(rpn_bbox_pred) if grads else None
    nbytes = L.sb_loss_workspace_bytes()
    ws = workspace(nbytes, dev, "loss")
    check(L.sb_rpn_loss(ptr(_f32c(rpn_cls_score)), ptr(_f32c(rpn_bbox_pred)), ptr(_f32c(labels)),
                        ptr(_f32c(targets_left)), ptr(_f32c(targets_right)), ptr(_f32c(inside_w)),
                        ptr(_f32c(outside_w)), B, A, ptr(uncert) if uncert is not None else None, ptr(ws), nbytes,
                        ptr(losses), ptr(d_cls) if grads else None, ptr(d_box) if grads else None, stream_ptr()),
          "sb_rpn_loss")
    return (losses, d_cls, d_box) if grads else losses


def rcnn_loss(cls_score, bbox_pred, dim_orien_pred, kpts_pred, left_border_pred, right_border_pred, tgt, uncert=None,
              grads=True, kpts_grid=28):
    """stereo_rcnn.py:201-311: predictions of the R = B*S sampled RoIs (bbox_pred [R,6C], dim_orien_pred [R,5C] per
    class), tgt = proposal_targets(...) -> losses [4] (cls, bbox, dim_orien, kpts) and, with grads, the six gradients"""
    L = _l.load()
    R, C = cls_score.shape
    dev = cls_score.device
    losses = torch.empty(4, dtype=torch.float32, device=dev)
    preds = [_f32c(t) for t in (cls_score, bbox_pred, dim_orien_pred, kpts_pred, left_border_pred, right_border_pred)]
    g = [torch.empty_like(t) for t in preds] if grads else [None] * 6
    check(L.sb_rcnn_loss(*[ptr(t) for t in preds], ptr(_f32c(tgt["labels"])), ptr(_f32c(tgt["bbox_targets_left"])),
                         ptr(_f32c(tgt["bbox_targets_right"])), ptr(_f32c(tgt["dim_orien_targets"])),
                         ptr(tgt["kpts_targets"]), ptr(_f32c(tgt["kpts_weight"])), ptr(_f32c(tgt["inside_w"])),
                         ptr(_f32c(tgt["outside_w"])), R, C, kpts_grid, ptr(uncert) if uncert is not None else None,
                         ptr(losses), *[ptr(t) if t is not None else None for t in g], stream_ptr()), "sb_rcnn_loss")
    return (losses, g) if grads else losses


def multitask_loss(losses, uncert, total=None, d_uncert=None):
    """trainval_net.py:214-219: losses [n], uncert [n] -> total [1], d total / d uncert [n] (written into `total` /
    `d_uncert` when given)"""
    L = _l.load()
    n = losses.numel()
    total = torch.empty(1, dtype=torch.float32, device=losses.device) if total is None else total
    d_u = torch.empty(n, dtype=torch.float32, device=losses.device) if d_uncert is None else d_uncert
    assert total.is_contiguous() and d_u.is_contiguous() and d_u.numel() == n
    check(L.sb_multitask_loss(ptr(_f32c(losses)), ptr(_f32c(uncert)), n, ptr(total), ptr(d_u), stream_ptr()),
          "sb_multitask_loss")
    return total, d_u


def clip_gradient(grads, clip_norm, out=None):
    """net_utils.clip_gradient over a list of fp32 gradient tensors, in place -> norm [2] (total norm, factor; written
    into `out` when given)"""
    L = _l.load()
    n = len(grads)
    dev = grads[0].device
    assert all(g.dtype == torch.float32 and g.is_contiguous() for g in grads)
    ptrs = (ctypes.c_void_p * n)(*[g.data_ptr() for g in grads])
    counts = (ctypes.c_size_t * n)(*[g.numel() for g in grads])
    nbytes = L.sb_clip_gradient_workspace(n)
    ws = workspace(nbytes, dev, "clip")
    out = torch.empty(2, dtype=torch.float32, device=dev) if out is None else out
    assert out.dtype == torch.float32 and out.is_contiguous() and out.numel() == 2
    check(L.sb_clip_gradient(ptrs, counts, n, float(clip_norm), ptr(ws), nbytes, ptr(out), stream_ptr()),
          "sb_clip_gradient")
    return out


def rpn_gradients(engine, im_left, im_right, gt_left, gt_right, gt_merge, keys, uncert=None, fixed_blocks=1,
                  grads=None, grad_scale=1.0):
    """The RPN loss of a stereo pair differentiated end to end on the device (stereo_rpn.py:114-140 through
    stereo_rpn.py:73-95 and the trunk + FPN): trunk_fpn and rpn with save_for_backward, the anchor targets for
    `keys` (anchor_targets), rpn_loss, then rpn_backward and trunk_fpn_backward(fixed_blocks).
    im_left / im_right [B,3,H,W] NCHW fp32 network inputs, gt_* [B,K,5], keys [B,A] int32 words.
    Returns (losses [2] = (rpn_loss_cls, rpn_loss_box), {state_dict name: fp32 gradient} of
    trainable_trunk_fpn_params(fixed_blocks) + trainable_rpn_params()) and, with uncert [>= 2] (the multi-task
    weights of trainval_net.py:214-219), d total / d uncert[0:2] as a third item; the gradients are then those of
    losses[i] * exp(-uncert[i]).  grads / grad_scale as in rpn_backward; engine.found_inf covers both backward
    passes.  No optimizer step, no host synchronisation."""
    B, _, H, W = im_left.shape
    with torch.no_grad():
        im = torch.cat((im_left, im_right), 0).contiguous()
        feats, saved_t = engine.trunk_fpn(im, save_for_backward=True)
        _cls_prob, bbox, shapes, saved_r, score = engine.rpn(feats, B, save_for_backward=True)
        anchors = generate_anchors(shapes, im.device)
        labels, tl, tr, iw, ow = anchor_targets(anchors, gt_left, gt_right, gt_merge, (H, W), keys)
        u = uncert[0:2] if uncert is not None else None
        losses, d_cls, d_box = rpn_loss(score, bbox, labels, tl, tr, iw, ow, uncert=u)
        g, dp = engine.rpn_backward(saved_r, d_cls, d_box, grads=grads, grad_scale=grad_scale)
        g.update(engine.trunk_fpn_backward(saved_t, dp, fixed_blocks=fixed_blocks, grads=grads, grad_scale=grad_scale,
                                           clear_found_inf=False))
        if uncert is None:
            return losses, g
        _total, d_u = multitask_loss(losses, u)
        return losses, g, d_u


_IM_INFO = {}


def _im_info(B, H, W, device):
    """im_info [B,3] = (H, W, 1) on the device, built once per (device, B, H, W): later calls, and CUDA graphs captured
    after a first eager call, read the same tensor (the proposal layer reads only H and W)"""
    key = (str(device), B, H, W)
    if key not in _IM_INFO:
        _IM_INFO[key] = torch.tensor([[float(H), float(W), 1.0]] * B, dtype=torch.float32).to(device)
    return _IM_INFO[key]


def rcnn_head_gradients(engine, im_left, im_right, gt_left, gt_right, gt_merge, gt_dim_orien, gt_kpts, keys, words,
                        dropout_words=None, uncert=None, grads=None, grad_scale=1.0):
    """The R-CNN loss of a stereo pair differentiated through the heads on a frozen trunk and RPN
    (stereo_rcnn.py:198-311): trunk_fpn and rpn (no gradient), proposal_layer(..., "TRAIN"), proposal_targets for
    `keys` [B,R+K] / `words` [B,S], heads(save_for_backward=True) on the S sampled RoIs per image, rcnn_loss, then
    heads_backward.  im_left / im_right [B,3,H,W] NCHW fp32 network inputs, gt_* [B,K,5], gt_dim_orien [B,K,5],
    gt_kpts [B,K,6]; gt_merge is part of the ground truth of a step but only the RPN's targets read it.
    dropout_words (int32 [2,B*S,2048], random_words): RCNN_top's training-mode dropout (engine.heads).
    Returns (losses [4] = (RCNN_loss_cls, RCNN_loss_bbox, RCNN_loss_dim_orien, RCNN_loss_kpts),
    {state_dict name: fp32 gradient} of trainable_rcnn_head_params(n_classes),
    {"pooled_box": [B*S,7,7,512], "pooled_kpts": [B*S,14,14,256]} fp32 gradients of the pooled features) and, with
    uncert [6] (the multi-task weights of trainval_net.py:214-219; uncert[2:6] weight these four losses),
    d total / d uncert[2:6] as a fourth item; the gradients are then those of losses[i] * exp(-uncert[2 + i]).
    grads / grad_scale as in heads_backward.  No optimizer step, no host synchronisation."""
    B, _, H, W = im_left.shape
    with torch.no_grad():
        im = torch.cat((im_left, im_right), 0).contiguous()
        feats = engine.trunk_fpn(im)
        cls_prob, bbox, shapes = engine.rpn(feats, B)
        from .ops import proposal_layer
        rl, rr = proposal_layer(cls_prob, bbox, _im_info(B, H, W, im.device), "TRAIN", shapes)
        tgt = proposal_targets(rl, rr, gt_left, gt_right, gt_dim_orien, gt_kpts, keys, words)
        out, saved = engine.heads(feats, B, tgt["rois_left"].view(-1, 5), tgt["rois_right"].view(-1, 5), float(H),
                                  save_for_backward=True, dropout_words=dropout_words)
        # sb_rcnn_loss reads uncert[2..5] of the whole vector
        losses, g = rcnn_loss(out["cls_score"], out["bbox_pred"], out["dim_orien_pred"], out["kpts_pred"],
                              out["left_border_pred"], out["right_border_pred"], tgt, uncert=uncert)
        hg, dpooled = engine.heads_backward(saved, *g, grads=grads, grad_scale=grad_scale)
        if uncert is None:
            return losses, hg, dpooled
        assert uncert.numel() >= 6
        _total, d_u = multitask_loss(losses, uncert[2:6])
        return losses, hg, dpooled, d_u


def loss_gradients(engine, im_left, im_right, gt_left, gt_right, gt_merge, gt_dim_orien, gt_kpts, keys, words,
                   rpn_keys, dropout_words=None, uncert=None, fixed_blocks=1, grads=None, grad_scale=1.0,
                   total=None, d_uncert=None):
    """The whole training loss of a stereo pair (trainval_net.py:214-219) differentiated end to end on the device, each
    step once: trunk_fpn and rpn with save_for_backward, the anchor targets for `rpn_keys` [B,A] and rpn_loss,
    proposal_layer(..., "TRAIN") and proposal_targets for `keys` [B,R+K] / `words` [B,S], heads(save_for_backward=True,
    dropout_words) and rcnn_loss, then rpn_backward, heads_backward, roi_align_backward of the pooled gradients into the
    RPN's dP2..dP5, and trunk_fpn_backward(fixed_blocks).  Arguments as rpn_gradients and rcnn_head_gradients.
    Returns (losses [6] = (rpn_loss_cls, rpn_loss_box, RCNN_loss_cls, RCNN_loss_bbox, RCNN_loss_dim_orien,
    RCNN_loss_kpts), {state_dict name: fp32 gradient} of trainable_trunk_fpn_params(fixed_blocks) +
    trainable_rpn_params() + trainable_rcnn_head_params(n_classes)) and, with uncert [6], d total / d uncert [6] as a
    third item; the gradients are then those of total = sum_i losses[i] exp(-uncert[i]) + uncert[i].
    grads / grad_scale as in the backward passes; engine.found_inf is cleared once and covers every backward pass.
    total [1] / d_uncert [6] (with uncert): fp32 device tensors that receive the multi-task total and d total /
    d uncert in place.  No optimizer step, no host synchronisation."""
    B, _, H, W = im_left.shape
    with torch.no_grad():
        im = torch.cat((im_left, im_right), 0).contiguous()
        feats, saved_t = engine.trunk_fpn(im, save_for_backward=True)
        cls_prob, bbox, shapes, saved_r, score = engine.rpn(feats, B, save_for_backward=True)
        anchors = generate_anchors(shapes, im.device)
        labels, tl, tr, iw, ow = anchor_targets(anchors, gt_left, gt_right, gt_merge, (H, W), rpn_keys)
        rpn_losses, d_cls, d_box = rpn_loss(score, bbox, labels, tl, tr, iw, ow,
                                            uncert=uncert[0:2] if uncert is not None else None)
        from .ops import proposal_layer
        rl, rr = proposal_layer(cls_prob, bbox, _im_info(B, H, W, im.device), "TRAIN", shapes)
        tgt = proposal_targets(rl, rr, gt_left, gt_right, gt_dim_orien, gt_kpts, keys, words)
        out, saved_h = engine.heads(feats, B, tgt["rois_left"].view(-1, 5), tgt["rois_right"].view(-1, 5), float(H),
                                    save_for_backward=True, dropout_words=dropout_words)
        # sb_rcnn_loss reads uncert[2..5] of the whole vector
        rcnn_losses, g = rcnn_loss(out["cls_score"], out["bbox_pred"], out["dim_orien_pred"], out["kpts_pred"],
                                   out["left_border_pred"], out["right_border_pred"], tgt, uncert=uncert)
        grad, dp = engine.rpn_backward(saved_r, d_cls, d_box, grads=grads, grad_scale=grad_scale)
        hg, dpooled = engine.heads_backward(saved_h, *g, grads=grads, grad_scale=grad_scale, clear_found_inf=False)
        grad.update(hg)
        engine.roi_align_backward(saved_h, dpooled, dp)
        grad.update(engine.trunk_fpn_backward(saved_t, dp, fixed_blocks=fixed_blocks, grads=grads,
                                              grad_scale=grad_scale, clear_found_inf=False))
        losses = torch.cat((rpn_losses, rcnn_losses))
        if uncert is None:
            return losses, grad
        assert uncert.numel() >= 6
        _total, d_u = multitask_loss(losses, uncert[0:6], total=total, d_uncert=d_uncert)
        return losses, grad, d_u


# ------------------------------------------------------------------------------------------------ the training step
def _f32_ptrs(ts):
    assert all(t.dtype == torch.float32 and t.is_contiguous() and t.is_cuda for t in ts)
    return (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


class _SgdArgs(object):
    """the host arrays of one sb_sgd_step table (built once, reused by every step)"""

    def __init__(self, params, grads, moms, weight_decay, lr_mult):
        n = len(params)
        assert len(grads) == n and len(moms) == n and len(weight_decay) == n and len(lr_mult) == n
        for p, g, m in zip(params, grads, moms):
            assert p.shape == g.shape == m.shape
        self.n, self.keep = n, (list(params), list(grads), list(moms))
        self.p, self.g, self.m = _f32_ptrs(params), _f32_ptrs(grads), _f32_ptrs(moms)
        self.counts = (ctypes.c_size_t * n)(*[p.numel() for p in params])
        self.wd = (ctypes.c_float * n)(*[float(w) for w in weight_decay])
        self.lrm = (ctypes.c_float * n)(*[float(m) for m in lr_mult])

    def __call__(self, lr, momentum, skip, skipped):
        L = _l.load()
        assert lr.dtype == torch.float32 and skip.dtype == torch.int32 and skipped.dtype == torch.int32
        check(L.sb_sgd_step(self.p, self.g, self.m, self.counts, self.wd, self.lrm, self.n, ptr(lr), float(momentum),
                            ptr(skip), ptr(skipped), stream_ptr()), "sb_sgd_step")


def sgd_step(params, grads, moms, lr, momentum, weight_decay, lr_mult, skip, skipped):
    """torch.optim.SGD.step (dampening 0, no Nesterov) over lists of fp32 device tensors, in place (sb_sgd_step):
    per element d = g + wd p, m = momentum m + d, p = p - (lr lr_mult) m, each an fp32 operation rounded to nearest.
    lr: fp32 [1] device tensor; weight_decay / lr_mult: one float per tensor; momentum buffers start at zero.
    skip (int32 [1], device; e.g. engine.found_inf): when set nothing is written and skipped (int32 [1]) is
    incremented.  No host synchronisation.  -> skipped"""
    _SgdArgs(params, grads, moms, weight_decay, lr_mult)(lr, momentum, skip, skipped)
    return skipped


LOSS_SCALE_MIN, LOSS_SCALE_MAX = 2.0 ** -32, 2.0 ** 32      # sb_loss_scale_update's bounds


def _fp32_power_of_two(v):
    """v is a positive power of two that float32 holds exactly"""
    v = float(v)
    return v > 0 and np.isfinite(v) and ctypes.c_float(v).value == v and np.frexp(v)[0] == 0.5


class DynamicLossScale(object):
    """torch.cuda.amp.GradScaler's dynamic loss scale for Trainer(grad_scale=DynamicLossScale(...)): the scale starts at
    init_scale; a step whose backward raised found_inf multiplies it by backoff_factor, growth_interval steps in a row
    without one multiply it by growth_factor (sb_loss_scale_update).  The scale stays within [2^-32, 2^32]: the fp16
    chain spans about 2^-24..2^16, so no useful scale lies outside, and power-of-two factors keep the scale and its
    reciprocal exact.  The constructor raises ValueError for an init_scale that is not a power of two in
    [LOSS_SCALE_MIN, LOSS_SCALE_MAX], factors that are not powers of two, growth_factor <= 1, backoff_factor >= 1 or
    growth_interval < 1."""

    def __init__(self, init_scale=2.0 ** 16, growth_factor=2.0, backoff_factor=0.5, growth_interval=2000):
        if not _fp32_power_of_two(init_scale) or not LOSS_SCALE_MIN <= float(init_scale) <= LOSS_SCALE_MAX:
            raise ValueError("init_scale must be a power of two in [2^-32, 2^32], got %r" % (init_scale,))
        if not _fp32_power_of_two(growth_factor) or not float(growth_factor) > 1.0:
            raise ValueError("growth_factor must be a power of two > 1, got %r" % (growth_factor,))
        if not _fp32_power_of_two(backoff_factor) or not float(backoff_factor) < 1.0:
            raise ValueError("backoff_factor must be a power of two < 1, got %r" % (backoff_factor,))
        if int(growth_interval) != growth_interval or int(growth_interval) < 1:
            raise ValueError("growth_interval must be an integer >= 1, got %r" % (growth_interval,))
        self.init_scale, self.growth_factor = float(init_scale), float(growth_factor)
        self.backoff_factor, self.growth_interval = float(backoff_factor), int(growth_interval)

    def __repr__(self):
        return "DynamicLossScale(init_scale=%g, growth_factor=%g, backoff_factor=%g, growth_interval=%d)" % (
            self.init_scale, self.growth_factor, self.backoff_factor, self.growth_interval)


def loss_scale_update(found_inf, scale, growth_tracker, growth_factor=2.0, backoff_factor=0.5, growth_interval=2000):
    """torch._amp_update_scale_ on the device (sb_loss_scale_update), in place: found_inf / growth_tracker int32 [1],
    scale fp32 [1], all CUDA tensors.  No host synchronisation.  -> scale"""
    L = _l.load()
    assert found_inf.dtype == torch.int32 and growth_tracker.dtype == torch.int32 and scale.dtype == torch.float32
    check(L.sb_loss_scale_update(ptr(found_inf), ptr(scale), ptr(growth_tracker), float(growth_factor),
                                 float(backoff_factor), int(growth_interval), stream_ptr()), "sb_loss_scale_update")
    return scale


def trainable_names(fixed_blocks=1, n_classes=2):
    """[(name, shape)] of every trainable tensor of the model in the order loss_gradients produces them"""
    from . import engine as E
    return (E.trainable_trunk_fpn_params(fixed_blocks) + E.trainable_rpn_params() +
            E.trainable_rcnn_head_params(n_classes))


def param_groups(names, weight_decay=1e-4, double_bias=False, bias_decay=False):
    """trainval_net.py:158-166 per tensor -> [(lr_mult, weight_decay)]: a name containing 'bias' gets
    lr (DOUBLE_BIAS + 1) and weight decay only with BIAS_DECAY, any other weight_decay; "uncert" gets lr and no
    decay"""
    out = []
    for n in names:
        if n == "uncert":
            out.append((1.0, 0.0))
        elif "bias" in n:
            out.append((float(int(double_bias) + 1), float(bias_decay and weight_decay or 0)))
        else:
            out.append((1.0, float(weight_decay)))
    return out


def state_buckets(shapes, device, world=1, dist=None):
    """master parameters, gradients and momentum buffers as three parallel.GradientBuckets over the same shapes:
    one bucket plan, so view i sits at the same bucket and offset in all three.  All start at zero."""
    from .parallel import GradientBuckets
    return tuple(GradientBuckets(shapes, device, world=world, dist=dist) for _ in range(3))


class Trainer(object):
    """The training step of trainval_net.py:198-227 on the device: loss_gradients, the data-parallel gradient
    average, clip_gradient over the model's gradients, SGD with momentum, then the engine's packed weights refreshed
    in place from the updated masters.

    Masters, gradients and momentum live in three GradientBuckets with one plan; the last view of each is `uncert`
    [6] (trainval_net.py:155-156, initialised to -1), which is optimised with lr and no decay and is not clipped
    (net_utils.py:37-49 walks the model's parameters only).  A step whose backward raised engine.found_inf (grad_scale
    overflow) writes no master, momentum or packed weight and counts itself in `skipped`: GradScaler's skip, the one
    deliberate difference from the reference.  The defaults are the reference's (config.py:22-46,
    trainval_net.py:153-168,226).  `engine` must have been built from `state_dict` (fp16 operands); the constructor
    uploads the refresh table and synchronises once.  At world > 1 `rank` is dist.get_rank(), otherwise 0.

    grad_scale is either a host float, the same constant loss scale in every step, or a DynamicLossScale.  A dynamic
    scale lives on the device: `loss_scale` (fp32 [1]) and `growth_tracker` (int32 [1]).  Every backward kernel reads
    the scale there and the unscale vectors are its reciprocal computed on the device, so a captured step follows the
    scale from replay to replay.  After the SGD step (skipped on found_inf) and the weight refresh, the step runs
    sb_loss_scale_update on the same found_inf -- at world > 1 the flag already reduced over the ranks, so every rank
    holds the same scale without another collective: an overflow halves the scale (backoff_factor), growth_interval
    clean steps in a row double it (growth_factor).  Steps skipped while the scale backs off are counted in
    `skipped`."""

    def __init__(self, engine, state_dict, fixed_blocks=1, lr=1e-3, momentum=0.9, weight_decay=1e-4,
                 double_bias=False, bias_decay=False, clip_norm=10.0, grad_scale=1.0, world=1, dist=None, seed=0):
        self.engine, self.fixed_blocks, self.momentum = engine, int(fixed_blocks), float(momentum)
        self.clip_norm, self.world, self.dist = float(clip_norm), int(world), dist
        self.rank = int(dist.get_rank()) if self.world > 1 and dist is not None else 0
        dev = engine.device
        self.dynamic = grad_scale if isinstance(grad_scale, DynamicLossScale) else None
        if self.dynamic is not None:
            self.loss_scale = torch.full((1,), self.dynamic.init_scale, dtype=torch.float32, device=dev)
            self.growth_tracker = torch.zeros(1, dtype=torch.int32, device=dev)
            self.grad_scale = self.loss_scale
        else:
            self.grad_scale = float(grad_scale)
        named = trainable_names(fixed_blocks, engine.n_classes)
        self.names = [n for n, _ in named]
        self.masters, self.grads, self.moms = state_buckets([s for _, s in named] + [(6,)], dev, world, dist)
        self._sd = {k: v.detach().cpu() for k, v in state_dict.items()}
        with torch.no_grad():
            for n, v in zip(self.names, self.masters.grads):
                v.copy_(self._sd[n].to(torch.float32))
            self.masters.grads[-1].copy_(torch.full((6,), -1.0))
        self.params = dict(zip(self.names, self.masters.grads))
        self.uncert = self.masters.grads[-1]
        self.grad_views = dict(zip(self.names, self.grads.grads))
        self.groups = param_groups(self.names + ["uncert"], weight_decay, double_bias, bias_decay)
        self._sgd = _SgdArgs(self.masters.grads, self.grads.grads, self.moms.grads, [g[1] for g in self.groups],
                             [g[0] for g in self.groups])
        f32 = lambda n: torch.zeros(n, dtype=torch.float32, device=dev)
        self.lr = f32(1)
        self.total, self.norm = f32(1), f32(2)
        self.skipped = torch.zeros(4, dtype=torch.int32, device=dev)[:1]
        # step_from_frames: the key of the step's random words and the device-side count of the steps taken
        self.seed, self.step_count = int(seed), torch.zeros(1, dtype=torch.int64, device=dev)
        self.epoch, self.sampler_state = 1, None     # the next epoch of fit and the state of its host generator
        self.val_summaries = {}                      # fit(val=...): {epoch: evaluate's summary without "curves"}
        self.set_lr(lr)
        engine.refresh_weights(self.params)          # builds and uploads the refresh table
        torch.cuda.synchronize(dev)

    def set_lr(self, lr):
        """the learning rate of every group, as float32(lr) of the host double (adjust_learning_rate multiplies the
        Python value, so this follows torch's rounding); a host -> device copy: call it outside any capture.  A
        captured step reads the new value on its next replay."""
        self.lr_value = float(lr)
        self.lr.copy_(torch.tensor([self.lr_value], dtype=torch.float32))

    def step(self, im_left, im_right, gt_left, gt_right, gt_merge, gt_dim_orien, gt_kpts, keys, words, rpn_keys,
             dropout_words=None):
        """One training step on one stereo batch (arguments as loss_gradients).  Returns device tensors (losses [6],
        total [1], [norm, clip factor] [2], skipped [1]); losses are those of the weights before the update.
        No host synchronisation and no torch operator on the compute path (at world 1): capturable with
        engine.GraphRunner."""
        eng = self.engine
        d_u = self.grads.grads[-1]
        losses, _g, _du = loss_gradients(eng, im_left, im_right, gt_left, gt_right, gt_merge, gt_dim_orien, gt_kpts,
                                         keys, words, rpn_keys, dropout_words=dropout_words, uncert=self.uncert,
                                         fixed_blocks=self.fixed_blocks, grads=self.grad_views,
                                         grad_scale=self.grad_scale, total=self.total, d_uncert=d_u)
        if self.world > 1 and self.dist is not None:
            self.grads.all_reduce()
            # every rank skips the step when any rank overflowed
            self.dist.all_reduce(eng.found_inf, op=self.dist.ReduceOp.MAX)
        clip_gradient(self.grads.grads[:-1], self.clip_norm, out=self.norm)
        self._sgd(self.lr, self.momentum, eng.found_inf, self.skipped)
        eng.refresh_weights(self.params)
        if self.dynamic is not None:
            d = self.dynamic
            loss_scale_update(eng.found_inf, self.loss_scale, self.growth_tracker, d.growth_factor, d.backoff_factor,
                              d.growth_interval)
        return losses, self.total, self.norm, self.skipped

    def step_from_frames(self, inp):
        """One training step from the buffers of a StepInputs (its B stereo pairs): sb_prep_stereo_pairs, the random
        words of this step (sb_random_words keyed by `seed` and the device step counter; tensor i of
        inp.word_tensors takes stream id 5 rank + i, so every rank draws its own words and rank 0 those of a
        one-process run), sb_train_gt, step, then sb_step_advance -- so the next call, or the next replay of a captured
        call, draws new words; a skipped (overflowed) step advances too.  Returns what step returns.  Outside a stream
        capture the current stream first waits for inp.load's copies and afterwards marks the buffers as consumed; a
        captured call holds the kernels only, and whoever replays it calls inp.ready() before and inp.release()
        after."""
        capturing = torch.cuda.is_current_stream_capturing()
        if not capturing:
            inp.ready()
        from .ops import prep_stereo_pair
        prep_stereo_pair(inp.left_u8, inp.right_u8, inp.scale, inp.flip, rgb_input=inp.rgb_input,
                         out=(inp.im_left, inp.im_right))
        n_ids = len(inp.word_tensors)
        for stream_id, t in enumerate(inp.word_tensors):
            fill_random_words(t, self.seed, self.step_count, n_ids * self.rank + stream_id)
        train_gt(inp.rows, inp.n_rows, inp.shuffle_words, inp.scale, inp.im_left.shape[3], out=inp.gt)
        out = self.step(inp.im_left, inp.im_right, *inp.gt[:5], inp.keys, inp.words, inp.rpn_keys,
                        dropout_words=inp.dropout_words)
        step_advance(self.step_count)
        if not capturing:
            inp.release()
        return out

    def state_dict(self):
        """host state_dict with the reference's keys: the trained masters, plus every other tensor (frozen weights,
        BN parameters and buffers) of the state_dict the trainer was built from.  Copies to the host: a sync point."""
        out = dict(self._sd)
        for n, v in self.params.items():
            out[n] = v.detach().cpu().clone()
        return out

    def checkpoint(self):
        """what save_checkpoint stores (trainval_net.py:249-254), on the host: {"model": state_dict(), "uncert": [6],
        "momentum": {name: momentum buffer}} (the buffers of torch.optim.SGD's state, by parameter name, "uncert"
        included), plus what a resumed run needs to continue as if it had not stopped: "epoch" (the next epoch of fit,
        as the reference stores epoch + 1), "step" (the device step counter that keys the random words), "lr" and
        "sampler_state" (fit's host generator).  With a DynamicLossScale also "loss_scale" (fp32 [1]) and
        "growth_tracker" (int32 [1]).  A sync point."""
        mom = {n: v.detach().cpu().clone() for n, v in zip(self.names + ["uncert"], self.moms.grads)}
        out = {"model": self.state_dict(), "uncert": self.uncert.detach().cpu().clone(), "momentum": mom,
               "epoch": int(self.epoch), "step": int(self.step_count.item()), "lr": self.lr_value,
               "sampler_state": self.sampler_state}
        if self.dynamic is not None:
            out["loss_scale"] = self.loss_scale.detach().cpu().clone()
            out["growth_tracker"] = self.growth_tracker.detach().cpu().clone()
        return out

    def load_checkpoint(self, ckpt):
        """Resume from checkpoint(): the masters, uncert, every momentum buffer (which the reference's resume,
        trainval_net.py:170-179, leaves at zero), the step counter, the epoch and the lr, then the engine's packed
        weights refreshed from the masters; a dynamic trainer also restores "loss_scale" and "growth_tracker" when the
        checkpoint holds them.  The frozen tensors are the engine's own: build the engine and the trainer from the
        state_dict of the run that is resumed.  Host -> device copies: call it outside any capture."""
        with torch.no_grad():
            for n, v in self.params.items():
                v.copy_(ckpt["model"][n].to(torch.float32))
            self.uncert.copy_(ckpt["uncert"])
            for n, v in zip(self.names + ["uncert"], self.moms.grads):
                v.copy_(ckpt["momentum"][n])
            self.step_count.copy_(torch.tensor([int(ckpt["step"])], dtype=torch.int64))
            if self.dynamic is not None and "loss_scale" in ckpt:
                self.loss_scale.copy_(ckpt["loss_scale"].reshape(1).to(torch.float32))
                self.growth_tracker.copy_(ckpt["growth_tracker"].reshape(1).to(torch.int32))
        self.epoch, self.sampler_state = int(ckpt["epoch"]), ckpt.get("sampler_state")
        self.set_lr(ckpt["lr"])
        self.engine.refresh_weights(self.params)
        torch.cuda.synchronize(self.engine.device)


class StepInputs(object):
    """The static buffers of one in-flight step_from_frames over `batch` stereo pairs of one frame shape: the uint8
    frame pairs [B,H,W,3], the roidb rows [B,N,.] at capacity N = `max_rows` with their counts n_rows [B], the flip
    flags [B], the blobs [B,3,Ho,Wo], the ground truth of the step ([B,30,.], num_boxes [B]) and its random words in
    the shapes loss_gradients documents (keys [B,R+K], words [B,S], rpn_keys [B,A], the shuffle words [B,N], dropout
    words [2,B*S,2048]).  load() fills the inputs from pinned host memory on a copy stream of its own, so with two
    StepInputs the copy of batch k + 1 overlaps step k.  frame_hw: (H, W) of the camera frames; scale: im_scale of the
    blob (target size / shorter side, blob.py:51); rgb_input: the frames are RGB, as image decoders give them
    (minibatch.py:111-114), not BGR."""

    def __init__(self, frame_hw, scale, device, batch=1, max_rows=64, rgb_input=True, rois_per_image=None,
                 post_nms_top_n=None):
        from .ops import CFG as OPS_CFG
        L = _l.load()
        H, W, B = int(frame_hw[0]), int(frame_hw[1]), int(batch)
        if B < 1:
            raise ValueError("a StepInputs holds at least one pair, not %d" % B)
        self.frame_hw, self.scale, self.rgb_input, self.device, N = (H, W), float(scale), bool(rgb_input), device, int(max_rows)
        self.batch = B
        ho, wo = ctypes.c_int(), ctypes.c_int()
        check(L.sb_prep_image_size(H, W, self.scale, ctypes.byref(ho), ctypes.byref(wo)), "sb_prep_image_size")
        Ho, Wo = ho.value, wo.value
        S = int(rois_per_image or CFG["BATCH_SIZE"])
        R = int(post_nms_top_n or OPS_CFG["TRAIN"]["RPN_POST_NMS_TOP_N"])
        # anchors over the pyramid as the trunk makes it: the 7x7 stride-2 stem and the ceil-mode 3x3 stride-2 max
        # pool give P2, every further level halves with (n - 1) // 2 + 1 (ceil(n / stride) is one more for widths
        # such as 1985, the blob of a 370x1224 KITTI frame)
        h, w, A = ((Ho - 1) // 2 - 1) // 2 + 1, ((Wo - 1) // 2 - 1) // 2 + 1, 0
        for _ in OPS_CFG["FPN_FEAT_STRIDES"]:
            A += h * w
            h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        A *= len(OPS_CFG["ANCHOR_RATIOS"])
        host = {"left_u8": torch.empty(B, H, W, 3, dtype=torch.uint8),
                "right_u8": torch.empty(B, H, W, 3, dtype=torch.uint8),
                "gt_classes": torch.zeros(B, N, dtype=torch.int32), "n_rows": torch.zeros(B, dtype=torch.int32),
                "flip": torch.zeros(B, dtype=torch.int32)}
        for k, w in GT_ROW_FIELDS:
            host[k] = torch.zeros(B, N, w, dtype=torch.float32)
        self._host = {k: v.pin_memory() for k, v in host.items()}
        self._dev = {k: torch.zeros_like(v, device=device) for k, v in host.items()}
        self.left_u8, self.right_u8 = self._dev["left_u8"], self._dev["right_u8"]
        self.n_rows, self.flip = self._dev["n_rows"], self._dev["flip"]
        self.rows = {k: self._dev[k] for k in ("gt_classes",) + tuple(k for k, _ in GT_ROW_FIELDS)}
        f = lambda *s: torch.zeros(*s, dtype=torch.float32, device=device)
        i32 = lambda *s: torch.zeros(*s, dtype=torch.int32, device=device)
        self.im_left, self.im_right = f(B, 3, Ho, Wo), f(B, 3, Ho, Wo)
        self.gt = (f(B, 30, 5), f(B, 30, 5), f(B, 30, 5), f(B, 30, 5), f(B, 30, 6), i32(B))
        self.shuffle_words, self.keys, self.words = i32(B, N), i32(B, R + MAX_NUM_GT_BOXES), i32(B, S)
        self.rpn_keys, self.dropout_words = i32(B, A), i32(2, B * S, 2048)
        # the index of a tensor here is its sb_random_words stream id (offset by 5 rank, Trainer.step_from_frames)
        self.word_tensors = (self.shuffle_words, self.keys, self.words, self.rpn_keys, self.dropout_words)
        self._copy_stream = torch.cuda.Stream(device)
        self._copied, self._consumed = torch.cuda.Event(), torch.cuda.Event()

    def load(self, entries, frames, right=None):
        """fill the inputs from B roidb entries and their B frame pairs [(left, right)] of uint8 [H,W,3] (numpy
        arrays or tensors); load(entry, left, right) is the one-pair form.  A host copy into pinned memory, then
        non_blocking copies on the copy stream, which first waits until the step that last read these buffers has
        finished.  The host waits only for the previous load's copies out of the pinned buffers."""
        if right is not None:
            entries, frames = [entries], [(frames, right)]
        B = self.batch
        if len(entries) != B or len(frames) != B:
            raise ValueError("%d entries and %d frame pairs for a StepInputs of %d pairs" % (len(entries), len(frames), B))
        self._copied.synchronize()
        h = self._host
        N = h["gt_classes"].shape[1]
        for b, (entry, (left, right)) in enumerate(zip(entries, frames)):
            n = int(len(entry["gt_classes"]))
            if n > N:
                raise ValueError("%d annotation rows exceed the capacity %d of this StepInputs" % (n, N))
            h["left_u8"][b].copy_(torch.as_tensor(left))
            h["right_u8"][b].copy_(torch.as_tensor(right))
            h["gt_classes"][b, :n] = torch.as_tensor(np.asarray(entry["gt_classes"], np.int32))
            for k, _ in GT_ROW_FIELDS:
                h[k][b, :n] = torch.as_tensor(np.asarray(entry[k], np.float32))
            h["n_rows"][b], h["flip"][b] = n, int(bool(entry.get("flipped", False)))
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


def epoch_order(n, generator):
    """the reference sampler's order of one epoch at one pair per batch (trainval_net.py:81-101): a permutation of
    the n entries from the host generator, no leftover"""
    return torch.randperm(n, generator=generator).tolist()


def epoch_batches(roidb, batch_size, generator, rank=0, world=1):
    """The batches of one epoch that rank `rank` of `world` trains on, as lists of roidb indices.

    batch_size 1: the batches of epoch_order(len(roidb), generator).  batch_size B > 1: every batch holds entries of
    one frame shape, the documented difference from the reference (its aspect-ratio grouping, roidb.py:49-73, gives
    every KITTI entry ratio 2, and its loader cannot stack blobs of different shapes): the entries are grouped by
    (entry["height"], entry["width"]); within each group, in order of first appearance, a permutation is drawn and
    cut into consecutive batches of B, a short tail dropped (as the reference drops int(train_size / bs)'s leftover);
    then a permutation of all the batches is drawn.  Every rank draws the same epoch from the same generator state;
    step k of rank r takes batch k world + r, so an epoch has floor(n_batches / world) steps."""
    B, world = int(batch_size), int(world)
    if B < 1 or world < 1 or not 0 <= rank < world:
        raise ValueError("batch_size %d, rank %d of world %d" % (B, rank, world))
    if B == 1:
        batches = [[i] for i in epoch_order(len(roidb), generator)]
    else:
        groups = {}
        for i, e in enumerate(roidb):
            if "height" not in e or "width" not in e:
                raise ValueError("roidb entry %d has no height / width: batches of %d pairs are grouped by frame "
                                 "shape" % (i, B))
            groups.setdefault((int(e["height"]), int(e["width"])), []).append(i)
        cut = []
        for members in groups.values():
            perm = torch.randperm(len(members), generator=generator).tolist()
            cut += [[members[j] for j in perm[k:k + B]] for k in range(0, len(perm) - B + 1, B)]
        batches = [cut[j] for j in torch.randperm(len(cut), generator=generator).tolist()]
    return [batches[k * world + rank] for k in range(len(batches) // world)]


def lr_schedule(lr, start_epoch, epochs, lr_decay_step=5, lr_decay_gamma=0.1):
    """[(epoch, lr)] of trainval_net.py:184-191: the lr is multiplied by gamma at the start of every epoch with
    epoch % (lr_decay_step + 1) == 0"""
    out = []
    for epoch in range(start_epoch, epochs + 1):
        if epoch % (lr_decay_step + 1) == 0:
            lr *= lr_decay_gamma
        out.append((epoch, lr))
    return out


VAL_KEYS = ("entries", "frames", "calib", "result_dir")
VAL_OPTIONAL = ("labels", "name", "empty_files", "inflight")


def fit(trainer, roidb, frames, epochs, start_epoch=1, lr_decay_step=5, lr_decay_gamma=0.1, save_dir=None, log=print,
        generator=None, target_size=600, max_rows=64, rgb_input=True, batch_size=1, val=None):
    """The training loop of trainval_net.py:183-258 at `batch_size` stereo pairs per step and rank (the reference's
    --bs, trainval_net.py:54-56) over Trainer.step_from_frames, two buffer sets per (frame shape) so that the copy of
    the next batch overlaps the running step.  At trainer.world == 1 every (frame shape, buffer set) replays a CUDA
    graph of its step; at world > 1 the steps run eagerly (the gradient all-reduce is a collective outside any graph).

    roidb: the reference's list of dicts (boxes_left, boxes_right, boxes_merge, dim_orien, kpts, gt_classes,
    flipped; see append_flipped; with batch_size > 1 also the frame's height and width, as kitti_data.train_roidb sets
    them); frames(entry) -> (left, right) uint8 [H,W,3] arrays of the unflipped pair, decoded by the caller (RGB
    unless rgb_input is False).  The batches of an epoch are epoch_batches(roidb, batch_size, generator,
    trainer.rank, trainer.world), drawn from `generator` (default: a torch.Generator seeded with trainer.seed, or
    continued from a loaded checkpoint), the same on every rank; the lr follows lr_schedule through trainer.set_lr
    (not scaled with the batch, as in the reference).  Per step rank 0 logs two lines in the reference's format
    (trainval_net.py:240-244) with the losses averaged over the ranks (parallel.average_losses) and [iter k/n] counting
    steps; the numbers are copied to pinned memory behind an event and read one step late, so the steady state has no
    device-wide synchronise.  A trainer with a DynamicLossScale adds a third line per step, "loss scale: %g, skipped
    steps: %d", the scale after the step and the trainer's skipped count, read through the same copy.  With save_dir, rank 0 saves trainer.checkpoint() after every epoch as
    stereo_rcnn_{epoch}_{last step}.pth (trainval_net.py:248-254).  To resume, on every rank:
    trainer.load_checkpoint(ckpt), then fit(..., start_epoch=ckpt["epoch"]).

    val: a validation split scored after every epoch -- a dict of evaluate's entries, frames, calib and result_dir,
    optionally labels, name, empty_files and inflight, each as pipeline.evaluate takes it.  At the first validation
    one StereoPipeline(trainer.state_dict(), throughput=True, precision of the trainer's engine) is built (one copy
    of the weights to the device); after every later epoch pipe.eng.refresh_weights(trainer.params) writes the
    trained masters into it in one launch.  After the epoch's checkpoint, evaluate runs on it at this target_size and
    rgb_input, sharded over the trainer's ranks, into result_dir/epoch_<n>, replaying the graphs the first
    validation captured.  Rank 0 logs its AP line; trainer.val_summaries[epoch] holds the summary without "curves"
    on every rank.  Validation reads the masters and writes nothing the training reads: the steps, the random
    words, the checkpoints and the return value are those of the same run without val.
    -> [total loss of every step, averaged over the ranks]"""
    import os
    from .engine import GraphRunner
    from .parallel import average_losses
    dev = trainer.engine.device
    world, rank, lead = trainer.world, trainer.rank, trainer.rank == 0
    gen = generator
    if gen is None:
        gen = torch.Generator()
        if trainer.sampler_state is not None:
            gen.set_state(trainer.sampler_state)
        else:
            gen.manual_seed(trainer.seed)
    if val is not None:
        missing = [k for k in VAL_KEYS if k not in val]
        unknown = [k for k in val if k not in VAL_KEYS + VAL_OPTIONAL]
        if missing or unknown:
            raise ValueError("val: missing %s, unknown %s; it takes %s and optionally %s"
                             % (missing, unknown, ", ".join(VAL_KEYS), ", ".join(VAL_OPTIONAL)))
    val_pipe, val_slots = None, {}
    slots, runners, turn = {}, {}, {}
    stats_host = [torch.zeros(7, dtype=torch.float32).pin_memory() for _ in range(2)]
    dynamic = trainer.dynamic is not None
    scale_host = [torch.zeros(1, dtype=torch.float32).pin_memory() for _ in range(2)] if dynamic else None
    skipped_host = [torch.zeros(1, dtype=torch.int32).pin_memory() for _ in range(2)] if dynamic else None
    stats_ev = [torch.cuda.Event() for _ in range(2)]
    totals = []

    def load(batch):
        entries = [roidb[i] for i in batch]
        pairs = [frames(e) for e in entries]
        hw = tuple(int(v) for v in pairs[0][0].shape[:2])
        if hw not in slots:
            slots[hw] = [StepInputs(hw, float(target_size) / float(min(hw)), dev, batch=batch_size,
                                    max_rows=max_rows, rgb_input=rgb_input) for _ in range(2)]
            turn[hw] = 0
        inp = slots[hw][turn[hw]]
        turn[hw] ^= 1
        inp.load(entries, pairs)
        return inp

    def report(k, epoch, it, n, lr):
        stats_ev[k].synchronize()
        v = stats_host[k].tolist()
        totals.append(v[6])
        if not lead:
            return
        log("[epoch %2d][iter %4d/%4d] loss: %.4f, lr: %.2e" % (epoch, it, n, v[6], lr))
        log("\t\t\trpn_cls: %.4f, rpn_box_left_right: %.4f, rcnn_cls: %.4f, rcnn_box_left_right %.4f,dim_orien %.4f, "
            "kpts %.4f" % tuple(v[:6]))
        if dynamic:
            log("\t\t\tloss scale: %g, skipped steps: %d" % (float(scale_host[k][0]), int(skipped_host[k][0])))

    for epoch, lr in lr_schedule(trainer.lr_value, start_epoch, epochs, lr_decay_step, lr_decay_gamma):
        if lr != trainer.lr_value:
            trainer.set_lr(lr)
        order = epoch_batches(roidb, batch_size, gen, rank, world)
        n = len(order)
        if n == 0:
            raise ValueError("an epoch of %d entries has no step of %d pairs on each of %d ranks"
                             % (len(roidb), batch_size, world))
        nxt = load(order[0])
        for it in range(n):
            inp = nxt
            if it + 1 < n:
                nxt = load(order[it + 1])
            with torch.no_grad():
                if world > 1:
                    out = trainer.step_from_frames(inp)
                    avg = average_losses(torch.cat((out[0], out[1])), world, trainer.dist)
                    out = (avg[:6], avg[6:])
                elif id(inp) not in runners:
                    # the first step on a buffer set runs eagerly (it creates the workspaces a capture needs); the
                    # capture that follows launches nothing
                    out = trainer.step_from_frames(inp)
                    runners[id(inp)] = GraphRunner(lambda inp=inp: trainer.step_from_frames(inp), [], warmup=0)
                else:
                    inp.ready()
                    out = runners[id(inp)]()
                    inp.release()
                k = it % 2
                stats_host[k][:6].copy_(out[0], non_blocking=True)
                stats_host[k][6:].copy_(out[1], non_blocking=True)
                if dynamic:
                    scale_host[k].copy_(trainer.loss_scale, non_blocking=True)
                    skipped_host[k].copy_(trainer.skipped, non_blocking=True)
                stats_ev[k].record()
            if it > 0:
                report(1 - k, epoch, it - 1, n, lr)
        report((n - 1) % 2, epoch, n - 1, n, lr)
        trainer.epoch, trainer.sampler_state = epoch + 1, gen.get_state()
        if save_dir is not None and lead:
            name = os.path.join(save_dir, "stereo_rcnn_%d_%d.pth" % (epoch, n - 1))
            torch.save(trainer.checkpoint(), name)
            log("save model: %s" % name)
        if val is not None:
            from . import pipeline
            if val_pipe is None:
                val_pipe = pipeline.StereoPipeline(trainer.state_dict(), dev, throughput=True,
                                                   precision=trainer.engine.precision)
            else:
                val_pipe.eng.refresh_weights(trainer.params)
            opts = {k: val[k] for k in VAL_OPTIONAL if k in val}
            summary = pipeline.evaluate(val_pipe, val["entries"], val["frames"], val["calib"],
                                        os.path.join(val["result_dir"], "epoch_%d" % epoch), target_size=target_size,
                                        rgb_input=rgb_input, log=log, world=world,
                                        dist=trainer.dist, slots=val_slots, **opts)
            if "ap" in summary:
                summary["ap"] = {k: v for k, v in summary["ap"].items() if k != "curves"}
            trainer.val_summaries[epoch] = summary
    return totals
