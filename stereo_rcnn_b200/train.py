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


def multitask_loss(losses, uncert):
    """trainval_net.py:214-219: losses [n], uncert [n] -> total [1], d total / d uncert [n]"""
    L = _l.load()
    n = losses.numel()
    total = torch.empty(1, dtype=torch.float32, device=losses.device)
    d_u = torch.empty(n, dtype=torch.float32, device=losses.device)
    check(L.sb_multitask_loss(ptr(_f32c(losses)), ptr(_f32c(uncert)), n, ptr(total), ptr(d_u), stream_ptr()),
          "sb_multitask_loss")
    return total, d_u


def clip_gradient(grads, clip_norm):
    """net_utils.clip_gradient over a list of fp32 gradient tensors, in place -> norm [2] (total norm, factor)"""
    L = _l.load()
    n = len(grads)
    dev = grads[0].device
    assert all(g.dtype == torch.float32 and g.is_contiguous() for g in grads)
    ptrs = (ctypes.c_void_p * n)(*[g.data_ptr() for g in grads])
    counts = (ctypes.c_size_t * n)(*[g.numel() for g in grads])
    nbytes = L.sb_clip_gradient_workspace(n)
    ws = workspace(nbytes, dev, "clip")
    out = torch.empty(2, dtype=torch.float32, device=dev)
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
                   rpn_keys, dropout_words=None, uncert=None, fixed_blocks=1, grads=None, grad_scale=1.0):
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
    No optimizer step, no host synchronisation."""
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
        _total, d_u = multitask_loss(losses, uncert[0:6])
        return losses, grad, d_u
