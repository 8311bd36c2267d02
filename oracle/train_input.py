"""numpy restatements of the training side of the input pipeline (SURVEY 8f-3), the checker of csrc/train_input.cu:

  * pair_blobs        -- _get_image_blob (minibatch.py:89-131): the flip of a frame pair, then oracle.ops.prep_image
  * append_flipped    -- imdb.append_flipped_images (imdb.py:117-176)
  * train_gt          -- get_minibatch's ground truth (minibatch.py:43-85) and roibatchLoader.__getitem__'s shuffle and
                         padding (roibatchLoader.py:72-107), the shuffle given by explicit words
  * philox4x32_10 / random_words -- the generator of sb_random_words

Every float32 operation of the reference is one float32 operation here: the roidb arrays are float32 (kitti.py:228-233)
and numpy keeps float32 when such an array meets a Python scalar, so `boxes * im_scale`, `width - x - 1` and
`math.pi - theta` are float32 operations on the float32 value of the scalar.  math.sin / math.cos read a float32 as a
double and the store rounds the result.
"""
import math

import numpy as np

from . import ops

MAX_NUM_GT_BOXES = 30                                    # config.py:283
f32 = np.float32


def pair_blobs(left_bgr_u8, right_bgr_u8, scale, flipped):
    """minibatch.py:116-123 -> (blob_left, blob_right) [3,Ho,Wo] fp32"""
    if flipped:
        left_bgr_u8, right_bgr_u8 = right_bgr_u8[:, ::-1, :].copy(), left_bgr_u8[:, ::-1, :].copy()
    return ops.prep_image(left_bgr_u8, scale), ops.prep_image(right_bgr_u8, scale)


def _mirror_boxes(boxes, width):
    out = boxes.astype(f32).copy()
    w = f32(width)
    out[:, 0] = (w - boxes[:, 2]).astype(f32) - f32(1)
    out[:, 2] = (w - boxes[:, 0]).astype(f32) - f32(1)
    assert (out[:, 2] >= out[:, 0]).all()
    return out


def _mirror_kpts(kpts, width):
    w = f32(width)
    return ((w - kpts[:, [3, 2, 1, 0, 5, 4]].astype(f32)).astype(f32) - f32(1)).astype(f32)


def flip_entry(e, width):
    """one iteration of imdb.py:120-175.  The flipped entry also carries `kpts_right` (the mirror of the entry's
    `kpts`), which the reference drops: with it the flip is an involution on every field"""
    th = e["dim_orien"].astype(f32).copy()
    pi, two_pi = f32(math.pi), f32(2.0 * math.pi)
    t = th[:, 3]
    t = np.where(t > pi, (t - two_pi).astype(f32), t)
    t = np.where(t < -pi, (t + two_pi).astype(f32), t)
    th[:, 3] = np.where(t >= 0, (pi - t).astype(f32), (-pi - t).astype(f32))
    out = dict(e)
    out.update(boxes_left=_mirror_boxes(e["boxes_right"], width), boxes_right=_mirror_boxes(e["boxes_left"], width),
               boxes_merge=_mirror_boxes(e["boxes_merge"], width), dim_orien=th,
               kpts=_mirror_kpts(e["kpts_right"], width), kpts_right=_mirror_kpts(e["kpts"], width),
               flipped=not e.get("flipped", False))
    return out


def append_flipped(roidb, widths):
    """imdb.append_flipped_images: roidb + the flip of every entry"""
    return list(roidb) + [flip_entry(e, w) for e, w in zip(roidb, widths)]


def word_order(words, valid):
    """indices of the valid rows ordered by (word, row index) ascending"""
    idx = np.nonzero(valid)[0]
    w = np.asarray(words).view(np.uint32)[idx].astype(np.int64)
    return idx[np.lexsort((idx, w))]


def train_gt(entry, im_scale, im_width, words, n=None):
    """entry: a roidb dict (float32 arrays; the first `n` rows are in use), words: one uint32 per row ->
    (gt_left, gt_right, gt_merge [30,5], gt_dim_orien [30,5], gt_kpts [30,6], num_boxes)"""
    cls = np.asarray(entry["gt_classes"])
    N = cls.shape[0]
    n = N if n is None else min(max(int(n), 0), N)
    valid = (cls != 0) & (np.arange(N) < n)
    order = word_order(words, valid)[:MAX_NUM_GT_BOXES]
    s = f32(im_scale)
    k = len(order)
    outs = []
    for name in ("boxes_left", "boxes_right", "boxes_merge"):
        g = np.zeros((MAX_NUM_GT_BOXES, 5), f32)
        g[:k, 0:4] = (entry[name].astype(f32)[order] * s).astype(f32)
        g[:k, 0] = np.minimum(g[:k, 0], f32(im_width))
        g[:k, 4] = cls[order]
        outs.append(g)
    d = np.zeros((MAX_NUM_GT_BOXES, 5), f32)
    do = entry["dim_orien"].astype(f32)[order]
    d[:k, 0:3] = do[:, 0:3]
    d[:k, 3] = [math.sin(float(t)) for t in do[:, 3]]
    d[:k, 4] = [math.cos(float(t)) for t in do[:, 3]]
    kp = np.zeros((MAX_NUM_GT_BOXES, 6), f32)
    v = (entry["kpts"].astype(f32)[order] * s).astype(f32)
    v[(v < 0) | (v > f32(im_width - 1))] = -1
    kp[:k] = v
    return outs[0], outs[1], outs[2], d, kp, k


# ---------------------------------------------------------------------------------------------------- Philox4x32-10
_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85


def philox4x32_10(counter, key):
    """counter [..., 4], key [..., 2] uint32 -> [..., 4] uint32 (Salmon et al., SC'11; ten rounds)"""
    c = [np.asarray(counter)[..., i].astype(np.uint64) for i in range(4)]
    k = [np.asarray(key)[..., i].astype(np.uint64) for i in range(2)]
    m32 = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(_M0) * c[0], np.uint64(_M1) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k[0], p1 & m32, (p0 >> np.uint64(32)) ^ c[3] ^ k[1], p0 & m32]
        k = [(k[0] + np.uint64(_W0)) & m32, (k[1] + np.uint64(_W1)) & m32]
    return np.stack(c, -1).astype(np.uint32)


def random_words(seed, step, stream_id, n):
    """the n words of sb_random_words as int32 bit patterns: key (seed lo, seed hi), counter
    (i / 4, stream_id, step lo, step hi)"""
    g = (n + 3) // 4
    ctr = np.empty((g, 4), np.uint32)
    ctr[:, 0] = np.arange(g, dtype=np.uint64).astype(np.uint32)
    ctr[:, 1] = stream_id
    ctr[:, 2], ctr[:, 3] = step & 0xFFFFFFFF, (step >> 32) & 0xFFFFFFFF
    key = np.array([seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF], np.uint32)
    return philox4x32_10(ctr, np.broadcast_to(key, (g, 2))).reshape(-1)[:n].view(np.int32)
