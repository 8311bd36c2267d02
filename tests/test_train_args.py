"""CPU: the six train-time entry points (sb_anchor_targets, sb_proposal_targets, sb_rpn_loss, sb_rcnn_loss,
sb_multitask_loss, sb_clip_gradient) refuse every invalid argument with SB_EINVAL before any CUDA call (so without a
GPU, and without a launch), and the cases of test_gpu_train_edges reach every branch of the kernels they test."""
import collections
import ctypes

import numpy as np
import pytest

from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import train as TR
from test_gpu_train_edges import CASES, at_cells, clip_inputs, pt_cells, rcnn_inputs, rpn_trips

SB_EINVAL = -22
FAKE = 1 << 20                                            # never dereferenced: every refusal precedes the first call


@pytest.fixture(scope="module")
def lib():
    from stereo_rcnn_b200 import build
    build.build()
    return L.load()


def test_anchor_targets_rejections(lib):
    B, A = 2, 1000
    nb = lib.sb_anchor_targets_workspace(B, A)
    assert nb > B * A * 8 and lib.sb_anchor_targets_workspace(0, A) == 0

    def call(anchors=FAKE, A=A, gl=FAKE, gr=FAKE, gm=FAKE, B=B, K=30, keys=FAKE, batch=512, num_fg=256, ws=FAKE,
             nbytes=nb, labels=FAKE, tl=FAKE, tr=FAKE, iw=FAKE, ow=FAKE):
        return lib.sb_anchor_targets(anchors, A, gl, gr, gm, B, K, 160, 256, keys, 0.3, 0.7, batch, num_fg, ws, nbytes,
                                     labels, tl, tr, iw, ow, None)
    n0 = lib.sb_launch_count()
    bad = {"null anchors": call(anchors=None), "null gt_left": call(gl=None), "null gt_right": call(gr=None),
           "null gt_merge": call(gm=None), "null keys": call(keys=None), "null workspace": call(ws=None),
           "null labels": call(labels=None), "null targets_left": call(tl=None), "null targets_right": call(tr=None),
           "null inside_w": call(iw=None), "null outside_w": call(ow=None), "A = 0": call(A=0), "B = 0": call(B=0),
           "K = 0": call(K=0), "K = 65": call(K=65), "batch 0": call(batch=0), "num_fg < 0": call(num_fg=-1),
           "short workspace": call(nbytes=nb - 1), "misaligned workspace": call(ws=FAKE + 4),
           "misaligned anchors": call(anchors=FAKE + 4), "misaligned targets_left": call(tl=FAKE + 8),
           "misaligned targets_right": call(tr=FAKE + 4)}
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}


def test_proposal_targets_rejections(lib):
    def call(rl=FAKE, B=2, R=2000, K=30, keys=FAKE, words=FAKE, tl=FAKE, iw=FAKE, ow=FAKE, status=FAKE, cfg=True,
             **over):
        c = TR._pt_cfg(TR.CFG)
        for k, v in over.items():
            setattr(c, k, v)
        outs = [FAKE] * 12
        outs[3], outs[8], outs[9], outs[11] = tl, iw, ow, status
        return lib.sb_proposal_targets(rl, FAKE, B, R, FAKE, FAKE, FAKE, FAKE, K, keys, words,
                                       ctypes.byref(c) if cfg else None, *outs, None)
    n0 = lib.sb_launch_count()
    bad = {"null rois": call(rl=None), "null keys": call(keys=None), "null words": call(words=None),
           "null cfg": call(cfg=False), "null status": call(status=None), "null targets": call(tl=None),
           "B = 0": call(B=0), "R < 0": call(R=-1), "K = 0": call(K=0), "K = 65": call(K=65),
           "R + K = 4097": call(R=4067, K=30), "rois_per_image 0": call(rois_per_image=0),
           "rois_per_image 1025": call(rois_per_image=1025, fg_rois_per_image=256),
           "fg > rois_per_image": call(rois_per_image=100, fg_rois_per_image=101),
           "fg < 0": call(fg_rois_per_image=-1), "kpts_grid 0": call(kpts_grid=0),
           "misaligned bbox targets": call(tl=FAKE + 4), "misaligned inside_w": call(iw=FAKE + 8),
           "misaligned outside_w": call(ow=FAKE + 12)}
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}


def test_rpn_loss_rejections(lib):
    nb = lib.sb_loss_workspace_bytes()

    def call(score=FAKE, lab=FAKE, tl=FAKE, tr=FAKE, B=2, A=1000, ws=FAKE, nbytes=nb, losses=FAKE, d_cls=FAKE,
             d_box=FAKE):
        return lib.sb_rpn_loss(score, FAKE, lab, tl, tr, FAKE, FAKE, B, A, None, ws, nbytes, losses, d_cls, d_box, None)
    n0 = lib.sb_launch_count()
    bad = {"null score": call(score=None), "null labels": call(lab=None), "null targets": call(tl=None),
           "null losses": call(losses=None), "null workspace": call(ws=None), "B = 0": call(B=0), "A = 0": call(A=0),
           "short workspace": call(nbytes=nb - 1), "misaligned workspace": call(ws=FAKE + 8),
           "misaligned targets_left": call(tl=FAKE + 4), "misaligned targets_right": call(tr=FAKE + 4),
           "d_cls without d_box": call(d_box=None), "d_box without d_cls": call(d_cls=None)}
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}


def test_rcnn_loss_rejections(lib):
    def call(ins=None, R=1024, C=2, G=28, losses=FAKE, grads=(FAKE,) * 6, tl=FAKE, iw=FAKE, ow=FAKE):
        ins = list(ins or [FAKE] * 14)
        ins[7], ins[12], ins[13] = tl, iw, ow
        return lib.sb_rcnn_loss(*ins, R, C, G, None, losses, *grads, None)
    n0 = lib.sb_launch_count()
    bad = {"null input %d" % i: call(ins=[None if j == i else FAKE for j in range(14)]) for i in (0, 1, 5, 6, 10, 11)}
    bad.update({"null losses": call(losses=None), "R = 0": call(R=0), "one class": call(C=1),
                "kpts_grid 0": call(G=0), "misaligned bbox targets": call(tl=FAKE + 4),
                "misaligned inside_w": call(iw=FAKE + 4), "misaligned outside_w": call(ow=FAKE + 8)})
    for k in range(1, 6):                                 # a partial gradient group
        bad["%d of 6 gradients" % k] = call(grads=[FAKE] * k + [None] * (6 - k))
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}


def test_multitask_loss_rejections(lib):
    n0 = lib.sb_launch_count()
    bad = {"n = 0": lib.sb_multitask_loss(FAKE, FAKE, 0, FAKE, FAKE, None),
           "n = 65": lib.sb_multitask_loss(FAKE, FAKE, 65, FAKE, FAKE, None),
           "null losses": lib.sb_multitask_loss(None, FAKE, 6, FAKE, FAKE, None),
           "null uncert": lib.sb_multitask_loss(FAKE, None, 6, FAKE, FAKE, None),
           "null total": lib.sb_multitask_loss(FAKE, FAKE, 6, None, FAKE, None)}
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), bad


def test_clip_gradient_rejections(lib):
    def call(n=97, counts=None, ptrs=None, clip=10.0, ws=FAKE, nbytes=None, out=FAKE, null_arrays=False):
        p = (ctypes.c_void_p * max(n, 1))(*(ptrs or [FAKE + 64 * i for i in range(max(n, 1))]))
        c = (ctypes.c_size_t * max(n, 1))(*(counts or [5] * max(n, 1)))
        nb = lib.sb_clip_gradient_workspace(max(n, 1)) if nbytes is None else nbytes
        return lib.sb_clip_gradient(None if null_arrays else p, c, n, clip, ws, nb, out, None)
    nb = lib.sb_clip_gradient_workspace(97)
    assert nb >= 97 * 32 * 8 and lib.sb_clip_gradient_workspace(0) == 0
    n0 = lib.sb_launch_count()
    bad = {"zero-count tensor": call(counts=[5] * 60 + [0] + [5] * 36),
           "null tensor": call(ptrs=[FAKE] * 96 + [None]), "null pointer array": call(null_arrays=True),
           "n = 0": call(n=0), "clip 0": call(clip=0.0), "clip < 0": call(clip=-1.0), "clip NaN": call(clip=float("nan")),
           "short workspace": call(nbytes=nb - 1), "misaligned workspace": call(ws=FAKE + 4),
           "null workspace": call(ws=None), "null norm": call(out=None)}
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}


def test_case_census():
    """every branch cell of the target kernels and the losses is reached by at least one case of
    test_gpu_train_edges, evaluated with the oracle on the CPU"""
    cnt = collections.Counter()
    for c in CASES:
        if c.kind == "at":
            cnt.update(at_cells(c))
        elif c.kind == "pt":
            cnt.update(pt_cells(c))
        elif c.kind == "rpn":
            cnt["RPN loss, %s grid-stride trip" % ("one" if rpn_trips(c) == 1 else "several")] += 1
        elif c.kind == "rcnn":
            _preds, tgt, _u, _g = rcnn_inputs(c)
            for h in range(3):
                cnt["rcnn sum(w) %s 1" % ("<" if tgt["kpts_weight"][:, h].sum() < 1 else ">=")] += 1
            cnt["rcnn R %% 1024 %s 0" % ("=" if c.p["R"] % 1024 == 0 else "!=")] += 1
            cnt["rcnn C = %d" % c.p["C"]] += 1
        elif c.kind == "clip":
            grads, clip, norm = clip_inputs(c)
            cnt["clip %d chunk(s)" % -(-len(grads) // 48)] += 1
            cnt["clip tensor < 32 elements"] += sum(g.size < 32 for g in grads)
            cnt["clip norm %s clip" % ("=" if norm == clip else ">" if norm > clip else "<")] += 1
    print("\ntrain target / loss census:")
    for k, v in sorted(cnt.items()):
        print("  %-40s %d" % (k, v))
    need = ["K <= 32", "K > 32", "no sampling", "everything goes", "unique threshold", "threshold tie",
            "tie past the first 1024-block", "proposals fg+bg", "proposals fg only", "proposals bg only",
            "proposals none", "fg rank with equal keys", "fg list > 1024", "fg subsampled",
            "proposal IoU = 0", "proposal IoU = -1", "RPN loss, one grid-stride trip",
            "RPN loss, several grid-stride trip", "rcnn sum(w) < 1", "rcnn sum(w) >= 1", "rcnn R % 1024 = 0",
            "rcnn R % 1024 != 0", "rcnn C = 2", "rcnn C = 3", "rcnn C = 4", "clip 1 chunk(s)", "clip 2 chunk(s)",
            "clip 3 chunk(s)", "clip tensor < 32 elements", "clip norm = clip", "clip norm > clip",
            "clip norm < clip"]
    for tag, t in (("RPN", 0.7), ("RPN", 0.3), ("proposal", 0.5)):
        need += ["%s IoU = %g" % (tag, t), "%s IoU just above %g" % (tag, t), "%s IoU just below %g" % (tag, t)]
    assert not [k for k in need if not cnt[k]], [k for k in need if not cnt[k]]
    for t in (0.7, 0.3, 0.5):                             # pairs an FMA-contracted union would flip
        assert cnt["FMA flips at %g" % t] >= 10, (t, cnt["FMA flips at %g" % t])
    assert {c.p["K"] for c in CASES if c.kind == "at" and "K" in c.p} >= {1, 31, 32, 33, 63, 64}
    assert {c.p.get("batch", 512) for c in CASES if c.kind == "at"} >= {1, 7, 256, 512}
    assert {c.p["B"] for c in CASES if c.kind == "at" and "B" in c.p} >= {1, 2, 4}
    assert {c.p.get("batch", 512) for c in CASES if c.kind == "pt"} >= {1, 100, 512, 1024}
    assert {c.p.get("frac", 0.25) for c in CASES if c.kind == "pt"} >= {0.0, 0.25, 1.0}
    assert {c.p["B"] * c.p["A"] for c in CASES if c.kind == "rpn"} >= {1, 255, 131071, 131072, 131073, 2 * 298476}
    assert {c.p["R"] for c in CASES if c.kind == "rcnn"} >= {1, 31, 1023, 1024, 1025, 2048}
    assert {c.p["n"] for c in CASES if c.kind == "clip"} >= {47, 48, 49, 96, 97}
