"""GPU: backward of the R-CNN heads (sb_box_tail_scores, sb_kpts_logits, sb_dropout_words, sb_box_tail_backward,
sb_kpts_tail_backward, sb_permute3, engine.heads(save_for_backward=True), engine.heads_backward,
train.rcnn_head_gradients).

New kernels against float64 on the operands they read (relative L2 <= 2e-6 for the fp32 tails, <= 2e-5 for fp16
outputs); heads_backward layer by layer against float64 on the engine's own fp16 operands and saved masks; the R-CNN loss
differentiated end to end against fp32 autograd through a train-mode restatement of oracle.model.box_head / kpts_head
and oracle.train_targets.rcnn_losses.  Every test prints its measured worst error per tensor."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import model as OM
from oracle import train_targets as T
from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200 import lib as _l
from stereo_rcnn_b200 import ops as G
from stereo_rcnn_b200 import train as TR
from stereo_rcnn_b200.synth import synth_pair, synth_train_gt

pytestmark = pytest.mark.gpu

TAIL_TOL = 2e-6
KERNEL_TOL = 2e-5
MODEL_TOL = 5e-3
# the keypoint convs, the deconv and the two pooled gradients: the fp16 forward's rounding and ReLU-mask flips through the
# 14x14 chain (as for the trunk, DESIGN 6); test_rcnn_head_gradients_*_vs_oracle print the oracle's own shift under
# fp16-rounded weights, which is of the same size
KPTS_TOL = 1e-1
LOSS_TOL = 1e-3
SENT32 = 0x7FA5A5A5
SENT16 = 0x7E55
SB_EINVAL = -22
THR = int(np.ceil(E.DROPOUT_P * 2.0 ** 32))


def l2_err(a, b):
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    return float((a - b).norm() / max(float(b.norm()), 1e-300))


def h16(t):
    return t.half().double()


def guarded(shape, dtype, lead=64, tail=96):
    """a view of `shape` inside a NaN-sentinel buffer -> (view, check() that nothing outside it was written)"""
    n = int(np.prod(shape))
    if dtype == torch.float16:
        buf = torch.full((lead + n + tail,), SENT16, dtype=torch.int16, device="cuda")
        s = SENT16
    else:
        buf = torch.full((lead + n + tail,), SENT32, dtype=torch.int32, device="cuda")
        s = SENT32
    view = buf[lead:lead + n].view(dtype).view(*shape)

    def check():
        assert bool((buf[:lead] == s).all()) and bool((buf[lead + n:] == s).all()), "written outside the output"
    return view, check


@pytest.fixture(scope="module")
def sd():
    return OM.make_state_dict(3)


def _small_hw():
    import os
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "forward_small.npz"))
    return int(g["H"]), int(g["W"])


def _pairs(H, W, B, seed=5):
    ps = [synth_pair(H, W, seed + b, 12) for b in range(B)]
    return torch.from_numpy(np.stack([p[0] for p in ps] + [p[1] for p in ps], 0)).contiguous()


def _words(shape, seed):
    w = np.random.RandomState(seed).randint(0, 2 ** 32, shape, dtype=np.uint64).astype(np.uint32)
    return torch.from_numpy(w.view(np.int32)).cuda()


def _test_rois(eng, H, W, B, seed=5):
    with torch.no_grad():
        feats = eng.trunk_fpn(_pairs(H, W, B, seed).cuda())
        cp, bb, shapes = eng.rpn(feats, B)
        info = torch.tensor([[float(H), float(W), 1.0]] * B, device="cuda")
        rl, rr = G.proposal_layer(cp, bb, info, "TEST", shapes)
    return feats, rl.view(-1, 5), rr.view(-1, 5)


# ---------------------------------------------------------------- 1. the training-mode forward
@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("forks", [True, False])
def test_heads_forward_unchanged_with_save(sd, B, forks):
    H, W = _small_hw()
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16", forks=forks)
    feats, rl, rr = _test_rois(eng, H, W, B)
    with torch.no_grad():
        a = eng.heads(feats, B, rl, rr, float(H))
        b, saved = eng.heads(feats, B, rl, rr, float(H), save_for_backward=True)
    torch.cuda.synchronize()
    for k, v in a.items():
        assert torch.equal(v, b[k]), k
    R = rl.shape[0]
    assert saved.R == R and not saved.dropout
    assert torch.equal(saved.fc7, a["fc7"]) and torch.equal(saved.pooled_box, a["pooled_box"])
    assert saved.top0.shape == (R, 1, 1, 2048) and saved.top0.dtype == torch.float16
    assert len(saved.kpts) == 6 and saved.up.shape == (R, 28, 28, 256)
    ka = a["kpts_pred_all"]
    assert torch.equal(b["kpts_pred"], ka[:, :4].reshape(R, -1)) and torch.equal(b["left_border_pred"], ka[:, 4])
    assert torch.equal(b["right_border_pred"], ka[:, 5])
    errs = {"cls": (torch.softmax(b["cls_score"].double(), 1) - a["cls_prob"].double()).abs().max().item(),
            "kpts": (torch.softmax(b["kpts_pred"].double(), 1) - a["kpts_prob"].double()).abs().max().item()}
    print("B=%d forks=%s raw scores through a float64 softmax vs the probabilities: %s" % (B, forks, errs))
    assert errs["cls"] < 1e-6 and errs["kpts"] < 1e-6


def test_heads_save_requires_fp16(sd):
    eng = E.StereoRCNNEngine(sd, "cuda", precision="tf32")
    with pytest.raises(ValueError):
        eng.heads({}, 1, torch.zeros(1, 5), torch.zeros(1, 5), 10.0, save_for_backward=True)


# ---------------------------------------------------------------- 2. dropout
@pytest.mark.parametrize("dtype", [torch.float16, torch.float32])
def test_dropout_words_kernel(dtype):
    n = 3 * 2048 + 5
    x = torch.randn(n, generator=torch.Generator().manual_seed(1)).to(dtype).cuda()
    w = _words((n,), 2)
    # words on both sides of the threshold
    w[:4] = torch.tensor([THR - 1, THR, THR + 1, 0], dtype=torch.int64).to(torch.int32).cuda()
    y = G.dropout_words_(x.clone(), w, E.DROPOUT_P)
    drop = w.cpu().numpy().view(np.uint32).astype(np.uint64) < THR
    ref = (x.float() * 1.25).to(dtype).cpu()
    ref[torch.from_numpy(drop)] = 0
    assert torch.equal(y.cpu(), ref)
    assert drop[0] and not drop[1] and not drop[2] and drop[3]


def test_heads_dropout(sd):
    H, W = _small_hw()
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    feats, rl, rr = _test_rois(eng, H, W, 1)
    R = rl.shape[0]
    words = _words((2, R, 2048), 3)
    with torch.no_grad():
        _, s0 = eng.heads(feats, 1, rl, rr, float(H), save_for_backward=True)
        _, s1 = eng.heads(feats, 1, rl, rr, float(H), save_for_backward=True, dropout_words=words)
    torch.cuda.synchronize()
    assert s1.dropout
    drop = torch.from_numpy(words.cpu().numpy().view(np.uint32).astype(np.int64) < THR)
    x0, x1 = s0.top0.view(R, 2048).cpu(), s1.top0.view(R, 2048).cpu()
    ref = (x0.float() * 1.25).half()
    ref[drop[0] | (x0 <= 0)] = 0
    assert torch.equal(x1, ref)
    f1 = s1.fc7.cpu()
    assert bool((f1[drop[1]] == 0).all()) and bool((f1 >= 0).all())
    kept = 1.0 - drop.double().mean().item()
    sigma = (0.8 * 0.2 / drop.numel()) ** 0.5
    print("dropout: kept fraction %.5f over %d words (0.8 +- %.1e)" % (kept, drop.numel(), sigma))
    assert abs(kept - 0.8) < 5 * sigma


# ---------------------------------------------------------------- 3. the new kernels against float64
def _box_case(R, C, seed):
    g = torch.Generator().manual_seed(seed)
    K = 2048
    fc7 = torch.relu(torch.randn(R, K, generator=g))
    ws = [torch.randn(n * C, K, generator=g) * 0.02 for n in (1, 6, 5)]
    ds = [torch.randn(R, n * C, generator=g) * 1e-2 for n in (1, 6, 5)]
    return fc7, ws, ds


@pytest.mark.parametrize("R", [1, 37, 512])
@pytest.mark.parametrize("C", [2, 3])
def test_box_tail_backward_vs_float64(R, C):
    fc7, ws, ds = _box_case(R, C, R + C)
    K = fc7.shape[1]
    gs, ms = 8.0, 1.25
    outs = [guarded(s, torch.float32) for s in ((C, K), (C,), (6 * C, K), (6 * C,), (5 * C, K), (5 * C,))]
    nf = torch.zeros(1, dtype=torch.int32, device="cuda")
    dz16, dz32 = G.box_tail_backward(*[d.cuda() for d in ds], fc7.cuda(), *[w.cuda() for w in ws],
                                     [o[0] for o in outs], mask_scale=ms, grad_scale=gs, nonfinite=nf)
    torch.cuda.synchronize()
    for o in outs:
        o[1]()
    d = torch.cat([t.double() for t in ds], 1)
    W = torch.cat([t.double() for t in ws], 0)
    f = fc7.double()
    dz = (d @ W) * (f > 0).double() * ms * gs
    errs = {"dz32": l2_err(dz32, dz), "dz16": l2_err(dz16, h16(dz))}
    lo = 0
    for i, n in enumerate((1, 6, 5)):
        errs["dw%d" % i] = l2_err(outs[2 * i][0], d[:, lo:lo + n * C].t() @ f)
        errs["db%d" % i] = l2_err(outs[2 * i + 1][0], d[:, lo:lo + n * C].sum(0))
        lo += n * C
    print("box_tail_backward R=%d C=%d vs float64: %s" % (R, C, ", ".join("%s %.1e" % kv for kv in errs.items())))
    assert all(e <= TAIL_TOL for k, e in errs.items() if k != "dz16"), errs
    assert errs["dz16"] <= KERNEL_TOL and int(nf.item()) == 0


def _kpts_ref(up, w, dkp, dl, dr, gs):
    """float64 on the GPU: up [R,G,G,C] (the fp16 values), w [6,C]"""
    R, Gd, _, C = up.shape
    u = up.double()
    dp = torch.cat([dkp.double().view(R, 4, Gd), dl.double().view(R, 1, Gd), dr.double().view(R, 1, Gd)], 1)
    g = torch.einsum("kc,rkx->rxc", w.double(), dp)                       # [R,x,C]
    on = (u > 0).double()
    dfull = g[:, None] * on                                                # [R,y,x,C]
    cs = u.sum(1)                                                          # [R,x,C]
    dw = torch.einsum("rkx,rxc->kc", dp, cs)
    db = dp.sum((0, 2)) * Gd
    dbu = dfull.sum((0, 1, 2))
    ph = (dfull * gs).view(R, Gd // 2, 2, Gd // 2, 2, C).permute(0, 1, 3, 2, 4, 5).reshape(R, Gd // 2, Gd // 2, 4 * C)
    return ph, dw, db, dbu


@pytest.mark.parametrize("R", [1, 37, 512])
def test_kpts_tail_backward_vs_float64(R):
    g = torch.Generator().manual_seed(R)
    Gd, C = 28, 256
    up = torch.relu(torch.randn(R, Gd, Gd, C, generator=g)).half().cuda()
    w = (torch.randn(6, C, generator=g) * 0.05).cuda()
    dkp, dl, dr = [(torch.randn(R, n * Gd, generator=g) * 1e-3).cuda() for n in (4, 1, 1)]
    gs = 1024.0
    outs = [guarded(s, torch.float32) for s in ((6 * C,), (6,), (C,))]
    nf = torch.zeros(1, dtype=torch.int32, device="cuda")
    dup = G.kpts_tail_backward(up, w, dkp, dl, dr, *[o[0] for o in outs], grad_scale=gs, nonfinite=nf)
    torch.cuda.synchronize()
    for o in outs:
        o[1]()
    ph, dw, db, dbu = _kpts_ref(up, w, dkp, dl, dr, gs)
    errs = {"dup16": l2_err(dup, h16(ph)), "dw": l2_err(outs[0][0], dw.view(-1)), "db": l2_err(outs[1][0], db),
            "db_up": l2_err(outs[2][0], dbu)}
    print("kpts_tail_backward R=%d vs float64: %s" % (R, ", ".join("%s %.1e" % kv for kv in errs.items())))
    assert errs["dup16"] <= KERNEL_TOL and all(errs[k] <= TAIL_TOL for k in ("dw", "db", "db_up")), errs
    assert int(nf.item()) == 0
    # an fp16 overflow of the scaled gradient sets the flag
    G.kpts_tail_backward(up, w, dkp * 1e9, dl, dr, *[o[0] for o in outs], grad_scale=2.0 ** 20, nonfinite=nf)
    torch.cuda.synchronize()
    assert int(nf.item()) == 1


def test_permute3_reference_layouts():
    g = torch.Generator().manual_seed(4)
    a = torch.randn(2048, 49 * 512, generator=g).cuda()          # [co][(ph,pw,c)] -> [co][c][ph][pw]
    out = torch.empty(2048, 512, 7, 7, device="cuda")
    G.permute3(a, (2048, 49, 512), (49 * 512, 1, 49), out)
    assert torch.equal(out, a.view(2048, 7, 7, 512).permute(0, 3, 1, 2))
    b = torch.randn(1024, 256, generator=g).cuda()               # [(a,b,co)][ci] -> [ci][co][a][b]
    out = torch.empty(256, 256, 2, 2, device="cuda")
    G.permute3(b, (4, 256, 256), (1, 4, 1024), out)
    assert torch.equal(out, b.view(2, 2, 256, 256).permute(3, 2, 0, 1))


def test_new_entry_points_reject_invalid_arguments():
    """every refusal returns SB_EINVAL before any launch"""
    L = _l.load()
    st = G.stream_ptr()
    buf = torch.zeros(1 << 20, device="cuda")
    p = lambda off=0: ctypes.c_void_p(buf.data_ptr() + off)
    ws_n = L.sb_kpts_tail_backward_workspace(4, 256)
    torch.cuda.synchronize()
    n0 = G.launch_count()

    def box(R=4, K=64, nc=2, ms=1.0, gs=1.0, dz16=None):
        return L.sb_box_tail_backward(p(), p(), p(), p(), R, K, nc, p(), p(), p(), ms, gs, p(), p(), p(), p(), p(), p(),
                                      dz16 or p(), p(), None, st)

    def kpts(R=4, Gd=28, C=256, gs=1.0, up=None, nb=ws_n, ws=None):
        return L.sb_kpts_tail_backward(up or p(), R, Gd, C, p(), p(), p(), p(), gs, p(), p(), p(), p(), None,
                                       ws or p(), nb, st)

    def perm(d=(4, 5, 6), s=(30, 6, 1), dst=None):
        return L.sb_permute3(p(), *d, *s, dst or p(1 << 19), st)
    bad = {"box R=0": box(R=0), "box nc=5": box(nc=5), "box nc=0": box(nc=0), "box K=0": box(K=0),
           "box mask_scale 0": box(ms=0.0), "box grad_scale inf": box(gs=float("inf")),
           "box misaligned dz16": box(dz16=p(1)),
           "kpts R=0": kpts(R=0), "kpts odd G": kpts(Gd=27), "kpts G=66": kpts(Gd=66), "kpts C%32": kpts(C=100),
           "kpts C>1024": kpts(C=2048), "kpts gs 0": kpts(gs=0.0), "kpts misaligned up": kpts(up=p(1)),
           "kpts short workspace": kpts(nb=ws_n - 1), "kpts misaligned workspace": kpts(ws=p(2)),
           "dropout p=1": L.sb_dropout_words(p(), 0, 16, p(), 1.0, st),
           "dropout p<0": L.sb_dropout_words(p(), 0, 16, p(), -0.1, st),
           "dropout n<0": L.sb_dropout_words(p(), 0, -1, p(), 0.2, st),
           "dropout misaligned half": L.sb_dropout_words(p(1), 1, 16, p(), 0.2, st),
           "logits G=0": L.sb_kpts_logits(p(), 4, 0, p(), p(), p(), st),
           "logits null": L.sb_kpts_logits(p(), 4, 28, None, p(), p(), st),
           "scores null": L.sb_box_tail_scores(p(), 4, 64, 2, *[p()] * 9, None, st),
           "perm not dense": perm(s=(30, 6, 2)), "perm overlap": perm(dst=p(4)), "perm d0=0": perm(d=(0, 5, 6)),
           "perm repeated stride": perm(s=(1, 6, 1))}
    assert G.launch_count() == n0
    assert all(rc == SB_EINVAL for rc in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}
    assert perm() == 0 and box() == 0


# ---------------------------------------------------------------- 4. heads_backward layer by layer against float64
def _heads_backward_ref(eng, sd, saved, d, gs):
    """float64 on the GPU, layer by layer: fp16-rounded weights, the engine's saved fp16 operands and masks, and the
    engine's own fp16 inter-layer gradients (recomputed with the same deterministic kernels, so the same bits as inside
    heads_backward) as each layer's input.  Returns the references and the engine's inter-layer fp32 gradients with
    theirs."""
    R = saved.R
    d_cls, d_box, d_dim, dkp, dl, dr = d
    keep = 1.25 if saved.dropout else 1.0
    ref, mid = {}, {}
    fc7 = saved.fc7.double()
    fcw = [t.double() for t in eng.fc]
    dd = torch.cat([d_cls.double(), d_box.double(), d_dim.double()], 1)
    Wt = torch.cat([fcw[0], fcw[2], fcw[4]], 0)
    nc = d_cls.shape[1]
    lo = 0
    for name, n in (("RCNN_cls_score", 1), ("RCNN_bbox_pred", 6), ("RCNN_dim_orien_pred", 5)):
        ref[name + ".weight"] = dd[:, lo:lo + n * nc].t() @ fc7
        ref[name + ".bias"] = dd[:, lo:lo + n * nc].sum(0)
        lo += n * nc
    scratch = [torch.empty(n * nc * k, device="cuda") for n in (1, 6, 5) for k in (2048, 1)]
    dz16, dz32 = G.box_tail_backward(d_cls, d_box, d_dim, saved.fc7, eng.fc[0], eng.fc[2], eng.fc[4], scratch,
                                     mask_scale=keep, grad_scale=gs)
    mid["dz"] = (dz32, (dd @ Wt) * (fc7 > 0).double() * keep * gs)
    x0 = saved.top0.view(R, 2048).double()
    ref["RCNN_top.3.weight"] = (dz16.double().t() @ x0 / gs).view(2048, 2048, 1, 1)
    ref["RCNN_top.3.bias"] = dz32.double().sum(0) / gs
    w3 = h16(sd["RCNN_top.3.weight"].view(2048, 2048).cuda())
    t3 = eng._bwd["RCNN_top.3"]
    d0_32 = torch.empty(R, 1, 1, 2048, device="cuda")
    d0_16 = torch.empty(R, 1, 1, 2048, dtype=torch.float16, device="cuda")
    kv = G.fill_(torch.empty(2048, device="cuda"), keep) if saved.dropout else None
    G.conv2d_dgrad(G.conv_desc(dz16.view(R, 1, 1, 2048), t3.w16, d0_32, 2048, 2048, 1, 1, 1, 0, 1, 1, scale=kv,
                               out16=d0_16), saved.top0)
    mid["d0"] = (d0_32.view(R, 2048), (dz16.double() @ w3) * (x0 > 0).double() * keep)
    d0 = d0_16.view(R, 2048).double()
    pooled = saved.pooled_box.view(R, -1).double()
    ref["RCNN_top.0.weight"] = (d0.t() @ pooled / gs).view(2048, 7, 7, 512).permute(0, 3, 1, 2)
    ref["RCNN_top.0.bias"] = d0_32.double().sum((0, 1, 2)) / gs
    w0 = h16(sd["RCNN_top.0.weight"].permute(0, 2, 3, 1).reshape(2048, -1).cuda())     # [co][(ph, pw, c)]
    dpool = (d0 @ w0 / gs).view(R, 7, 7, 512)
    ph, dw, db, dbu = _kpts_ref(saved.up, eng.kpts_class[0], dkp, dl, dr, gs)
    ref["kpts_class.weight"], ref["kpts_class.bias"], ref["RCNN_kpts.12.bias"] = dw.view(6, 256, 1, 1), db, dbu
    scratch = [torch.empty(n, device="cuda") for n in (6 * 256, 6, 256)]
    dup16 = G.kpts_tail_backward(saved.up, eng.kpts_class[0], dkp, dl, dr, *scratch, grad_scale=gs)
    mid["dup"] = (dup16, h16(ph))
    x6 = saved.kpts[5].double()
    dph = dup16.double()                                                # [R,14,14,(a,b,co)]
    ref["RCNN_kpts.12.weight"] = torch.einsum("rijp,rijc->pc", dph, x6).view(2, 2, 256, 256).permute(3, 2, 0, 1) / gs
    wd = h16(sd["RCNN_kpts.12.weight"].cuda())                          # [ci,co,a,b]
    wf = wd.permute(2, 3, 1, 0).reshape(1024, 256)
    g32, g16 = eng._dgrad(dup16, "deconv", mask=saved.kpts[5])
    mid["d kpts.10 out"] = (g32, (dph @ wf) * (x6 > 0).double())
    for i in range(5, -1, -1):
        key = "RCNN_kpts.%d" % (2 * i)
        xin = (saved.kpts[i - 1] if i > 0 else saved.pooled_kpts).double()
        g = g16.double().permute(0, 3, 1, 2)
        ref[key + ".weight"] = torch.nn.grad.conv2d_weight(xin.permute(0, 3, 1, 2), (256, 256, 3, 3), g,
                                                           padding=1) / gs
        ref[key + ".bias"] = g32.double().sum((0, 1, 2)) / gs
        nxt = F.conv_transpose2d(g, h16(sd[key + ".weight"].cuda()), padding=1).permute(0, 2, 3, 1)
        if i > 0:
            g32, g16 = eng._dgrad(g16, key, mask=saved.kpts[i - 1])
            mid["d kpts.%d out" % (2 * i - 2)] = (g32, nxt * (xin > 0).double())
    return ref, {"pooled_box": dpool, "pooled_kpts": nxt / gs}, mid


@pytest.mark.parametrize("dropout", [False, True])
def test_heads_backward_vs_float64_from_state_dict(sd, dropout):
    H, W = _small_hw()
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    feats, rl, rr = _test_rois(eng, H, W, 1)
    R = rl.shape[0]
    with torch.no_grad():
        out, saved = eng.heads(feats, 1, rl, rr, float(H), save_for_backward=True,
                               dropout_words=_words((2, R, 2048), 4) if dropout else None)
    g = torch.Generator().manual_seed(6)
    d = [(torch.randn(*out[k].shape, generator=g) * 1e-2).cuda()
         for k in ("cls_score", "bbox_pred", "dim_orien_pred", "kpts_pred", "left_border_pred", "right_border_pred")]
    gs = 2.0 ** 10
    got, dpool = eng.heads_backward(saved, *d, grad_scale=gs)
    torch.cuda.synchronize()
    assert int(eng.found_inf.item()) == 0
    assert sorted(got) == sorted(n for n, _ in E.trainable_rcnn_head_params())
    with torch.no_grad():
        ref, rpool, mid = _heads_backward_ref(eng, sd, saved, d, gs)
    errs = {n: l2_err(got[n], ref[n]) for n in ref}
    errs.update({"d" + k: l2_err(dpool[k], rpool[k]) for k in rpool})
    errs.update({k: l2_err(a, b) for k, (a, b) in mid.items()})
    print("heads_backward R=%d dropout=%s vs float64: %s" % (R, dropout, ", ".join(
        "%s %.2e" % kv for kv in sorted(errs.items(), key=lambda kv: -kv[1]))))
    assert dpool["pooled_box"].shape == (R, 7, 7, 512) and dpool["pooled_kpts"].shape == (R, 14, 14, 256)
    assert all(e < KERNEL_TOL for e in errs.values()), errs


# ---------------------------------------------------------------- 5. end to end against fp32 autograd
def _oracle_heads(sd, pooled, pooled_k, words, tgt, names, weights16=False):
    """fp32 autograd (TF32 off) through a train-mode restatement of oracle.model.box_head / kpts_head (dropout with
    the engine's masks) and oracle.train_targets.rcnn_losses"""
    sdd = {k: v.cuda() for k, v in sd.items()}
    if weights16:
        sdd = {k: (v.half().float() if k.endswith("weight") else v) for k, v in sdd.items()}
    for n in names:
        sdd[n] = sdd[n].clone().requires_grad_(True)
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        with torch.enable_grad():
            pb = pooled.float().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
            pk = pooled_k.float().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
            R = pb.shape[0]
            keep = [None, None]
            if words is not None:
                w = words.cpu().numpy().view(np.uint32).astype(np.int64) >= THR
                keep = [torch.from_numpy(w[i]).float().cuda().view(R, 2048, 1, 1) * 1.25 for i in range(2)]
            x = F.relu(F.conv2d(pb, sdd["RCNN_top.0.weight"], sdd["RCNN_top.0.bias"], stride=7))
            x = x * keep[0] if keep[0] is not None else x
            x = F.relu(F.conv2d(x, sdd["RCNN_top.3.weight"], sdd["RCNN_top.3.bias"]))
            x = x * keep[1] if keep[1] is not None else x
            fc7 = x.mean(3).mean(2)
            cls = F.linear(fc7, sdd["RCNN_cls_score.weight"], sdd["RCNN_cls_score.bias"])
            bbox = F.linear(fc7, sdd["RCNN_bbox_pred.weight"], sdd["RCNN_bbox_pred.bias"])
            dim = F.linear(fc7, sdd["RCNN_dim_orien_pred.weight"], sdd["RCNN_dim_orien_pred.bias"])
            y = pk
            for k in range(0, 12, 2):
                y = F.relu(F.conv2d(y, sdd["RCNN_kpts.%d.weight" % k], sdd["RCNN_kpts.%d.bias" % k], padding=1))
            y = F.relu(F.conv_transpose2d(y, sdd["RCNN_kpts.12.weight"], sdd["RCNN_kpts.12.bias"], stride=2))
            ka = F.conv2d(y, sdd["kpts_class.weight"], sdd["kpts_class.bias"]).sum(2)
            g = ka.shape[2]
            losses = T.rcnn_losses(cls.cpu(), bbox.cpu(), dim.cpu(), ka[:, :4].reshape(-1, 4 * g).cpu(),
                                   ka[:, 4].cpu(), ka[:, 5].cpu(), tgt)
            total = sum(losses)
            gr = torch.autograd.grad(total, [sdd[n] for n in names] + [pb, pk])
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
    ref = {n: t.detach() for n, t in zip(names, gr)}
    ref["pooled_box"] = gr[-2].permute(0, 2, 3, 1)
    ref["pooled_kpts"] = gr[-1].permute(0, 2, 3, 1)
    return [float(l.detach()) for l in losses], ref


def _tol(n):
    return KPTS_TOL if n.startswith(("RCNN_kpts.", "pooled_")) else MODEL_TOL


def _end_to_end(sd, H, W, dropout, seed):
    B = 1
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    im = _pairs(H, W, B, seed).cuda()
    gl, gr, gm, dim, kp, _nb = [torch.from_numpy(t).cuda() for t in synth_train_gt(B, 30, H, W, seed)]
    keys = _words((B, 2000 + 30), seed + 1)
    words = _words((B, 512), seed + 2)
    dw = _words((2, B * 512, 2048), seed + 3) if dropout else None
    losses, got, dpool = TR.rcnn_head_gradients(eng, im[:B], im[B:], gl, gr, gm, dim, kp, keys, words,
                                                dropout_words=dw, grad_scale=2.0 ** 12)
    torch.cuda.synchronize()
    assert int(eng.found_inf.item()) == 0
    # the same forward again for the pooled features and the targets the oracle reads
    with torch.no_grad():
        feats = eng.trunk_fpn(torch.cat((im[:B], im[B:]), 0))
        cp, bb, shapes = eng.rpn(feats, B)
        rl, rr = G.proposal_layer(cp, bb, TR._im_info(B, H, W, "cuda"), "TRAIN", shapes)
        tgt = TR.proposal_targets(rl, rr, gl, gr, dim, kp, keys, words)
        out, saved = eng.heads(feats, B, tgt["rois_left"].view(-1, 5), tgt["rois_right"].view(-1, 5), float(H),
                               save_for_backward=True, dropout_words=dw)
    names = [n for n, _ in E.trainable_rcnn_head_params()]
    got.update(dpool)
    tg = {k: v.cpu() for k, v in tgt.items()}
    rl_, ref = _oracle_heads(sd, saved.pooled_box, saved.pooled_kpts, dw, tg, names)
    label = "%dx%d dropout=%s" % (H, W, dropout)
    print("%s: losses %s vs oracle %s" % (label, losses.cpu().tolist(), rl_))
    for a, b in zip(losses.cpu().tolist(), rl_):
        assert abs(a - b) <= LOSS_TOL * abs(b), (a, b)
    worst = sorted(((l2_err(got[n], ref[n]), n) for n in ref), reverse=True)
    print("%s: relative L2 error per tensor: %s" % (label, ", ".join("%s %.2e" % (n, e) for e, n in worst)))
    _, ref16 = _oracle_heads(sd, saved.pooled_box, saved.pooled_kpts, dw, tg, names, weights16=True)
    w16 = sorted(((l2_err(ref16[n], ref[n]), n) for n in ref), reverse=True)
    print("%s: oracle with fp16-rounded weights vs fp32: %s" % (label, ", ".join("%s %.2e" % (n, e) for e, n in w16)))
    bad = [(n, e) for e, n in worst if not e < _tol(n)]
    assert not bad, bad


@pytest.mark.parametrize("dropout", [False, True])
def test_rcnn_head_gradients_small_vs_oracle(sd, dropout):
    H, W = _small_hw()
    _end_to_end(sd, H, W, dropout, 7)


@pytest.mark.parametrize("dropout", [False, True])
def test_rcnn_head_gradients_benchmark_size_vs_oracle(sd, dropout):
    _end_to_end(sd, 600, 1987, dropout, 3)


# ---------------------------------------------------------------- 6-7. determinism, capture, scaling, overflow, uncert
@pytest.fixture(scope="module")
def step_case(sd):
    H, W = _small_hw()
    B = 1
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    im = _pairs(H, W, B, 7).cuda()
    gt = [torch.from_numpy(t).cuda() for t in synth_train_gt(B, 30, H, W, 7)[:5]]
    keys = _words((B, 2030), 8)
    words = _words((B, 512), 9)
    dw = _words((2, 512, 2048), 10)
    return eng, im[:B].contiguous(), im[B:].contiguous(), gt, keys, words, dw


def test_rcnn_head_gradients_deterministic_into_given_buffers_and_graph_capturable(step_case):
    eng, iml, imr, gt, keys, words, dw = step_case
    l0, a, pa = TR.rcnn_head_gradients(eng, iml, imr, *gt, keys, words, dropout_words=dw)
    a = {k: v.clone() for k, v in a.items()}
    a.update({k: v.clone() for k, v in pa.items()})
    l0 = l0.clone()
    bufs = {n: torch.full(s, float("nan"), device="cuda") for n, s in E.trainable_rcnn_head_params()}
    l1, b, pb = TR.rcnn_head_gradients(eng, iml, imr, *gt, keys, words, dropout_words=dw, grads=bufs)
    torch.cuda.synchronize()
    assert torch.equal(l0, l1)
    b = dict(b, **pb)
    for n in a:
        if n in bufs:
            assert b[n].data_ptr() == bufs[n].data_ptr(), n
        assert torch.equal(a[n], b[n]), n

    def step(x, y):
        return TR.rcnn_head_gradients(eng, x, y, *gt, keys, words, dropout_words=dw)
    with torch.no_grad():
        runner = E.GraphRunner(step, [iml, imr])
        lg, out, po = runner()
        torch.cuda.synchronize()
    assert torch.equal(lg, l0)
    out = dict(out, **po)
    for n in a:
        assert torch.equal(out[n], a[n]), n


def test_rcnn_head_gradients_scaling_overflow_and_uncert(step_case):
    eng, iml, imr, gt, keys, words, dw = step_case
    H = iml.shape[2]
    with torch.no_grad():
        f = eng.trunk_fpn(torch.cat((iml, imr), 0))
        cp, bb, shapes = eng.rpn(f, 1)
        rl, rr = G.proposal_layer(cp, bb, TR._im_info(1, H, iml.shape[3], "cuda"), "TRAIN", shapes)
        tgt = TR.proposal_targets(rl, rr, gt[0], gt[1], gt[3], gt[4], keys, words)
        out, saved = eng.heads(f, 1, tgt["rois_left"].view(-1, 5), tgt["rois_right"].view(-1, 5), float(H),
                               save_for_backward=True, dropout_words=dw)
    g = torch.Generator().manual_seed(11)
    d = [(torch.randn(*out[k].shape, generator=g) * 1e-3).cuda()
         for k in ("cls_score", "bbox_pred", "dim_orien_pred", "kpts_pred", "left_border_pred", "right_border_pred")]

    def run(scale, gs):
        r, p = eng.heads_backward(saved, *[t * scale for t in d], grad_scale=gs)
        r = dict({k: v.clone() for k, v in r.items()}, **{k: v.clone() for k, v in p.items()})
        torch.cuda.synchronize()
        return r, int(eng.found_inf.item())
    base, fi = run(1.0, 1.0)
    assert fi == 0
    tiny, fi = run(1e-6, 2.0 ** 20)
    assert fi == 0
    errs = {n: l2_err(tiny[n], base[n] * 1e-6) for n in base}
    print("grad_scale 2^20 on 1e-6 gradients vs unscaled: worst %s" % (max(errs.items(), key=lambda kv: kv[1]),))
    # the unscaled run itself loses the gradients below fp16's normal range, as in test_gpu_rpn_backward
    assert all(e < MODEL_TOL for e in errs.values()), errs
    _, fi = run(1.0, 2.0 ** 40)
    assert fi == 1
    _, fi = run(1.0, 1.0)
    assert fi == 0
    # the multi-task weights: d total / d uncert[2:6] = 1 - L_i exp(-u_i), gradients scaled by exp(-u_i)
    u = torch.tensor([0.3, -0.2, 0.1, 0.0, 0.5, -0.4], device="cuda")
    l0, a, _ = TR.rcnn_head_gradients(eng, iml, imr, *gt, keys, words, dropout_words=dw)
    l0 = l0.clone()
    a = {k: v.clone() for k, v in a.items()}
    l1, b, _, du = TR.rcnn_head_gradients(eng, iml, imr, *gt, keys, words, dropout_words=dw, uncert=u)
    torch.cuda.synchronize()
    assert torch.equal(l0, l1)
    L_ = l0.cpu().double().numpy()
    uc = u.cpu().double().numpy()[2:6]
    np.testing.assert_allclose(du.cpu().numpy(), 1 - L_ * np.exp(-uc), rtol=1e-5)
    f0 = float(np.exp(-uc[0]))           # the class scores read only the class loss
    assert l2_err(b["RCNN_cls_score.bias"], a["RCNN_cls_score.bias"] * f0) < 1e-6
