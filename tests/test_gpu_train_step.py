"""GPU: the training step -- sb_sgd_step against a float32 numpy restatement (bit for bit) and torch.optim.SGD (2 ulp),
engine.refresh_weights against a freshly built engine (bit for bit, in place, under a captured forward), and
train.Trainer: one step against its parts, eager against graph-replayed, the overflow skip, the checkpoint, progress
on a fixed batch and two data-parallel ranks against one process on the averaged gradients."""
import os

import numpy as np
import pytest
import torch

from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200 import train as TR
from stereo_rcnn_b200.synth import make_state_dict, synth_pair, synth_train_gt

pytestmark = pytest.mark.gpu

H, W = 160, 256
GS = 2.0 ** 12


def bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int32) if t.element_size() == 4 else t.view(torch.int16)


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(bits(a), bits(b))


def ulps_of_operands(got, ref, *operands):
    """|got - ref| in units in the last place of the largest of the update's operands and result: an FMA that skips
    one rounding of a product moves the result by up to half an ulp of that product, which is many ulps of a result
    that cancels to near zero"""
    scale = np.max(np.abs(np.stack([np.asarray(o, np.float32) for o in operands])), axis=0).astype(np.float32)
    return np.abs(got.astype(np.float64) - ref.astype(np.float64)) / np.spacing(np.maximum(scale, np.float32(1e-30)))


def np_sgd(p, g, m, wd, lrm, lr32, mom):
    """the documented order of sb_sgd_step, one float32 rounding per operation"""
    f = np.float32
    d = g + f(wd) * p
    m = f(mom) * m + d
    return p - (f(lr32) * f(lrm)) * m, m


# ------------------------------------------------------------------------------------------------ 1. sb_sgd_step
def _sgd_case(counts, seed, misalign=False):
    rs = np.random.RandomState(seed)
    host = [[rs.standard_normal(n).astype(np.float32) for n in counts] for _ in range(3)]
    host[2] = [np.zeros(n, np.float32) for n in counts]             # momentum buffers start at zero, as torch's

    def dev(a):
        if not misalign:
            return torch.from_numpy(a).cuda()
        buf = torch.empty(a.size + 1, dtype=torch.float32, device="cuda")   # 4-byte aligned only: the scalar path
        v = buf[1:]
        v.copy_(torch.from_numpy(a))
        return v
    return host, [[dev(a) for a in h] for h in host]


SGD_CASES = {"counts 1..9": list(range(1, 10)), "47 tensors": [3] * 47, "48 tensors": [5] * 48,
             "49 tensors": [7] * 48 + [4097], "97 tensors": [1, 2, 3, 4] * 24 + [9],
             "CTA edges": [4095, 4096, 4097, 8191, 8192, 8193, 4 * 4096 + 3]}


@pytest.mark.parametrize("case", sorted(SGD_CASES) + ["misaligned", "all 140 real shapes"])
@pytest.mark.parametrize("wd,lrm,mom", [(0.0, 1.0, 0.0), (1e-4, 2.0, 0.9), (1e-4, 1.0, 0.9), (0.0, 2.0, 0.9)])
def test_sgd_step_bitwise_against_numpy(case, wd, lrm, mom, capsys):
    """sb_sgd_step equals its float32 numpy restatement bit for bit over five steps with lr changed between them, and
    torch.optim.SGD (groups as trainval_net.py builds them, each step from the same state) to within two ulps of the
    largest operand or result of each update: torch's CPU kernels contract some products into FMAs, which skips the
    rounding this kernel's documented order keeps"""
    if case == "all 140 real shapes":
        if (wd, lrm, mom) != (1e-4, 2.0, 0.9):
            pytest.skip("the real shapes run once")
        counts = [int(np.prod(s)) for _, s in TR.trainable_names(1)] + [6]
        assert len(counts) == 140
    else:
        counts = SGD_CASES.get(case, [1, 5, 4096 + 7, 33])
    host, d = _sgd_case(counts, 7, misalign=case == "misaligned")
    n = len(counts)
    wds = [wd * (i % 2) if n > 1 else wd for i in range(n)]                  # mixed groups
    lrms = [lrm if i % 3 else 1.0 for i in range(n)]
    lr = torch.zeros(1, device="cuda")
    skip = torch.zeros(1, dtype=torch.int32, device="cuda")
    skipped = torch.zeros(1, dtype=torch.int32, device="cuda")
    args = TR._SgdArgs(d[0], d[1], d[2], wds, lrms)
    worst = 0
    for step, lr_host in enumerate((1e-3, 1e-3, 1e-4, 3.3e-3, 0.1)):
        lr32 = np.float32(lr_host)
        lr.copy_(torch.tensor([lr_host], dtype=torch.float32))              # what Trainer.set_lr writes
        rs = np.random.RandomState(100 + step)
        for i in range(n):                                                   # new gradients every step
            host[1][i] = rs.standard_normal(counts[i]).astype(np.float32)
            d[1][i].copy_(torch.from_numpy(host[1][i]))
        # torch.optim.SGD on the CPU from the same state, groups as trainval_net.py builds them
        if case != "all 140 real shapes":
            tp = [torch.nn.Parameter(torch.from_numpy(host[0][i].copy())) for i in range(n)]
            opt = torch.optim.SGD([{"params": [tp[i]], "lr": lr_host * lrms[i], "weight_decay": wds[i]}
                                   for i in range(n)], momentum=mom)
            for i in range(n):
                tp[i].grad = torch.from_numpy(host[1][i].copy())
                if step > 0 and mom != 0:
                    opt.state[tp[i]]["momentum_buffer"] = torch.from_numpy(host[2][i].copy())
            opt.step()
        args(lr, mom, skip, skipped)
        torch.cuda.synchronize()
        for i in range(n):
            p_ref, m_ref = np_sgd(host[0][i], host[1][i], host[2][i], wds[i], lrms[i], lr32, mom)
            got_p, got_m = d[0][i].cpu().numpy(), d[2][i].cpu().numpy()
            assert np.array_equal(got_p.view(np.int32), p_ref.view(np.int32)), (case, step, i)
            assert np.array_equal(got_m.view(np.int32), m_ref.view(np.int32)), (case, step, i)
            if case != "all 140 real shapes":
                f = np.float32
                m_old = host[2][i]
                dd = host[1][i] + f(wds[i]) * host[0][i]
                worst = max(worst, float(ulps_of_operands(got_p, tp[i].detach().numpy(), host[0][i],
                                                          (lr32 * f(lrms[i])) * m_ref, got_p).max()))
                if mom != 0:
                    worst = max(worst, float(ulps_of_operands(got_m, opt.state[tp[i]]["momentum_buffer"].numpy(),
                                                              f(mom) * m_old, dd, host[1][i], got_m).max()))
            host[0][i], host[2][i] = p_ref, m_ref
    assert int(skipped.item()) == 0
    assert worst <= 2.0
    with capsys.disabled():
        print("sgd %s wd %g lr_mult %g momentum %g: numpy bit-exact over 5 steps%s" % (
            case, wd, lrm, mom, "" if case == "all 140 real shapes" else
            "; torch.optim.SGD within %.3g ulp of the largest operand" % worst))


def test_sgd_step_skip():
    host, d = _sgd_case([5, 4096 + 3] + [2] * 60, 3)                        # two chunks: counted once
    args = TR._SgdArgs(d[0], d[1], d[2], [1e-4] * 62, [1.0] * 62)
    before = [[bits(t).clone() for t in ts] for ts in d]
    lr = torch.full((1,), 1e-3, device="cuda")
    skip = torch.ones(1, dtype=torch.int32, device="cuda")
    skipped = torch.zeros(1, dtype=torch.int32, device="cuda")
    args(lr, 0.9, skip, skipped)
    args(lr, 0.9, skip, skipped)
    torch.cuda.synchronize()
    assert int(skipped.item()) == 2
    for ts, bs in zip(d, before):
        assert all(torch.equal(bits(t), b) for t, b in zip(ts, bs))
    skip.zero_()
    args(lr, 0.9, skip, skipped)
    torch.cuda.synchronize()
    assert int(skipped.item()) == 2 and not torch.equal(bits(d[0][0]), before[0][0])


# ------------------------------------------------------------------------------------------------ 2. refresh_weights
def engine_tensors(eng):
    """every device tensor the engine holds, by a stable name"""
    out = {}
    pcs = list(eng.p.items()) + [("deconv%d%d" % (a, b), eng.deconv[a][b]) for a in range(2) for b in range(2)]
    for k, pc in pcs:
        for f in ("w", "w16", "scale", "shift"):
            if getattr(pc, f) is not None:
                out["p.%s.%s" % (k, f)] = getattr(pc, f)
    for k, d in (eng._bwd or {}).items():
        out["bwd.%s" % k] = d.w16
    for i, t in enumerate(eng.fc):
        out["fc%d" % i] = t
    for i, t in enumerate(eng.kpts_class):
        out["kpts_class%d" % i] = t
    for i, t in enumerate(eng.stem):
        out["stem%d" % i] = t
    out["stem_w16"] = eng.stem_w16
    return out


def perturbed(sd, names, seed):
    g = torch.Generator().manual_seed(seed)
    out = dict(sd)
    for n in names:
        v = sd[n].float()
        out[n] = (v + 0.05 * v.abs().mean() * torch.randn(v.shape, generator=g)).contiguous()
    return out


def small_inputs(seed=7, B=1):
    p = synth_pair(H, W, seed, 12)
    iml, imr = [torch.from_numpy(x[None]).cuda().contiguous() for x in p[:2]]
    info = torch.tensor([[float(H), float(W), 1.0]], device="cuda")
    return iml, imr, info


def forward_outputs(out):
    return {k: v for k, v in out.items() if torch.is_tensor(v)}


@pytest.mark.parametrize("fixed_blocks", [0, 1])
def test_refresh_equals_a_fresh_engine(fixed_blocks, capsys):
    sd = make_state_dict(3)
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    eng._pack_heads_backward()
    iml, imr, info = small_inputs()
    with torch.no_grad():
        runner = E.GraphRunner(lambda x, y: forward_outputs(eng.forward(x, y, info)), [iml, imr])
    names = [n for n, _ in TR.trainable_names(fixed_blocks)]
    sd2 = perturbed(sd, names, 11 + fixed_blocks)
    before = {k: (t.data_ptr(), bits(t).clone()) for k, t in engine_tensors(eng).items()}
    eng.refresh_weights({n: sd2[n].cuda() for n in names})
    torch.cuda.synchronize()
    fresh = E.StereoRCNNEngine(sd2, "cuda", precision="fp16")
    fresh._pack_heads_backward()
    got, ref = engine_tensors(eng), engine_tensors(fresh)
    assert sorted(got) == sorted(ref)
    changed = 0
    for k in ref:
        assert got[k].data_ptr() == before[k][0], k
        assert same_bits(got[k], ref[k]), k
        changed += not torch.equal(bits(got[k]), before[k][1])
    frozen = [k for k in ref if k.startswith(("p.stem", "stem")) or k.endswith(".scale")
              or (k.startswith("p.RCNN_layer") and k.endswith(".shift"))
              or any(k.startswith(pre + "RCNN_layer%d." % li) for li in range(1, fixed_blocks + 1)
                     for pre in ("p.", "bwd."))]
    assert frozen and all(torch.equal(bits(got[k]), before[k][1]) for k in frozen)
    with torch.no_grad():
        replay = runner()
        eager = forward_outputs(fresh.forward(iml, imr, info))
        torch.cuda.synchronize()
    for k in eager:
        assert same_bits(replay[k], eager[k]), k
    with capsys.disabled():
        print("refresh at FIXED_BLOCKS %d: %d engine tensors bit-identical to a fresh engine (%d rewritten, %d frozen "
              "untouched), pointers unchanged, captured forward = fresh eager forward" % (
                  fixed_blocks, len(ref), changed, len(frozen)))


# ------------------------------------------------------------------------------------------------ 3-5. Trainer
def _words(shape, seed):
    w = np.random.RandomState(seed).randint(0, 2 ** 32, shape, dtype=np.uint64).astype(np.uint32)
    return torch.from_numpy(w.view(np.int32)).cuda()


def batch(seed=7):
    iml, imr, _ = small_inputs(seed)
    gt = [torch.from_numpy(t).cuda() for t in synth_train_gt(1, 30, H, W, seed)[:5]]
    shapes = [[-(-H // s), -(-W // s)] for s in (4, 8, 16, 32, 64)]
    return (iml, imr, *gt, _words((1, 2030), seed + 2), _words((1, 512), seed + 3),
            _words((1, 3 * sum(h * w for h, w in shapes)), seed + 1)), _words((2, 512, 2048), seed + 4)


def snapshot(tr):
    return ([bits(v).clone() for v in tr.masters.grads], [bits(v).clone() for v in tr.moms.grads],
            {k: bits(t).clone() for k, t in engine_tensors(tr.engine).items()})


def test_step_equals_its_parts():
    sd = make_state_dict(3)
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    tr = TR.Trainer(eng, sd, grad_scale=GS)
    args, dw = batch()
    p0 = [v.cpu().numpy() for v in tr.masters.grads]
    u = tr.uncert.clone()
    losses_m, g, du = TR.loss_gradients(eng, *args, dropout_words=dw, uncert=u, grad_scale=GS)
    gl = [g[n].clone() for n in tr.names]
    norm_m = TR.clip_gradient(gl, 10.0)
    gl = [x.cpu().numpy() for x in gl] + [du.cpu().numpy()]
    torch.cuda.synchronize()
    assert int(eng.found_inf.item()) == 0
    losses, total, norm, skipped = tr.step(*args, dropout_words=dw)
    torch.cuda.synchronize()
    assert torch.equal(losses, losses_m) and torch.equal(norm, norm_m) and int(skipped.item()) == 0
    L_, uc = losses.double().cpu().numpy(), u.double().cpu().numpy()
    np.testing.assert_allclose(float(total), float((L_ * np.exp(-uc) + uc).sum()), rtol=1e-5)
    lr32 = np.float32(1e-3)
    for i, (p, gg, (lrm, wd)) in enumerate(zip(p0, gl, tr.groups)):
        p_ref, m_ref = np_sgd(p, gg, np.zeros_like(p), wd, lrm, lr32, 0.9)
        assert np.array_equal(tr.masters.grads[i].cpu().numpy().view(np.int32), p_ref.view(np.int32)), i
        assert np.array_equal(tr.moms.grads[i].cpu().numpy().view(np.int32), m_ref.view(np.int32)), i
    # the engine now holds exactly the packing of the new masters; a fresh engine from the checkpoint agrees
    fresh = E.StereoRCNNEngine(tr.state_dict(), "cuda", precision="fp16")
    fresh._pack_heads_backward()
    got, ref = engine_tensors(eng), engine_tensors(fresh)
    assert all(same_bits(got[k], ref[k]) for k in ref)
    iml, imr, info = small_inputs()
    with torch.no_grad():
        a, b = forward_outputs(eng.forward(iml, imr, info)), forward_outputs(fresh.forward(iml, imr, info))
    assert all(same_bits(a[k], b[k]) for k in b)
    ck = tr.checkpoint()
    assert same_bits(ck["uncert"], tr.uncert.cpu()) and sorted(ck["momentum"]) == sorted(tr.names + ["uncert"])
    assert sorted(ck["model"]) == sorted(k for k in sd)


def test_eager_and_graph_replayed_steps_agree():
    sd = make_state_dict(3)
    args, dw = batch()
    tra = TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, grad_scale=GS)
    trb = TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, grad_scale=GS)
    for _ in range(3):
        tra.step(*args, dropout_words=dw)
    with torch.no_grad():
        runner = E.GraphRunner(lambda *x: trb.step(*x, dropout_words=dw), list(args), warmup=2)   # steps 1, 2
        runner()                                                                                    # step 3
    torch.cuda.synchronize()
    sa, sb = snapshot(tra), snapshot(trb)
    assert all(torch.equal(x, y) for x, y in zip(sa[0] + sa[1], sb[0] + sb[1]))
    assert all(torch.equal(sa[2][k], sb[2][k]) for k in sa[2])
    # an lr change between replays takes effect
    tra.set_lr(3e-4)
    trb.set_lr(3e-4)
    tra.step(*args, dropout_words=dw)
    runner()
    torch.cuda.synchronize()
    sa, sb = snapshot(tra), snapshot(trb)
    assert all(torch.equal(x, y) for x, y in zip(sa[0] + sa[1], sb[0] + sb[1]))
    assert int(trb.skipped.item()) == 0


def test_overflow_skips_the_update():
    sd = make_state_dict(3)
    tr = TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, grad_scale=2.0 ** 40)
    args, dw = batch()
    tr.step(*args, dropout_words=dw)                 # warm: the first step of a fresh trainer overflows as well
    torch.cuda.synchronize()
    before = snapshot(tr)
    _, _, _, skipped = tr.step(*args, dropout_words=dw)
    torch.cuda.synchronize()
    assert int(tr.engine.found_inf.item()) == 1 and int(skipped.item()) == 2
    after = snapshot(tr)
    assert all(torch.equal(x, y) for x, y in zip(before[0] + before[1], after[0] + after[1]))
    assert all(torch.equal(before[2][k], after[2][k]) for k in before[2])


def test_progress_on_a_fixed_batch(capsys):
    sd = make_state_dict(3)
    tr = TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, grad_scale=GS)
    args, dw = batch(5)
    totals = []
    for _ in range(30):
        _, total, _, _ = tr.step(*args, dropout_words=dw)
        totals.append(float(total))
    with capsys.disabled():
        print("30 steps on one %dx%d batch, total loss: %s" % (H, W, " ".join("%.4f" % t for t in totals)))
    assert int(tr.skipped.item()) == 0 and all(np.isfinite(totals))
    assert np.mean(totals[-5:]) < np.mean(totals[:5])


def _dp_worker(rank, world, port, out_dir, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    try:
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        sd = make_state_dict(3)
        tr = TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, grad_scale=GS, world=world, dist=dist)
        args, dw = batch(20 + rank)
        for _ in range(3):
            tr.step(*args, dropout_words=dw)
        torch.cuda.synchronize()
        torch.save([b.cpu() for b in tr.masters.buckets], os.path.join(out_dir, "rank%d.pt" % rank))
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except Exception as e:             # reported to the parent
        q.put((rank, "%s: %s" % (type(e).__name__, e)))


def test_two_ranks_equal_one_process_on_averaged_gradients(tmp_path):
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, str(tmp_path), q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=900) for _ in range(2))
    for p in procs:
        p.join(timeout=120)
    assert res == [(0, "ok"), (1, "ok")], res
    r0, r1 = [torch.load(os.path.join(tmp_path, "rank%d.pt" % r)) for r in range(2)]
    assert all(same_bits(a, b) for a, b in zip(r0, r1))
    # one process: each rank's gradients on the same weights, averaged as the bucket all-reduce does, then the step
    sd = make_state_dict(3)
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    tr = TR.Trainer(eng, sd, grad_scale=GS)
    data = [batch(20 + r) for r in range(2)]
    for _ in range(3):
        parts = []
        for args, dw in data:
            _, g, du = TR.loss_gradients(eng, *args, dropout_words=dw, uncert=tr.uncert, grad_scale=GS)
            parts.append([g[n].clone() for n in tr.names] + [du.clone()])
            assert int(eng.found_inf.item()) == 0
        with torch.no_grad():
            for v, a, b in zip(tr.grads.grads, *parts):
                v.copy_((a + b) / 2)
        TR.clip_gradient(tr.grads.grads[:-1], 10.0, out=tr.norm)
        tr._sgd(tr.lr, tr.momentum, eng.found_inf, tr.skipped)
        eng.refresh_weights(tr.params)
    torch.cuda.synchronize()
    assert all(same_bits(a, b.cpu()) for a, b in zip(r0, tr.masters.buckets))
