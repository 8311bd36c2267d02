"""GPU: the dynamic loss scale -- each _devscale backward entry point bit for bit against its float twin,
sb_fill_reciprocal, loss_gradients with the scale as a device tensor against the float call, sb_loss_scale_update
against torch._amp_update_scale_ and its bounds, and train.Trainer with a DynamicLossScale: a captured step that backs
off from an overflowing scale, eager against replayed over a growth, a checkpoint resume, two data-parallel ranks, and
fit's log line."""
import os

import numpy as np
import pytest
import torch

from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200 import ops
from stereo_rcnn_b200 import train as TR
from stereo_rcnn_b200.synth import make_state_dict, synth_pair, synth_train_gt

pytestmark = pytest.mark.gpu

H, W = 160, 256
SCALES = [2.0 ** -3, 1.0, 2.0 ** 12]


def bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int32) if t.element_size() == 4 else t.view(torch.int16)


def same_bits(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(bits(a), bits(b))


def dev_scale(S):
    return torch.full((1,), S, dtype=torch.float32, device="cuda")


def flag():
    return torch.zeros(1, dtype=torch.int32, device="cuda")


def randn(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, generator=g, device="cuda") * scale


# ------------------------------------------------------------------------------------------------ 1. the twins
@pytest.mark.parametrize("S", SCALES)
@pytest.mark.parametrize("k", [1, 3])
@pytest.mark.parametrize("bad", [False, True])
def test_conv_wgrad_devscale_equals_float(S, k, bad):
    """Cout = Cin = 192 (a 64-wide tile tail), W = 70 (a pixel-chunk tail), split-K over 2 x 24 x 70 pixels, the folded
    per-channel scale and the bias gradient; bad puts an inf into dy32 (a non-finite bias gradient)"""
    N, Hh, Ww, Cin, Cout = 2, 24, 70, 192, 192
    dy32 = randn(N, Hh, Ww, Cout, seed=1)
    if bad:
        dy32[1, 3, 5, 7] = float("inf")
    dy16, x16 = dy32.half(), randn(N, Hh, Ww, Cin, seed=2).half()
    sc = randn(Cout, seed=3).abs() + 0.5
    out = []
    for gs in (S, dev_scale(S)):
        dw = torch.full((Cout, Cin, k, k), 7.0, device="cuda")
        db = torch.full((Cout,), 7.0, device="cuda")
        nf = flag()
        ops.conv_wgrad(dy16, x16, k, dw, scale=sc, grad_scale=gs, dy32=dy32, db=db, nonfinite=nf)
        out.append((dw, db, nf))
    torch.cuda.synchronize()
    for a, b in zip(*out):
        assert same_bits(a, b)
    assert int(out[0][2]) == int(bad)


@pytest.mark.parametrize("S", SCALES)
def test_conv_wgrad_acc_devscale_equals_float(S):
    """the fused RPN head's layout (rows 24, split 6, two destinations) and a 3x3 conv on a channel slice of a wider
    tensor, each accumulated over two calls"""
    Hh, Ww = 37, 45
    head32 = [randn(1, Hh, Ww, 64, seed=10 + i) for i in range(2)]
    head32[1][0, 2, 3, 4] = 1e30
    cat = randn(1, Hh, Ww, 192, seed=12).half()
    wide32 = [randn(2, 20, 70, 256, seed=13 + i) for i in range(2)]
    x = randn(2, 20, 70, 64, seed=15).half()
    out = []
    for gs in (S, dev_scale(S)):
        nf = flag()
        wc, wb = torch.zeros(6, 192, device="cuda"), torch.zeros(18, 192, device="cuda")
        bc, bb = torch.zeros(6, device="cuda"), torch.zeros(18, device="cuda")
        for i in range(2):
            ops.conv_wgrad_acc(head32[i].half(), cat, 1, wc, db=bc, dy32=head32[i], grad_scale=gs, accumulate=i > 0,
                               rows=24, split=6, dw_hi=wb, db_hi=bb, nonfinite=nf)
        wconv, bconv = torch.zeros(128, 64, 3, 3, device="cuda"), torch.zeros(128, device="cuda")
        for i in range(2):
            w16 = wide32[i].half()
            ops.conv_wgrad_acc(w16[..., 128:], x, 3, wconv, db=bconv, dy32=wide32[i][..., 128:], grad_scale=gs,
                               accumulate=i > 0, nonfinite=nf)
        out.append((wc, wb, bc, bb, wconv, bconv, nf))
    torch.cuda.synchronize()
    for a, b in zip(*out):
        assert same_bits(a, b)
    assert int(out[0][-1]) == 1                                 # 1e30 is inf in the fp16 operand


@pytest.mark.parametrize("S", SCALES)
def test_fpn_grad_combine_devscale_equals_float(S):
    """odd level sizes with the P6 scatter, an upsampled finer level, and a value that overflows fp16 at 2^12"""
    dp = randn(2, 13, 21, 256, seed=20)
    dp[0, 1, 2, 3] = 20.0
    dt = randn(2, 25, 41, 256, seed=21)
    dp6 = randn(2, 7, 11, 256, seed=22)
    a = ops.fpn_grad_combine(dp, dt=dt, dp6=dp6, scale=S)
    b = ops.fpn_grad_combine(dp, dt=dt, dp6=dp6, scale=dev_scale(S))
    torch.cuda.synchronize()
    assert same_bits(a[0], b[0]) and same_bits(a[1], b[1])
    assert bool(torch.isinf(a[1]).any()) == (S == 2.0 ** 12)


@pytest.mark.parametrize("S", SCALES)
def test_rpn_head_grad_devscale_equals_float(S):
    B, P = 2, 77
    d_cls, d_box = randn(B, 3 * P, 2, seed=30), randn(B, 3 * P, 6, seed=31)
    d_box[1, 5, 2] = 20.0
    a = ops.rpn_head_grad(d_cls, d_box, B, P, S)
    b = ops.rpn_head_grad(d_cls, d_box, B, P, dev_scale(S))
    torch.cuda.synchronize()
    assert same_bits(a[0], b[0]) and same_bits(a[1], b[1])
    assert bool(torch.isinf(a[0]).any()) == (S == 2.0 ** 12)


@pytest.mark.parametrize("S", SCALES)
@pytest.mark.parametrize("dropout", [False, True])
def test_box_tail_backward_devscale_equals_float(S, dropout):
    """R = 37, K = 300 (a 256-column tail), two classes; one RoI's class gradient overflows fp16 at 2^12"""
    R, K, nc = 37, 300, 2
    fc7 = torch.relu(randn(R, K, seed=40))
    ws = [randn(n * nc, K, seed=41 + i, scale=0.05) for i, n in enumerate((1, 6, 5))]
    d_cls, d_box, d_dim = randn(R, nc, seed=44), randn(R, 6 * nc, seed=45), randn(R, 5 * nc, seed=46)
    d_cls[3, 1] = 1000.0
    out = []
    for gs in (S, dev_scale(S)):
        grads = [torch.full((n,), 7.0, device="cuda") for n in (nc * K, nc, 6 * nc * K, 6 * nc, 5 * nc * K, 5 * nc)]
        nf = flag()
        dz16, dz32 = ops.box_tail_backward(d_cls, d_box, d_dim, fc7, *ws, grads, mask_scale=1.25 if dropout else 1.0,
                                           grad_scale=gs, nonfinite=nf)
        out.append(grads + [dz16, dz32, nf])
    torch.cuda.synchronize()
    for a, b in zip(*out):
        assert same_bits(a, b)
    assert int(out[0][-1]) == int(S == 2.0 ** 12)


@pytest.mark.parametrize("S", SCALES)
@pytest.mark.parametrize("R,G,C", [(5, 28, 256), (3, 6, 96)])
def test_kpts_tail_backward_devscale_equals_float(S, R, G, C):
    up = torch.relu(randn(R, G, G, C, seed=50)).half()
    w = randn(6, C, seed=51, scale=0.1)
    d_kp, d_l, d_r = randn(R, 4 * G, seed=52), randn(R, G, seed=53), randn(R, G, seed=54)
    d_kp[R - 1, :G] = 400.0
    out = []
    for gs in (S, dev_scale(S)):
        dw, db, db_up = torch.full((6 * C,), 7.0, device="cuda"), torch.full((6,), 7.0, device="cuda"), \
            torch.full((C,), 7.0, device="cuda")
        nf = flag()
        dup = ops.kpts_tail_backward(up, w, d_kp, d_l, d_r, dw, db, db_up, grad_scale=gs, nonfinite=nf)
        out.append((dup, dw, db, db_up, nf))
    torch.cuda.synchronize()
    for a, b in zip(*out):
        assert same_bits(a, b)
    assert int(out[0][-1]) == int(S == 2.0 ** 12)


@pytest.mark.parametrize("S", SCALES + [2.0 ** -32, 2.0 ** 32])
def test_fill_reciprocal_is_exact(S):
    t = torch.full((1001,), 7.0, device="cuda")
    ops.fill_reciprocal_(t[:1000], dev_scale(S))
    torch.cuda.synchronize()
    assert torch.equal(t[:1000].cpu(), torch.full((1000,), 1.0 / S)) and float(t[1000]) == 7.0


# ------------------------------------------------------------------------------------------------ 2. loss_gradients
def _words(shape, seed):
    w = np.random.RandomState(seed).randint(0, 2 ** 32, shape, dtype=np.uint64).astype(np.uint32)
    return torch.from_numpy(w.view(np.int32)).cuda()


def batch(seed=7, B=1):
    pairs = [synth_pair(H, W, seed + b, 12) for b in range(B)]
    iml, imr = [torch.from_numpy(np.stack([p[i] for p in pairs])).cuda().contiguous() for i in range(2)]
    gt = [torch.from_numpy(t).cuda() for t in synth_train_gt(B, 30, H, W, seed)[:5]]
    shapes = [[-(-H // s), -(-W // s)] for s in (4, 8, 16, 32, 64)]
    return (iml, imr, *gt, _words((B, 2030), seed + 2), _words((B, 512), seed + 3),
            _words((B, 3 * sum(h * w for h, w in shapes)), seed + 1)), _words((2, B * 512, 2048), seed + 4)


@pytest.mark.parametrize("B", [1, 2])
@pytest.mark.parametrize("fixed_blocks", [0, 1])
def test_loss_gradients_with_a_device_scale_equal_the_float_call(B, fixed_blocks):
    S = 2.0 ** 12
    sd = make_state_dict(3)
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    args, dw = batch(7, B)
    u = torch.full((6,), -1.0, device="cuda")
    res = []
    for gs in (S, dev_scale(S)):
        losses, g, du = TR.loss_gradients(eng, *args, dropout_words=dw, uncert=u, fixed_blocks=fixed_blocks,
                                          grad_scale=gs)
        res.append((losses.clone(), {k: v.clone() for k, v in g.items()}, du.clone(), eng.found_inf.clone()))
    torch.cuda.synchronize()
    (la, ga, dua, fa), (lb, gb, dub, fb) = res
    assert same_bits(la, lb) and same_bits(dua, dub) and same_bits(fa, fb)
    assert sorted(ga) == sorted(gb) == sorted(n for n, _ in TR.trainable_names(fixed_blocks))
    assert all(same_bits(ga[k], gb[k]) for k in ga), [k for k in ga if not same_bits(ga[k], gb[k])]
    assert int(fa) == 0


# ------------------------------------------------------------------------------------------------ 3. the update rule
def _rule(s, t, found, growth, backoff, interval):
    """sb_loss_scale_update restated: torch's rule held within [2^-32, 2^32]"""
    if found:
        return max(s * backoff, 2.0 ** -32), 0
    t += 1
    if t >= interval:
        return (s * growth if s * growth <= 2.0 ** 32 else s), 0
    return s, t


def test_loss_scale_update_matches_torch_amp_update_scale():
    rs = np.random.RandomState(0)
    seq = rs.rand(200) < 0.3
    seq[40:52] = False                                         # long enough clean runs to grow more than once
    fi, scale, tracker = flag(), dev_scale(2.0 ** 16), flag()
    ts, tt = torch.tensor([2.0 ** 16]), torch.zeros(1, dtype=torch.int32)
    grew = backed = 0
    for found in seq:
        fi.fill_(int(found))
        TR.loss_scale_update(fi, scale, tracker, 2.0, 0.5, 3)
        before = float(ts)
        torch._amp_update_scale_(ts, tt, torch.tensor([float(found)]), 2.0, 0.5, 3)
        grew += float(ts) > before
        backed += float(ts) < before
        torch.cuda.synchronize()
        assert float(scale) == float(ts) and int(tracker) == int(tt)
    assert grew > 0 and backed > 0


@pytest.mark.parametrize("start,growth,backoff,interval,found", [
    (2.0 ** 30, 4.0, 0.5, 1, [False] * 4),                     # up to 2^32, then a growth past the top is refused
    (2.0 ** 31, 2.0, 0.5, 2, [False] * 7),
    (2.0 ** 31, 4.0, 0.5, 1, [False] * 3),                     # 2^33 would pass the top: unchanged below it
    (2.0 ** -30, 2.0, 0.25, 3, [True] * 4),                    # down to the floor and held there
    (2.0 ** -31, 2.0, 0.5, 3, [True, True, False, False, False, True]),
    (2.0 ** 32, 2.0, 2.0 ** -8, 2, [True, False, False, True, False, False, False])])
def test_loss_scale_update_bounds(start, growth, backoff, interval, found):
    fi, scale, tracker = flag(), dev_scale(start), flag()
    s, t = start, 0
    for f in found:
        fi.fill_(int(f))
        TR.loss_scale_update(fi, scale, tracker, growth, backoff, interval)
        s, t = _rule(s, t, f, growth, backoff, interval)
        torch.cuda.synchronize()
        assert (float(scale), int(tracker)) == (s, t)
        assert 2.0 ** -32 <= s <= 2.0 ** 32


# ------------------------------------------------------------------------------------------------ 4-8. Trainer
def snapshot(tr):
    return [bits(v).clone() for v in tr.masters.grads] + [bits(v).clone() for v in tr.moms.grads]


def same_state(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def dynamic_trainer(sd, **kw):
    return TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, grad_scale=TR.DynamicLossScale(**kw))


def test_a_captured_step_backs_off_from_an_overflowing_scale(capsys):
    sd = make_state_dict(3)
    tr = dynamic_trainer(sd, init_scale=2.0 ** 32)
    args, dw = batch()
    init = snapshot(tr)
    with torch.no_grad():
        runner = E.GraphRunner(lambda *x: tr.step(*x, dropout_words=dw), list(args), warmup=1)
    torch.cuda.synchronize()
    # the eager warm-up step overflowed too: back to the start, so every step below is a replay
    assert int(tr.engine.found_inf) == 1 and same_state(snapshot(tr), init)
    tr.loss_scale.fill_(2.0 ** 32)
    tr.growth_tracker.zero_()
    tr.skipped.zero_()
    k = 0
    while True:
        runner()
        torch.cuda.synchronize()
        if int(tr.engine.found_inf) == 0:
            break
        k += 1
        assert int(tr.skipped) == k and float(tr.loss_scale) == 2.0 ** (32 - k) and int(tr.growth_tracker) == 0
        assert same_state(snapshot(tr), init)
        assert k < 40
    assert k >= 1 and int(tr.skipped) == k
    assert float(tr.loss_scale) == 2.0 ** (32 - k) and int(tr.growth_tracker) == 1
    # the applied step is a static trainer's first step at the scale that step used
    ref = TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, grad_scale=2.0 ** (32 - k))
    ref.step(*args, dropout_words=dw)
    torch.cuda.synchronize()
    assert int(ref.skipped) == 0
    assert same_state(snapshot(tr), snapshot(ref))
    with capsys.disabled():
        print("captured step from 2^32: %d replays skipped, first applied step at 2^%d equals a static trainer's"
              % (k, 32 - k))


def test_eager_and_replayed_dynamic_trainers_agree_over_a_growth():
    sd = make_state_dict(3)
    args, dw = batch()
    kw = dict(init_scale=2.0 ** 10, growth_interval=2)
    tra, trb = dynamic_trainer(sd, **kw), dynamic_trainer(sd, **kw)
    for _ in range(3):
        tra.step(*args, dropout_words=dw)
    with torch.no_grad():
        runner = E.GraphRunner(lambda *x: trb.step(*x, dropout_words=dw), list(args), warmup=2)   # steps 1, 2
        runner()                                                                                    # step 3
    torch.cuda.synchronize()
    assert same_state(snapshot(tra), snapshot(trb))
    for lr in (3e-4, 1e-4, 1e-4):
        tra.set_lr(lr)
        trb.set_lr(lr)
        tra.step(*args, dropout_words=dw)
        runner()
        torch.cuda.synchronize()
        assert same_state(snapshot(tra), snapshot(trb))
        assert same_bits(tra.loss_scale, trb.loss_scale) and same_bits(tra.growth_tracker, trb.growth_tracker)
    # six clean steps at interval 2: three growths
    assert int(trb.skipped) == int(tra.skipped) == 0
    assert float(trb.loss_scale) == 2.0 ** 13 and int(trb.growth_tracker) == 0


def test_checkpoint_resume_restores_the_scale():
    sd = make_state_dict(3)
    args, dw = batch()
    kw = dict(init_scale=2.0 ** 10, growth_interval=3)
    full = dynamic_trainer(sd, **kw)
    for _ in range(8):
        full.step(*args, dropout_words=dw)
    part = dynamic_trainer(sd, **kw)
    for _ in range(5):
        part.step(*args, dropout_words=dw)
    ck = part.checkpoint()
    assert float(ck["loss_scale"]) == 2.0 ** 11 and int(ck["growth_tracker"]) == 2
    resumed = dynamic_trainer(sd, **kw)
    resumed.load_checkpoint(ck)
    for _ in range(3):
        resumed.step(*args, dropout_words=dw)
    torch.cuda.synchronize()
    assert same_bits(resumed.loss_scale, full.loss_scale) and same_bits(resumed.growth_tracker, full.growth_tracker)
    assert same_state(snapshot(resumed), snapshot(full))
    static = TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, grad_scale=2.0 ** 10)
    keys = ["epoch", "lr", "model", "momentum", "sampler_state", "step", "uncert"]
    assert sorted(static.checkpoint()) == keys
    assert sorted(ck) == sorted(keys + ["growth_tracker", "loss_scale"])


DP_KW = dict(init_scale=2.0 ** 32, backoff_factor=2.0 ** -4, growth_interval=2)
DP_STEPS = 9


def _dp_worker(rank, world, port, out_dir, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    try:
        torch.cuda.set_device(0)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        sd = make_state_dict(3)
        tr = TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd,
                        grad_scale=TR.DynamicLossScale(**DP_KW), world=world, dist=dist)
        args, dw = batch(20 + rank)
        trace = []
        for _ in range(DP_STEPS):
            tr.step(*args, dropout_words=dw)
            trace.append((float(tr.loss_scale), int(tr.growth_tracker), int(tr.skipped)))
        torch.cuda.synchronize()
        torch.save({"masters": [b.cpu() for b in tr.masters.buckets], "trace": trace},
                   os.path.join(out_dir, "rank%d.pt" % rank))
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except Exception as e:             # reported to the parent
        q.put((rank, "%s: %s" % (type(e).__name__, e)))


def test_two_ranks_hold_one_scale_and_equal_one_process(tmp_path, capsys):
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
    assert r0["trace"] == r1["trace"]
    assert all(same_bits(a, b) for a, b in zip(r0["masters"], r1["masters"]))
    # one process: each rank's gradients at the shared scale, the flags reduced as the step's MAX all-reduce does,
    # the gradients averaged as the bucket all-reduce does, then the step and the scale update on the reduced flag
    sd = make_state_dict(3)
    eng = E.StereoRCNNEngine(sd, "cuda", precision="fp16")
    tr = TR.Trainer(eng, sd, grad_scale=TR.DynamicLossScale(**DP_KW))
    data = [batch(20 + r) for r in range(2)]
    trace = []
    for _ in range(DP_STEPS):
        parts, flags = [], []
        for args, dw in data:
            _, g, du = TR.loss_gradients(eng, *args, dropout_words=dw, uncert=tr.uncert, grad_scale=tr.loss_scale)
            parts.append([g[n].clone() for n in tr.names] + [du.clone()])
            flags.append(eng.found_inf.clone())
        with torch.no_grad():
            for v, a, b in zip(tr.grads.grads, *parts):
                v.copy_((a + b) / 2)
            eng.found_inf.copy_(torch.maximum(*flags))
        TR.clip_gradient(tr.grads.grads[:-1], 10.0, out=tr.norm)
        tr._sgd(tr.lr, tr.momentum, eng.found_inf, tr.skipped)
        eng.refresh_weights(tr.params)
        d = tr.dynamic
        TR.loss_scale_update(eng.found_inf, tr.loss_scale, tr.growth_tracker, d.growth_factor, d.backoff_factor,
                             d.growth_interval)
        trace.append((float(tr.loss_scale), int(tr.growth_tracker), int(tr.skipped)))
    torch.cuda.synchronize()
    assert trace == r0["trace"]
    assert all(same_bits(a, b.cpu()) for a, b in zip(r0["masters"], tr.masters.buckets))
    skipped = trace[-1][2]
    assert 1 <= skipped < DP_STEPS
    with capsys.disabled():
        print("two ranks from 2^32: (scale, tracker, skipped) per step %s" % trace)


# ------------------------------------------------------------------------------------------------ fit's log
FH, FW = 100, 160


def _frame(seed):
    rs = np.random.RandomState(seed)
    base = rs.randint(0, 256, (FH // 8 + 2, FW // 8 + 2, 3)).astype(np.float32)
    im = np.kron(base, np.ones((8, 8, 1), np.float32))[:FH, :FW] + rs.randn(FH, FW, 3) * 6
    return np.clip(im, 0, 255).astype(np.uint8)


def _roidb():
    rs = np.random.RandomState(0)
    f = np.float32
    out = []
    for i in range(2):
        n = 3 + i
        w, h = rs.uniform(0.1 * FW, 0.35 * FW, n), rs.uniform(0.12 * FH, 0.4 * FH, n)
        x1, y1 = rs.uniform(6, FW - w - 1), rs.uniform(0, FH - h - 1)
        bl = np.stack([x1, y1, x1 + w, y1 + h], 1).astype(f)
        br = bl.copy()
        br[:, [0, 2]] -= f(4)
        bm = np.stack([br[:, 0], bl[:, 1], bl[:, 2], bl[:, 3]], 1).astype(f)
        kp = np.full((n, 6), -1, f)
        kp[np.arange(n), rs.randint(0, 4, n)] = rs.uniform(x1, x1 + w)
        kp[:, 4], kp[:, 5] = rs.uniform(x1, x1 + 0.3 * w), rs.uniform(x1 + 0.7 * w, x1 + w)
        do = np.stack([rs.uniform(1.3, 1.8, n), rs.uniform(1.4, 1.9, n), rs.uniform(3.2, 4.6, n),
                       rs.uniform(-3.1, 3.1, n)], 1).astype(f)
        out.append(dict(boxes_left=bl, boxes_right=br, boxes_merge=bm, dim_orien=do, kpts=kp,
                        kpts_right=np.where(kp >= 0, kp - f(4), kp).astype(f), gt_classes=np.ones(n, np.int32),
                        flipped=False, index=i))
    return TR.append_flipped(out, [FW] * 2)


@pytest.mark.parametrize("dynamic", [False, True])
def test_fit_logs_the_scale_of_a_dynamic_trainer(dynamic):
    import re
    sd = make_state_dict(3)
    gs = TR.DynamicLossScale(init_scale=2.0 ** 32, backoff_factor=2.0 ** -8) if dynamic else 2.0 ** 12
    tr = TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, grad_scale=gs, seed=5)
    lines = []
    db = _roidb()
    TR.fit(tr, db, lambda e: (_frame(100 + e["index"]), _frame(200 + e["index"])), epochs=1, log=lines.append,
           target_size=160, max_rows=16)
    head = [l for l in lines if l.startswith("[epoch")]
    scale = [l for l in lines if "loss scale" in l]
    assert len(head) == len(db) == 4
    if not dynamic:
        assert scale == [] and len(lines) == 2 * len(db)
        return
    assert len(scale) == len(db) and len(lines) == 3 * len(db)
    line = "\t\t\tloss scale: %g, skipped steps: %d"
    # 2^32 overflows; every step that overflows divides the scale by 2^8 and counts itself
    skipped = [int(re.fullmatch(r"\t\t\tloss scale: \S+, skipped steps: (\d+)", l).group(1)) for l in scale]
    assert skipped[0] == 1 and skipped == sorted(skipped)
    assert scale == [line % (2.0 ** (32 - 8 * k), k) for k in skipped]
    assert scale[-1] == line % (float(tr.loss_scale), int(tr.skipped))
