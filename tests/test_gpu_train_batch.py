"""GPU: training at several stereo pairs per step and on several ranks -- sb_prep_stereo_pairs bit for bit against B
launches of sb_prep_stereo_pair, Trainer.step_from_frames on a two-pair StepInputs against Trainer.step on
oracle-prepared inputs, eager against graph-replayed, train.fit(batch_size=2) on one rank with its checkpoints and
resume, and on two ranks over gloo against a one-process emulation of the averaged step (and over NCCL where two GPUs
are visible)."""
import os
import re
import socket

import numpy as np
import pytest
import torch

from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import ops
from stereo_rcnn_b200 import train as TR
from stereo_rcnn_b200.synth import make_state_dict

pytestmark = pytest.mark.gpu

ROW_KEYS = ("boxes_left", "boxes_right", "boxes_merge", "dim_orien", "kpts")
# -> 160x256 and 160x258 blobs at target size 160; the trunk makes P2 of the latter 64 wide, not ceil(258 / 4) = 65
SHAPE_A, SHAPE_B = (100, 160), (100, 161)
TARGET = 160
GS = 2.0 ** 12
SEED = 5
ROWS = 16


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def frame(h, w, seed):
    rs = np.random.RandomState(seed)
    base = rs.randint(0, 256, (h // 8 + 2, w // 8 + 2, 3)).astype(np.float32)
    im = np.kron(base, np.ones((8, 8, 1), np.float32))[:h, :w] + rs.randn(h, w, 3) * 6
    return np.clip(im, 0, 255).astype(np.uint8)


def synth_entries(hw, n_base, n_flip, first_index, seed):
    """n_base entries of an hw frame with the reference's keys and kitti_data's height / width, entry 1 with a class-0
    row, then the flips of the first n_flip of them"""
    FH, FW = hw
    rs = np.random.RandomState(seed)
    f = np.float32
    out = []
    for i in range(n_base):
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
        cls = np.ones(n, np.int32)
        if i == 1:
            cls[1] = 0
        out.append(dict(boxes_left=bl, boxes_right=br, boxes_merge=bm, dim_orien=do, kpts=kp,
                        kpts_right=np.where(kp >= 0, kp - f(4), kp).astype(f), gt_classes=cls, flipped=False,
                        index=first_index + i, height=FH, width=FW))
    return TR.append_flipped(out, [FW] * n_base)[:n_base + n_flip]


def two_shape_roidb():
    """shape A: 3 entries and their flips (3 batches of 2); shape B: 3 entries and 2 flips (2 batches, one dropped)"""
    return synth_entries(SHAPE_A, 3, 3, 0, 0) + synth_entries(SHAPE_B, 3, 2, 10, 1)


def frames_of(e):
    return frame(e["height"], e["width"], 100 + e["index"]), frame(e["height"], e["width"], 200 + e["index"])


def new_trainer(sd=None, world=1, dist=None):
    sd = sd or make_state_dict(3)
    return TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, grad_scale=GS, seed=SEED, world=world,
                      dist=dist)


def state(tr):
    return [bits(v).clone() for v in tr.masters.grads] + [bits(v).clone() for v in tr.moms.grads]


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


# -------------------------------------------------------------------------------------------- sb_prep_stereo_pairs
@pytest.mark.parametrize("B", [1, 2, 5])
@pytest.mark.parametrize("h,w,scale", [(37, 300, 1.6), (33, 161, 600.0 / 370.0)])
@pytest.mark.parametrize("rgb", [False, True])
def test_prep_stereo_pairs_equal_one_launch_per_pair(B, h, w, scale, rgb):
    lib = L.load()
    left = torch.from_numpy(np.stack([frame(h, w, 10 + b) for b in range(B)])).cuda()
    right = torch.from_numpy(np.stack([frame(h, w, 20 + b) for b in range(B)])).cuda()
    flips = [(0, 1, 7, 0, 1)[b] for b in range(B)] if B > 1 else [1]
    flip = torch.tensor(flips, dtype=torch.int32, device="cuda")
    Ho, Wo = ops.prep_image_size(h, w, scale)
    assert Wo % 256 != 0
    n, guard = B * 3 * Ho * Wo, 1024
    buf = torch.full((2 * n + 3 * guard,), -12345.0, device="cuda")
    out = (buf[guard:guard + n].view(B, 3, Ho, Wo), buf[2 * guard + n:2 * guard + 2 * n].view(B, 3, Ho, Wo))
    ops.prep_stereo_pair(left, right, scale, flip, rgb, out=out)
    want = [torch.empty(B, 3, Ho, Wo, device="cuda") for _ in range(2)]
    for b in range(B):
        L.check(lib.sb_prep_stereo_pair(L.ptr(left[b]), L.ptr(right[b]), h, w, scale, int(rgb), L.ptr(flip[b:b + 1]),
                                        L.ptr(want[0][b]), L.ptr(want[1][b]), L.stream_ptr()), "sb_prep_stereo_pair")
    torch.cuda.synchronize()
    assert torch.equal(bits(out[0]), bits(want[0])) and torch.equal(bits(out[1]), bits(want[1]))
    for a, b in ((0, guard), (guard + n, 2 * guard + n), (2 * guard + 2 * n, 3 * guard + 2 * n)):
        assert bool((buf[a:b] == -12345.0).all())


# ------------------------------------------------------------------------------------- step_from_frames at B = 2
def oracle_inputs(batch, step, rank, inp):
    """blobs, ground truth and words of one step from oracle/train_input.py, as device tensors"""
    from oracle import train_input as TI
    cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    n_ids = len(inp.word_tensors)
    words = [TI.random_words(SEED, step, n_ids * rank + sid, t.numel()).reshape(t.shape)
             for sid, t in enumerate(inp.word_tensors)]
    bl, br, gts = [], [], []
    for b, e in enumerate(batch):
        left, right = frames_of(e)
        pl, pr = TI.pair_blobs(left[:, :, ::-1], right[:, :, ::-1], inp.scale, e["flipped"])
        bl.append(pl)
        br.append(pr)
        n = len(e["gt_classes"])
        pad = {k: np.concatenate([e[k], np.zeros((ROWS - n,) + e[k].shape[1:], e[k].dtype)]) for k in
               ROW_KEYS + ("gt_classes",)}
        gts.append(TI.train_gt(pad, inp.scale, pl.shape[2], words[0][b], n))
    gt = [cu(np.stack([g[i] for g in gts])) for i in range(5)]
    return cu(np.stack(bl)), cu(np.stack(br)), gt, [cu(w) for w in words], [g[5] for g in gts]


def test_two_pair_step_from_frames_equals_step_on_oracle_prepared_inputs():
    db = synth_entries(SHAPE_A, 3, 3, 0, 0)
    tra, trb = new_trainer(), new_trainer()
    inp = TR.StepInputs(SHAPE_A, TARGET / min(SHAPE_A), "cuda", batch=2, max_rows=ROWS)
    assert inp.im_left.shape == (2, 3, 160, 256) and inp.dropout_words.shape == (2, 2 * 512, 2048)
    assert inp.rpn_keys.shape == (2, 3 * sum(h * w for h, w in ((40, 64), (20, 32), (10, 16), (5, 8), (3, 4))))
    assert TR.StepInputs(SHAPE_B, TARGET / min(SHAPE_B), "cuda").rpn_keys.shape == \
        (1, 3 * sum(h * w for h, w in ((40, 64), (20, 32), (10, 16), (5, 8), (3, 4))))
    # an unflipped entry with a class-0 row beside a flipped one, then the flip of the first beside an unflipped one
    for step, batch in enumerate(([db[1], db[3]], [db[4], db[0]])):
        inp.load(batch, [frames_of(e) for e in batch])
        la, total_a, _, _ = tra.step_from_frames(inp)
        la, total_a = la.clone(), total_a.clone()
        bl, br, gt, words, nb = oracle_inputs(batch, step, 0, inp)
        assert nb == [int((e["gt_classes"] != 0).sum()) for e in batch] == inp.gt[5].tolist()
        lb, total_b, _, _ = trb.step(bl, br, *gt, words[1], words[2], words[3], dropout_words=words[4])
        torch.cuda.synchronize()
        assert torch.equal(bits(inp.im_left), bits(bl)) and torch.equal(bits(inp.im_right), bits(br)), step
        assert torch.equal(bits(la), bits(lb)) and torch.equal(bits(total_a), bits(total_b)), step
        assert all(torch.equal(x, y) for x, y in zip(state(tra), state(trb))), step
    assert int(tra.step_count.item()) == 2 and int(tra.skipped.item()) == 0


def test_two_pair_graph_replayed_steps_equal_eager_ones():
    db = synth_entries(SHAPE_A, 3, 3, 0, 0)
    seq = [[db[0], db[4]], [db[0], db[4]], [db[3], db[1]], [db[2], db[5]]]   # one graph, any mix of flips
    tra, trb = new_trainer(), new_trainer()
    ia, ib = (TR.StepInputs(SHAPE_A, TARGET / min(SHAPE_A), "cuda", batch=2, max_rows=ROWS) for _ in range(2))
    for batch in seq:
        ia.load(batch, [frames_of(e) for e in batch])
        tra.step_from_frames(ia)
    drawn = []
    with torch.no_grad():
        ib.load(seq[0], [frames_of(e) for e in seq[0]])
        runner = E.GraphRunner(lambda: trb.step_from_frames(ib), [], warmup=2)            # steps 1, 2
        for batch in seq[2:]:                                                              # steps 3, 4
            ib.load(batch, [frames_of(e) for e in batch])
            ib.ready()
            runner()
            ib.release()
            drawn.append([t.clone() for t in ib.word_tensors] + [runner.outputs[0].clone()])
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(state(tra), state(trb)))
    assert int(tra.step_count.item()) == 4 == int(trb.step_count.item()) and int(trb.skipped.item()) == 0
    assert all(not torch.equal(x, y) for x, y in zip(drawn[0], drawn[1]))


# ----------------------------------------------------------------------------------------- fit at 2 pairs, 1 rank
def test_fit_at_two_pairs_trains_saves_and_resumes(tmp_path, capsys):
    db = two_shape_roidb()
    assert len(db) == 11
    sd = make_state_dict(3)
    lines = []
    tr = new_trainer(sd)
    totals = TR.fit(tr, db, frames_of, epochs=3, save_dir=str(tmp_path), log=lines.append, target_size=TARGET,
                    max_rows=ROWS, batch_size=2)
    with capsys.disabled():
        print("fit, 3 epochs of 5 batches of 2 pairs, total loss: %s" % " ".join("%.4f" % t for t in totals))
    assert len(totals) == 15 and all(np.isfinite(totals)) and int(tr.skipped.item()) == 0
    assert int(tr.step_count.item()) == 15 and tr.epoch == 4
    head = [l for l in lines if l.startswith("[epoch")]
    assert len(head) == 15 and len([l for l in lines if l.startswith("save model: ")]) == 3
    for k, l in enumerate(head):
        assert re.fullmatch(r"\[epoch  %d\]\[iter    %d/   5\] loss: -?\d+\.\d{4}, lr: 1\.00e-03" % (k // 5 + 1, k % 5), l), l
    assert len([l for l in lines if l.startswith("\t\t\trpn_cls: ")]) == 15
    files = ["stereo_rcnn_%d_4.pth" % e for e in (1, 2, 3)]
    assert sorted(f for f in os.listdir(tmp_path) if f.endswith(".pth")) == files
    cks = [torch.load(tmp_path / f) for f in files]
    assert [c["epoch"] for c in cks] == [2, 3, 4] and [c["step"] for c in cks] == [5, 10, 15]
    assert np.mean(totals[10:]) < np.mean(totals[:5])
    tr2 = new_trainer(sd)
    tr2.load_checkpoint(cks[0])
    os.makedirs(tmp_path / "resumed")
    TR.fit(tr2, db, frames_of, epochs=3, start_epoch=cks[0]["epoch"], save_dir=str(tmp_path / "resumed"),
           log=lambda s: None, target_size=TARGET, max_rows=ROWS, batch_size=2)
    for f, ref in zip(files[1:], cks[1:]):
        got = torch.load(tmp_path / "resumed" / f)
        assert got["epoch"] == ref["epoch"] and got["step"] == ref["step"] and got["lr"] == ref["lr"]
        assert torch.equal(bits(got["uncert"]), bits(ref["uncert"]))
        assert all(torch.equal(bits(got["momentum"][k]), bits(ref["momentum"][k])) for k in ref["momentum"])
        assert all(torch.equal(got["model"][k], ref["model"][k]) for k in ref["model"])


# ---------------------------------------------------------------------------------------- fit at 2 pairs, 2 ranks
def _fit_worker(rank, world, port, backend, out_dir, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    try:
        torch.cuda.set_device(0 if backend == "gloo" else rank)
        dist.init_process_group(backend, rank=rank, world_size=world)
        db = two_shape_roidb()
        sd = make_state_dict(3)
        tr = new_trainer(sd, world, dist)
        assert tr.rank == rank
        ckdir = os.path.join(out_dir, "ck")
        os.makedirs(ckdir, exist_ok=True)
        masters, lines = [], []
        for epoch in (1, 2, 3):                  # one epoch per call: fit continues from the trainer's sampler state
            TR.fit(tr, db, frames_of, epochs=epoch, start_epoch=epoch, save_dir=ckdir, log=lines.append,
                   target_size=TARGET, max_rows=ROWS, batch_size=2)
            torch.cuda.synchronize()
            masters.append([b.cpu() for b in tr.masters.buckets])
        dist.barrier()
        # resume on every rank from the first checkpoint, which rank 0 alone wrote
        tr2 = new_trainer(sd, world, dist)
        tr2.load_checkpoint(torch.load(os.path.join(ckdir, "stereo_rcnn_1_1.pth")))
        resdir = os.path.join(out_dir, "resumed")
        os.makedirs(resdir, exist_ok=True)
        TR.fit(tr2, db, frames_of, epochs=3, start_epoch=2, save_dir=resdir, log=lambda s: None,
               target_size=TARGET, max_rows=ROWS, batch_size=2)
        torch.cuda.synchronize()
        torch.save({"masters": masters, "lines": lines, "step": int(tr.step_count.item()),
                    "skipped": int(tr.skipped.item())}, os.path.join(out_dir, "rank%d.pt" % rank))
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except Exception as e:             # reported to the parent
        import traceback
        q.put((rank, "%s: %s\n%s" % (type(e).__name__, e, traceback.format_exc())))


def _run_ranks(world, backend, out_dir):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_fit_worker, args=(r, world, port, backend, out_dir, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=1200) for _ in range(world))
    for p in procs:
        p.join(timeout=120)
    assert res == [(r, "ok") for r in range(world)], res
    return [torch.load(os.path.join(out_dir, "rank%d.pt" % r)) for r in range(world)]


def emulate(db, epochs, world):
    """one process: per step, loss_gradients on each rank's batch with that rank's words, the gradients averaged as
    the bucket all-reduce does (sum over ranks, then / world), clip_gradient and SGD -> the master buckets per epoch"""
    sd = make_state_dict(3)
    tr = new_trainer(sd)
    eng = tr.engine
    gen = torch.Generator().manual_seed(SEED)
    scale = {hw: TARGET / min(hw) for hw in (SHAPE_A, SHAPE_B)}
    inps = {hw: TR.StepInputs(hw, scale[hw], "cuda", batch=2, max_rows=ROWS) for hw in scale}
    out, step = [], 0
    for _epoch in range(epochs):
        state_ = gen.get_state()
        per_rank = []
        for r in range(world):
            gen.set_state(state_)
            per_rank.append(TR.epoch_batches(db, 2, gen, r, world))
        for k in range(len(per_rank[0])):
            parts = []
            for r in range(world):
                batch = [db[i] for i in per_rank[r][k]]
                inp = inps[(batch[0]["height"], batch[0]["width"])]
                bl, br, gt, words, _nb = oracle_inputs(batch, step, r, inp)
                _, g, du = TR.loss_gradients(eng, bl, br, *gt, words[1], words[2], words[3], dropout_words=words[4],
                                             uncert=tr.uncert, grad_scale=GS)
                parts.append([g[n].clone() for n in tr.names] + [du.clone()])
                assert int(eng.found_inf.item()) == 0
            with torch.no_grad():
                for i, v in enumerate(tr.grads.grads):
                    acc = parts[0][i].clone()
                    for p in parts[1:]:
                        acc += p[i]
                    v.copy_(acc / world)
            TR.clip_gradient(tr.grads.grads[:-1], 10.0, out=tr.norm)
            tr._sgd(tr.lr, tr.momentum, eng.found_inf, tr.skipped)
            eng.refresh_weights(tr.params)
            step += 1
        torch.cuda.synchronize()
        out.append([b.cpu() for b in tr.masters.buckets])
    return out


def test_fit_on_two_ranks_over_gloo_equals_one_process_emulation(tmp_path):
    r0, r1 = _run_ranks(2, "gloo", str(tmp_path))
    for e in range(3):
        assert all(torch.equal(bits(a), bits(b)) for a, b in zip(r0["masters"][e], r1["masters"][e])), e
    assert r0["step"] == r1["step"] == 6 and r0["skipped"] == r1["skipped"] == 0
    # rank 0 logs two lines per step (5 batches over 2 ranks: 2 steps per epoch) and a save line per epoch
    head = [l for l in r0["lines"] if l.startswith("[epoch")]
    assert len(head) == 6 and all("/   2] loss: " in l for l in head) and r1["lines"] == []
    files = ["stereo_rcnn_%d_1.pth" % e for e in (1, 2, 3)]
    assert sorted(os.listdir(tmp_path / "ck")) == files
    cks = [torch.load(tmp_path / "ck" / f) for f in files]
    assert [c["epoch"] for c in cks] == [2, 3, 4] and [c["step"] for c in cks] == [2, 4, 6]
    # the resumed run's later checkpoints, bit for bit
    assert sorted(os.listdir(tmp_path / "resumed")) == files[1:]
    for f, ref in zip(files[1:], cks[1:]):
        got = torch.load(tmp_path / "resumed" / f)
        assert got["epoch"] == ref["epoch"] and got["step"] == ref["step"]
        assert all(torch.equal(bits(got["momentum"][k]), bits(ref["momentum"][k])) for k in ref["momentum"])
        assert all(torch.equal(got["model"][k], ref["model"][k]) for k in ref["model"])
    want = emulate(two_shape_roidb(), 3, 2)
    for e in range(3):
        assert all(torch.equal(bits(a), bits(b)) for a, b in zip(r0["masters"][e], want[e])), e


def test_fit_on_two_gpus_over_nccl_keeps_the_ranks_identical(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    r0, r1 = _run_ranks(2, "nccl", str(tmp_path))
    for e in range(3):
        assert all(torch.equal(bits(a), bits(b)) for a, b in zip(r0["masters"][e], r1["masters"][e])), e
    assert r0["step"] == 6 and r0["skipped"] == 0
