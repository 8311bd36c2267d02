"""GPU: the training side of the input pipeline -- sb_prep_stereo_pair bit for bit against sb_prep_image on host-flipped
frames, sb_train_gt bit for bit against oracle/train_input.py and the reference golden, sb_random_words against the
numpy Philox4x32-10, Trainer.step_from_frames against Trainer.step on oracle-prepared inputs, eager against
graph-replayed, resume in a second process, and train.fit with its checkpoints."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:                                   # the resume worker runs this file as a script
    sys.path.insert(0, ROOT)

from stereo_rcnn_b200 import engine as E  # noqa: E402
from stereo_rcnn_b200 import ops  # noqa: E402
from stereo_rcnn_b200 import train as TR  # noqa: E402
from stereo_rcnn_b200.synth import make_state_dict  # noqa: E402

pytestmark = pytest.mark.gpu

GOLD = os.path.join(ROOT, "tests", "golden", "train_batch.npz")
ROW_KEYS = ("boxes_left", "boxes_right", "boxes_merge", "dim_orien", "kpts")
GT_KEYS = ("gt_left", "gt_right", "gt_merge", "gt_dim_orien", "gt_kpts")
FH, FW, SCALE = 100, 160, 1.6                              # frames -> the 160x256 blobs of the other train tests
GS = 2.0 ** 12
SEED = 5


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def frame(h, w, seed):
    rs = np.random.RandomState(seed)
    base = rs.randint(0, 256, (h // 8 + 2, w // 8 + 2, 3)).astype(np.float32)
    im = np.kron(base, np.ones((8, 8, 1), np.float32))[:h, :w] + rs.randn(h, w, 3) * 6
    return np.clip(im, 0, 255).astype(np.uint8)


# --------------------------------------------------------------------------------------------- sb_prep_stereo_pair
@pytest.mark.parametrize("h,w,scale", [(20, 63, 1.6), (37, 300, 1.6), (33, 161, 600.0 / 370.0), (375, 1242, 1.6)])
@pytest.mark.parametrize("rgb", [False, True])
def test_prep_stereo_pair_equals_prep_image_on_host_flipped_frames(h, w, scale, rgb):
    left, right = frame(h, w, 1), frame(h, w, 2)
    dl, dr = torch.from_numpy(left).cuda(), torch.from_numpy(right).cuda()
    ref = {0: (ops.prep_image(dl, scale, rgb), ops.prep_image(dr, scale, rgb)),
           1: (ops.prep_image(torch.from_numpy(right[:, ::-1].copy()).cuda(), scale, rgb),
               ops.prep_image(torch.from_numpy(left[:, ::-1].copy()).cuda(), scale, rgb))}
    _, Ho, Wo = ref[0][0].shape
    assert Wo % 256 != 0
    n, guard = 3 * Ho * Wo, 1024
    for flip in (0, 1, 7):
        buf = torch.full((2 * n + 3 * guard,), -12345.0, device="cuda")
        out = (buf[guard:guard + n].view(3, Ho, Wo), buf[2 * guard + n:2 * guard + 2 * n].view(3, Ho, Wo))
        ops.prep_stereo_pair(dl, dr, scale, torch.tensor([flip], dtype=torch.int32, device="cuda"), rgb, out=out)
        torch.cuda.synchronize()
        want = ref[1 if flip else 0]
        assert torch.equal(bits(out[0]), bits(want[0])) and torch.equal(bits(out[1]), bits(want[1])), flip
        for a, b in ((0, guard), (guard + n, 2 * guard + n), (2 * guard + 2 * n, 3 * guard + 2 * n)):
            assert bool((buf[a:b] == -12345.0).all())


# ----------------------------------------------------------------------------------------------------- sb_train_gt
def run_train_gt(entries, ns, words, scale, width):
    """entries: dicts of [N, .] arrays -> the six outputs as numpy, with guard rows checked"""
    B, N = len(entries), len(entries[0]["gt_classes"])
    rows = {k: torch.from_numpy(np.stack([np.asarray(e[k], np.float32) for e in entries])).cuda() for k in ROW_KEYS}
    rows["gt_classes"] = torch.from_numpy(np.stack([np.asarray(e["gt_classes"], np.int32) for e in entries])).cuda()
    n_rows = torch.tensor(ns, dtype=torch.int32, device="cuda")
    w = torch.from_numpy(np.stack(words).astype(np.uint32).view(np.int32)).cuda()
    bufs = [torch.full((B + 2, 30, c), -7.0, device="cuda") for c in (5, 5, 5, 5, 6)]
    nb = torch.full((B + 2,), -7, dtype=torch.int32, device="cuda")
    TR.train_gt(rows, n_rows, w, scale, width, out=tuple(b[1:B + 1] for b in bufs) + (nb[1:B + 1],))
    torch.cuda.synchronize()
    for b in bufs + [nb]:
        assert bool((b[0] == -7).all()) and bool((b[B + 1] == -7).all())
    return [b[1:B + 1].cpu().numpy() for b in bufs] + [nb[1:B + 1].cpu().numpy()]


def gold_entry(g, i):
    return {k: g[k][i] for k in ROW_KEYS + ("gt_classes",)}


def test_train_gt_equals_the_reference_golden():
    from oracle import train_input as TI
    g = dict(np.load(GOLD))
    for i in range(12):                                   # every golden entry, alone
        out = run_train_gt([gold_entry(g, i)], [int(g["n_rows"][i])], [g["words"][i]], float(g["scale"]), 101)
        for k, o in zip(GT_KEYS, out[:5]):
            assert np.array_equal(o[0].view(np.int32), g[k][i].view(np.int32)), (i, k)
        assert out[5][0] == g["num_boxes"][i]
    # B = 2 (the 38-row entry and the edge entry's flip), then all twelve in one launch
    for sel in ([1, 8], list(range(12))):
        out = run_train_gt([gold_entry(g, i) for i in sel], [int(g["n_rows"][i]) for i in sel],
                           [g["words"][i] for i in sel], float(g["scale"]), 101)
        for k, o in zip(GT_KEYS, out[:5]):
            assert np.array_equal(o.view(np.int32), g[k][sel].view(np.int32)), k
        assert np.array_equal(out[5], g["num_boxes"][sel])
    # row counts 0, 1, 30, 31, N and above N (clamped), with random and with tied words, against the oracle
    e = gold_entry(g, 1)
    rs = np.random.RandomState(3)
    for n in (0, 1, 30, 31, 40, 41, 1000, -3):
        for words in (rs.randint(0, 2 ** 32, 40, dtype=np.uint64).astype(np.uint32),
                      rs.randint(0, 3, 40).astype(np.uint32), np.zeros(40, np.uint32)):
            out = run_train_gt([e], [n], [words], 1.6, 101)
            ref = TI.train_gt(e, 1.6, 101, words, n)
            for k, o, r in zip(GT_KEYS, out[:5], ref[:5]):
                assert np.array_equal(o[0].view(np.int32), r.view(np.int32)), (n, k)
            assert out[5][0] == ref[5]
    # the capacity limit of the kernel
    big = {k: np.tile(v, (26,) + (1,) * (v.ndim - 1))[:1024] for k, v in e.items()}
    words = rs.randint(0, 2 ** 32, 1024, dtype=np.uint64).astype(np.uint32)
    out = run_train_gt([big], [1024], [words], 1.6, 101)
    ref = TI.train_gt(big, 1.6, 101, words, 1024)
    assert all(np.array_equal(o[0].view(np.int32), r.view(np.int32)) for o, r in zip(out[:5], ref[:5]))


# ------------------------------------------------------------------------------------------------- sb_random_words
def test_random_words_equal_the_numpy_philox():
    from oracle import train_input as TI
    step = torch.tensor([(3 << 32) + 9], dtype=torch.int64, device="cuda")
    seed = 0xFEDCBA9876543210
    A = 3 * sum(-(-600 // s) * -(-1987 // s) for s in (4, 8, 16, 32, 64))
    seen = {}
    for sid, n in enumerate((1, 7, 4, 2030, 512, A, 2 * 512 * 2048)):
        buf = torch.full((n + 9,), 77, dtype=torch.int32, device="cuda")
        for off in (4, 5):                                 # 16-byte aligned and not
            buf.fill_(77)
            TR.fill_random_words(buf[off:off + n], seed, step, sid)
            torch.cuda.synchronize()
            got = buf.cpu().numpy()
            assert (got[:off] == 77).all() and (got[off + n:] == 77).all()
            assert np.array_equal(got[off:off + n], TI.random_words(seed, (3 << 32) + 9, sid, n)), (n, off)
        seen[sid] = got[off:off + n]
    w = lambda sd, st, sid: TI.random_words(sd, st, sid, 512)
    assert not np.array_equal(seen[3][:512], seen[4]) and not np.array_equal(w(1, 0, 0), w(1, 1, 0))
    out = torch.zeros(2, 512, dtype=torch.int32, device="cuda")
    TR.fill_random_words(out[0], 1, step, 2)
    TR.step_advance(step)
    TR.fill_random_words(out[1], 1, step, 2)
    assert int(step.item()) == (3 << 32) + 10 and not torch.equal(out[0], out[1])
    assert np.array_equal(out[1].cpu().numpy(), TI.random_words(1, (3 << 32) + 10, 2, 512))
    step.fill_((3 << 32) + 9)
    TR.fill_random_words(out[1], 1, step, 2)
    assert torch.equal(out[0], out[1])


# ------------------------------------------------------------------------------------------------ step_from_frames
def synth_roidb(n_entries=3, seed=0):
    """roidb entries in the coordinates of a FH x FW frame, the reference's keys, plus their flips"""
    rs = np.random.RandomState(seed)
    f = np.float32
    out = []
    for i in range(n_entries):
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
                        kpts_right=np.where(kp >= 0, kp - f(4), kp).astype(f), gt_classes=cls, flipped=False, index=i))
    return TR.append_flipped(out, [FW] * n_entries)


def frames_of(entry):
    return frame(FH, FW, 100 + entry["index"]), frame(FH, FW, 200 + entry["index"])


def new_trainer(sd=None):
    sd = sd or make_state_dict(3)
    return TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, grad_scale=GS, seed=SEED)


def state(tr):
    return [bits(v).clone() for v in tr.masters.grads] + [bits(v).clone() for v in tr.moms.grads]


def test_step_from_frames_equals_step_on_oracle_prepared_inputs():
    from oracle import train_input as TI
    roidb = synth_roidb()
    tra, trb = new_trainer(), new_trainer()
    inp = TR.StepInputs((FH, FW), SCALE, "cuda", max_rows=16)
    for step, e in enumerate((roidb[1], roidb[4])):       # an unflipped entry with a class-0 row, then a flipped one
        left, right = frames_of(e)
        inp.load(e, left, right)
        la, total_a, _, _ = tra.step_from_frames(inp)
        la, total_a = la.clone(), total_a.clone()
        bl, br = TI.pair_blobs(left[:, :, ::-1], right[:, :, ::-1], SCALE, e["flipped"])
        n = len(e["gt_classes"])
        pad = {k: np.concatenate([e[k], np.zeros((16 - n,) + e[k].shape[1:], e[k].dtype)]) for k in
               ROW_KEYS + ("gt_classes",)}
        words = [TI.random_words(SEED, step, sid, t.numel()).reshape(t.shape) for sid, t in enumerate(inp.word_tensors)]
        gt = TI.train_gt(pad, SCALE, bl.shape[2], words[0][0], n)
        assert gt[5] == int((e["gt_classes"] != 0).sum()) and int(inp.gt[5][0]) == gt[5]
        cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        lb, total_b, _, _ = trb.step(cu(bl)[None], cu(br)[None], *[cu(x)[None] for x in gt[:5]], cu(words[1]),
                                     cu(words[2]), cu(words[3]), dropout_words=cu(words[4]))
        torch.cuda.synchronize()
        assert torch.equal(bits(la), bits(lb)) and torch.equal(bits(total_a), bits(total_b)), step
        assert all(torch.equal(x, y) for x, y in zip(state(tra), state(trb))), step
    assert int(tra.step_count.item()) == 2 and int(tra.skipped.item()) == 0


def test_eager_and_graph_replayed_steps_from_frames_agree():
    roidb = synth_roidb()
    seq = [roidb[0], roidb[0], roidb[3], roidb[2]]        # one captured graph serves flipped and unflipped entries
    tra, trb = new_trainer(), new_trainer()
    ia, ib = (TR.StepInputs((FH, FW), SCALE, "cuda", max_rows=16) for _ in range(2))
    for e in seq:
        ia.load(e, *frames_of(e))
        tra.step_from_frames(ia)
    drawn = []
    with torch.no_grad():
        ib.load(seq[0], *frames_of(seq[0]))
        runner = E.GraphRunner(lambda: trb.step_from_frames(ib), [], warmup=2)            # steps 1, 2
        for e in seq[2:]:                                                                  # steps 3, 4
            ib.load(e, *frames_of(e))
            ib.ready()
            runner()
            ib.release()
            drawn.append([t.clone() for t in ib.word_tensors] + [runner.outputs[0].clone()])
    torch.cuda.synchronize()
    assert all(torch.equal(x, y) for x, y in zip(state(tra), state(trb)))
    assert int(tra.step_count.item()) == 4 and int(trb.step_count.item()) == 4
    assert int(trb.skipped.item()) == 0
    # successive replays drew different shuffle words, samples and dropout masks
    assert all(not torch.equal(x, y) for x, y in zip(drawn[0], drawn[1]))


# ----------------------------------------------------------------------------------------------------------- resume
def _steps(tr, roidb, first, count):
    inp = TR.StepInputs((FH, FW), SCALE, "cuda", max_rows=16)
    for k in range(first, first + count):
        e = roidb[k % len(roidb)]
        inp.load(e, *frames_of(e))
        tr.step_from_frames(inp)
    torch.cuda.synchronize()


def _final_state(tr):
    return {"masters": [v.cpu() for v in tr.masters.grads], "moms": [v.cpu() for v in tr.moms.grads],
            "uncert": tr.uncert.cpu(), "step": int(tr.step_count.item())}


def test_resume_in_a_second_process(tmp_path):
    roidb = synth_roidb()
    tr = new_trainer()
    _steps(tr, roidb, 0, 3)
    ck = tr.checkpoint()
    assert ck["step"] == 3 and ck["epoch"] == 1 and ck["lr"] == 1e-3
    torch.save(ck, tmp_path / "ck.pth")
    _steps(tr, roidb, 3, 3)
    want = _final_state(tr)
    res = subprocess.run([sys.executable, os.path.abspath(__file__), "resume", str(tmp_path / "ck.pth"),
                          str(tmp_path / "out.pth")], capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout + res.stderr
    got = torch.load(tmp_path / "out.pth")
    assert got["step"] == want["step"] == 6
    assert torch.equal(bits(got["uncert"]), bits(want["uncert"]))
    for k in ("masters", "moms"):
        assert all(torch.equal(bits(a), bits(b)) for a, b in zip(got[k], want[k])), k
    assert any(bool((m != 0).any()) for m in ck["momentum"].values())


def _resume_worker(ckpt_path, out_path):
    tr = new_trainer()
    tr.load_checkpoint(torch.load(ckpt_path))
    _steps(tr, synth_roidb(), 3, 3)
    torch.save(_final_state(tr), out_path)


# -------------------------------------------------------------------------------------------------------------- fit
def test_fit_trains_saves_and_resumes(tmp_path, capsys):
    roidb = synth_roidb()
    assert len(roidb) == 6
    sd = make_state_dict(3)
    lines = []
    tr = new_trainer(sd)
    totals = TR.fit(tr, roidb, frames_of, epochs=3, save_dir=str(tmp_path), log=lines.append, target_size=160,
                    max_rows=16)
    with capsys.disabled():
        print("fit, 3 epochs of 6 pairs at %dx%d, total loss: %s" % (160, 256, " ".join("%.4f" % t for t in totals)))
    assert len(totals) == 18 and all(np.isfinite(totals)) and int(tr.skipped.item()) == 0
    assert int(tr.step_count.item()) == 18 and tr.epoch == 4
    head = [l for l in lines if l.startswith("[epoch")]
    assert len(head) == 18 and len([l for l in lines if l.startswith("save model: ")]) == 3
    for k, l in enumerate(head):
        assert re.fullmatch(r"\[epoch  %d\]\[iter    %d/   6\] loss: -?\d+\.\d{4}, lr: 1\.00e-03" % (k // 6 + 1, k % 6), l), l
    body = [l for l in lines if l.startswith("\t\t\trpn_cls: ")]
    assert len(body) == 18 and all(re.fullmatch(
        r"\t\t\trpn_cls: \d+\.\d{4}, rpn_box_left_right: \d+\.\d{4}, rcnn_cls: \d+\.\d{4}, "
        r"rcnn_box_left_right \d+\.\d{4},dim_orien \d+\.\d{4}, kpts \d+\.\d{4}", l) for l in body)
    files = ["stereo_rcnn_%d_5.pth" % e for e in (1, 2, 3)]
    assert sorted(f for f in os.listdir(tmp_path) if f.endswith(".pth")) == files
    cks = [torch.load(tmp_path / f) for f in files]
    assert [c["epoch"] for c in cks] == [2, 3, 4] and [c["step"] for c in cks] == [6, 12, 18]
    assert np.mean(totals[12:]) < np.mean(totals[:6])
    # resumed from the first checkpoint: the later ones again, bit for bit
    tr2 = new_trainer(sd)
    tr2.load_checkpoint(cks[0])
    os.makedirs(tmp_path / "resumed")
    TR.fit(tr2, roidb, frames_of, epochs=3, start_epoch=cks[0]["epoch"], save_dir=str(tmp_path / "resumed"),
           log=lambda s: None, target_size=160, max_rows=16)
    for f, ref in zip(files[1:], cks[1:]):
        got = torch.load(tmp_path / "resumed" / f)
        assert got["epoch"] == ref["epoch"] and got["step"] == ref["step"] and got["lr"] == ref["lr"]
        assert torch.equal(bits(got["uncert"]), bits(ref["uncert"]))
        assert all(torch.equal(bits(got["momentum"][k]), bits(ref["momentum"][k])) for k in ref["momentum"])
        assert all(torch.equal(got["model"][k], ref["model"][k]) for k in ref["model"])


if __name__ == "__main__":
    assert sys.argv[1] == "resume"
    _resume_worker(sys.argv[2], sys.argv[3])
