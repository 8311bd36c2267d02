"""GPU: pipeline.evaluate over several ranks and the validation pass of train.fit.

* Two or three processes over gloo share the GPU: at world 2 (7 entries, two frame shapes, labels) the files rank 0
  writes are byte-identical to the one-rank run's, with the same set of files with and without empty_files; the AP
  tables, n_gt and the curves are equal element for element and every rank returns the same summary; at world 3 with
  2 entries one rank's block is empty.
* A non-empty result directory on rank 0 makes every rank raise FileExistsError before any launch.
* After a real Trainer.step, eng.refresh_weights(trainer.params) on a validation pipeline gives the files of a
  pipeline built from trainer.state_dict(), in the evaluation that follows the refresh and in a second one that
  replays the same graphs; the device memory the first refresh adds is printed.
* fit with val trains bit-identically to fit without it, and val_summaries[e]["ap"] is evaluate's on a pipeline
  built from epoch e's checkpoint."""
import os
import socket

import numpy as np
import pytest
import torch

from stereo_rcnn_b200 import ops as G
from stereo_rcnn_b200 import pipeline as PL
from stereo_rcnn_b200 import train as TR
from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200.synth import make_state_dict
from test_gpu_evaluate import TARGET, calib, frame_pair, read_dir, split

pytestmark = pytest.mark.gpu


def car_state_dict():
    """the weights of test_gpu_evaluate's pipeline: Car scores well above eval_thresh"""
    sd = make_state_dict(3)
    b = sd["RCNN_cls_score.bias"].clone()
    b[1] += 4.0
    sd["RCNN_cls_score.bias"] = b
    return sd


def frames(e):
    return frame_pair(*e["hw"], seed=e["seed"])


def cal(e):
    return calib(e["cal"], div=3.75)


def label_text(e):
    """a seeded label file in the frame's coordinates: two Cars, one of them partly occluded, and a DontCare"""
    rs = np.random.RandomState(e["seed"])
    out = []
    for j in range(2):
        x1, y1 = rs.uniform(10, 200), rs.uniform(20, 50)
        out.append("Car 0.00 %d %.2f %.2f %.2f %.2f %.2f 1.50 1.60 3.90 %.2f 1.60 %.2f %.2f" % (
            j, rs.uniform(-3, 3), x1, y1, x1 + rs.uniform(25, 90), y1 + rs.uniform(20, 45), rs.uniform(-6, 6),
            rs.uniform(8, 30), rs.uniform(-3, 3)))
    out.append("DontCare -1 -1 -10 250.00 30.00 300.00 60.00 -1 -1 -1 -1000 -1000 -1000 -10")
    return "\n".join(out) + "\n"


def same_ap(a, b):
    """equal element for element: the tables, n_gt and (where both have them) the curves"""
    if sorted(a) != sorted(b):
        return False
    for m in ("bbox", "aos", "bev", "3d"):
        if sorted(a[m]) != sorted(b[m]) or not all(np.array_equal(a[m][t], b[m][t]) for t in a[m]):
            return False
    if not np.array_equal(a["n_gt"], b["n_gt"]):
        return False
    if "curves" in a:
        for m, per in a["curves"].items():
            for t, cur in per.items():
                if not all(np.array_equal(v, b["curves"][m][t][k]) for k, v in cur.items()):
                    return False
    return True


# ---------------------------------------------------------------------------------------- several ranks, one GPU
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _collect(q, procs, timeout_s):
    """{rank: result} of every worker; fails as soon as a worker has exited without putting one"""
    import queue
    import time
    res, t0 = {}, time.time()
    while len(res) < len(procs):
        try:
            r, v = q.get(timeout=5)
            res[r] = v
        except queue.Empty:
            dead = [i for i, p in enumerate(procs) if p.exitcode not in (None, 0) and i not in res]
            assert not dead, "rank(s) %s exited with %s" % (dead, [procs[i].exitcode for i in dead])
            assert time.time() - t0 < timeout_s, "workers did not finish"
    return res


def _shard_worker(rank, world, port, root, n, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank % torch.cuda.device_count())
    # ranks share a GPU: NCCL refuses two ranks on one device, so gloo carries the collectives
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        pipe = PL.StereoPipeline(car_state_dict(), torch.device("cuda"), throughput=True)
        entries = split(n)                                 # 7: both frame shapes, both slots
        labels = lambda e: label_text(e)
        mine = os.path.join(root, "rank%d" % rank)
        res = {"ok": True, "notes": []}

        def check(cond, what):
            if not cond:
                res["ok"] = False
                res["notes"].append(what)
        for empty in (False, True):
            single = None
            if rank == 0:
                single = PL.evaluate(pipe, entries, frames, cal, os.path.join(mine, "single%d" % empty),
                                     inflight=2, target_size=TARGET, empty_files=empty, log=lambda s: None,
                                     labels=labels)
            got = PL.evaluate(pipe, entries, frames, cal, os.path.join(mine, "sharded%d" % empty), inflight=2,
                              target_size=TARGET, empty_files=empty, log=lambda s: None, labels=labels, world=world,
                              dist=dist)
            timings = ("write_s", "gather_s", "score_s", "loop_s")
            res[empty] = dict(summary={k: v for k, v in got.items() if k not in timings},
                              files=read_dir(os.path.join(mine, "sharded%d" % empty, "data"))
                              if os.path.isdir(os.path.join(mine, "sharded%d" % empty)) else None)
            if rank == 0:
                want = read_dir(os.path.join(mine, "single%d" % empty, "data"))
                check(res[empty]["files"] == want, "files differ from the one-rank run (empty_files %s)" % empty)
                check(len(want) == (n if empty else single["files"]) and (single["files"] > 0 or n < 7), "file count")
                for k in ("images", "lines", "files"):
                    check(got[k] == single[k], k)
                check(same_ap(got["ap"], single["ap"]), "AP, n_gt or curves differ")
                check(n < 7 or got["ap"]["n_gt"][2] >= n, "n_gt")       # the labels carry hard Cars
        # refusal: rank 0's result directory already holds files; nothing is launched on any rank
        n0 = G.launch_count()
        try:
            PL.evaluate(pipe, entries, frames, cal, os.path.join(mine if rank == 0 else root, "sharded1"),
                        target_size=TARGET, log=lambda s: None, world=world, dist=dist)
            check(False, "no refusal")
        except FileExistsError:
            pass
        check(G.launch_count() == n0, "a refused call launched kernels")
        torch.cuda.synchronize()
        q.put((rank, res))
    except BaseException:
        import sys
        import traceback
        msg = traceback.format_exc()
        print("rank %d: %s" % (rank, msg), file=sys.stderr, flush=True)
        q.put((rank, {"ok": False, "notes": [msg]}))
        raise
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,n", [(2, 7), (3, 2)])
def test_sharded_evaluate_equals_one_rank(world, n, tmp_path):
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_shard_worker, args=(r, world, port, str(tmp_path), n, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = _collect(q, procs, 900)
    for r in range(world):
        assert res[r]["ok"], (r, res[r]["notes"])
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    blocks = [PL.parallel.shard_pairs(n, r, world) for r in range(world)]
    for r in range(world):
        assert res[r]["ok"], (r, res[r]["notes"])
    for r in range(world):
        for empty in (False, True):
            s, s0 = res[r][empty]["summary"], res[0][empty]["summary"]
            assert sorted(s) == sorted(s0) and s["rank_images"] == [e - b for b, e in blocks]
            assert all(s[k] == s0[k] for k in ("images", "lines", "files", "graphs", "rank_images"))
            assert same_ap(s["ap"], s0["ap"])
            if r:
                assert res[r][empty]["files"] is None                  # only rank 0 writes
    if world == 3:
        assert blocks[2][0] == blocks[2][1]


# ------------------------------------------------------------------------------------- refreshed validation engine
def _train_one_step(tr):
    from test_gpu_train_input import FH, FW, SCALE, frames_of, synth_roidb
    e = synth_roidb()[1]
    inp = TR.StepInputs((FH, FW), SCALE, "cuda", max_rows=16)
    inp.load(e, *frames_of(e))
    with torch.no_grad():
        tr.step_from_frames(inp)
    torch.cuda.synchronize()


def test_refreshed_pipeline_writes_the_files_of_a_fresh_one(tmp_path, capsys):
    sd = car_state_dict()
    tr = TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, grad_scale=2.0 ** 12, seed=5)
    entries = split(5)
    run = lambda pipe, tag, slots=None: (PL.evaluate(pipe, entries, frames, cal, str(tmp_path / tag), inflight=2,
                                                     target_size=TARGET, log=lambda s: None, slots=slots),
                                         read_dir(str(tmp_path / tag / "data")))
    val = PL.StereoPipeline(tr.state_dict(), torch.device("cuda"), throughput=True, precision=tr.engine.precision)
    slots = {}
    s, _files = run(val, "before", slots)
    assert s["graphs"] == 4 and s["files"] > 0
    before_params = {k: v.clone() for k, v in tr.params.items()}
    for step in (1, 2):
        _train_one_step(tr)
        assert any(not torch.equal(tr.params[k], before_params[k]) for k in tr.params)
        m0 = torch.cuda.memory_allocated()
        val.eng.refresh_weights(tr.params)
        torch.cuda.synchronize()
        if step == 1:
            with capsys.disabled():
                print("\nthe first refresh_weights of an inference engine adds %.1f MB of device memory"
                      % ((torch.cuda.memory_allocated() - m0) / 2 ** 20))
        fresh = PL.StereoPipeline(tr.state_dict(), torch.device("cuda"), throughput=True)
        _s, want = run(fresh, "fresh%d" % step)
        for again in (0, 1):                      # both evaluations replay the graphs of the first one
            s, got = run(val, "refreshed%d_%d" % (step, again), slots)
            assert s["graphs"] == 0
            assert got == want, (step, again)
        del fresh


# --------------------------------------------------------------------------------------------- fit with validation
def test_fit_with_validation_trains_as_without(tmp_path, capsys):
    from test_gpu_train_input import frames_of, synth_roidb, bits
    sd = car_state_dict()
    roidb = synth_roidb()
    entries = split(4)
    labels = lambda e: label_text(e)
    runs = {}
    for tag in ("plain", "val"):
        tr = TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, grad_scale=2.0 ** 12, seed=5)
        os.makedirs(tmp_path / tag)
        lines = []
        val = dict(entries=entries, frames=frames, calib=cal, result_dir=str(tmp_path / tag / "val"), labels=labels,
                   inflight=2) if tag == "val" else None
        totals = TR.fit(tr, roidb, frames_of, epochs=2, save_dir=str(tmp_path / tag), log=lines.append,
                        target_size=TARGET, max_rows=16, val=val)
        runs[tag] = dict(totals=totals, tr=tr, lines=lines,
                         cks=[torch.load(tmp_path / tag / ("stereo_rcnn_%d_5.pth" % e)) for e in (1, 2)])
    a, b = runs["plain"], runs["val"]
    assert np.array_equal(np.array(a["totals"], np.float32).view(np.int32),
                          np.array(b["totals"], np.float32).view(np.int32))
    ca, cb = a["cks"][1], b["cks"][1]
    assert ca["step"] == cb["step"] == 12 and ca["epoch"] == cb["epoch"] == 3
    assert torch.equal(bits(ca["uncert"]), bits(cb["uncert"]))
    assert all(torch.equal(bits(ca["momentum"][k]), bits(cb["momentum"][k])) for k in ca["momentum"])
    assert all(torch.equal(ca["model"][k], cb["model"][k]) for k in ca["model"])
    assert a["tr"].val_summaries == {} and sorted(b["tr"].val_summaries) == [1, 2]
    assert len([l for l in b["lines"] if l.startswith("evaluate: Car AP")]) == 2
    for e, ck in zip((1, 2), b["cks"]):
        s = b["tr"].val_summaries[e]
        assert "curves" not in s["ap"] and s["images"] == len(entries)
        assert sorted(os.listdir(tmp_path / "val" / "val")) == ["epoch_1", "epoch_2"]
        pipe = PL.StereoPipeline(ck["model"], torch.device("cuda"), throughput=True)
        ref = PL.evaluate(pipe, entries, frames, cal, str(tmp_path / ("ref%d" % e)), target_size=TARGET,
                          log=lambda m: None, labels=labels)
        assert same_ap(s["ap"], {k: v for k, v in ref["ap"].items() if k != "curves"}), e
        assert read_dir(str(tmp_path / "val" / "val" / ("epoch_%d" % e) / "data")) == read_dir(
            str(tmp_path / ("ref%d" % e) / "data"))
        with capsys.disabled():
            print("\nfit validation, epoch %d: Car AP|R11 2D %s" % (e, "/".join(
                "%.2f" % v for v in s["ap"]["bbox"][0.7][:, 0])))
