"""CPU, gloo, world 2 and 3: the host side of pipeline.evaluate over several ranks, with a stub in place of the device
loop -- the shard of each rank, the merge of (entry index, lines) on rank 0 in entry order, the files only rank 0
writes (with and without empty_files), the summary every rank returns, a rank with an empty block, and the refusals
raised on every rank before any entry is read."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from stereo_rcnn_b200 import pipeline as PL

N_ENTRIES = 7


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def rows(k):
    """box_rectify-like rows of entry k: k % 3 valid detections (entries 0, 3, 6 have none) and one invalid row"""
    n = k % 3
    r = torch.zeros(n + 1, 13)
    for j in range(n):
        r[j] = torch.tensor([1.0, 0.5 + 0.01 * k, 10 + j, 20, 60 + k, 90, 1.0, 1.6, 10.0 + k, 1.5, 1.6, 3.9, 0.1 * j])
    return r


def stub_block(seen):
    """what _eval_block does for the host: emit(k, final, t_x) once per entry of the block, in entry order"""
    def block(pipe, entries, ks, frames, calib, inflight, use_graph, target_size, rgb_input, states, emit):
        ks = list(ks)
        seen.extend(ks)
        for k in ks:
            emit(k, rows(k), 0.06 * (k % 2))
        return len({entries[k]["shape"] for k in ks})          # one "graph" per frame shape of the block
    return block


def entries(n):
    return [dict(image_id="%06d" % (5 * k), shape=k % 2) for k in range(n)]


def expected_files(n, empty_files):
    from stereo_rcnn_b200 import ops
    out = {}
    for k in range(n):
        lines = ops.kitti_result_lines(rows(k), 0.06 * (k % 2))
        if lines or empty_files:
            out["%06d.txt" % (5 * k)] = "".join(lines)
    return out


def read_dir(d):
    return {f: open(os.path.join(d, f)).read() for f in sorted(os.listdir(d))} if os.path.isdir(d) else None


def _worker(rank, world, port, root, n, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        res = {}
        seen = []
        PL._eval_block = stub_block(seen)
        ents = entries(n)
        for empty in (False, True):
            # each rank has a directory of its own: only rank 0 may create or write one
            out = os.path.join(root, "rank%d" % rank, "run%d" % empty)
            logs = []
            s = PL.evaluate(None, ents, None, None, out, use_graph=False, empty_files=empty, log=logs.append,
                            world=world, dist=dist)
            assert len(s.pop("loop_s")) == world and s.pop("write_s") >= 0 and s.pop("gather_s") >= 0
            res[empty] = dict(summary=s, files=read_dir(os.path.join(out, "data")), seen=list(seen), logs=logs)
            del seen[:]
        # refusals: a non-empty result directory on rank 0, and a bad inflight on one rank only
        errs = []

        def boom(e):
            raise AssertionError("an entry was read")
        d0 = os.path.join(root, "rank0", "run0")
        for kw in (dict(result_dir=d0 if rank == 0 else os.path.join(root, "fresh%d" % rank)),
                   dict(result_dir=os.path.join(root, "rank%d" % rank, "bad"), inflight=0 if rank == world - 1 else 1)):
            try:
                PL.evaluate(None, ents, boom, boom, use_graph=False, world=world, dist=dist, **kw)
                errs.append(None)
            except (FileExistsError, ValueError) as e:
                errs.append(type(e).__name__)
        res["errs"] = errs
        res["fresh"] = os.path.exists(os.path.join(root, "fresh%d" % rank))
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


@pytest.mark.parametrize("world,n", [(2, N_ENTRIES), (3, 2)])
def test_sharded_evaluate_merges_writes_and_broadcasts(world, n, tmp_path):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, world, port, str(tmp_path), n, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=300) for _ in range(world))
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    blocks = [list(range(*PL.parallel.shard_pairs(n, r, world))) for r in range(world)]
    assert sum(blocks, []) == list(range(n)) and (world < 3 or blocks[2] == [])
    for empty in (False, True):
        want = expected_files(n, empty)
        s0 = res[0][empty]["summary"]
        assert res[0][empty]["files"] == want                 # rank 0 writes every file, in its own directory
        for r in range(world):
            got = res[r][empty]
            assert got["seen"] == blocks[r]                   # each rank ran its contiguous block only
            assert got["summary"] == s0                       # every rank returns rank 0's summary
            if r:
                assert got["files"] is None and got["logs"] == []   # other ranks create and log nothing
        assert s0["images"] == n and s0["files"] == len(want)
        assert s0["lines"] == sum(v.count("\n") for v in want.values())
        assert s0["rank_images"] == [len(b) for b in blocks]
        assert s0["graphs"] == sum(len({k % 2 for k in b}) for b in blocks)
        assert "ap" not in s0
        assert res[0][empty]["logs"][0] == "evaluate: %d images, %d lines in %d files, %d graphs on %d ranks" % (
            n, s0["lines"], s0["files"], s0["graphs"], world)
    for r in range(world):
        assert res[r]["errs"] == ["FileExistsError", "ValueError"], (r, res[r]["errs"])
        assert not res[r]["fresh"]


def test_world_one_and_no_dist_take_the_single_rank_path(tmp_path, monkeypatch):
    """world 1, or world > 1 without dist: no collective, every file written here"""
    seen = []
    monkeypatch.setattr(PL, "_eval_block", stub_block(seen))
    for i, (world, d) in enumerate(((1, dist), (4, None))):
        out = str(tmp_path / str(i))
        s = PL.evaluate(None, entries(N_ENTRIES), None, None, out, use_graph=False, log=lambda m: None,
                        world=world, dist=d)
        assert seen == list(range(N_ENTRIES))
        del seen[:]
        assert read_dir(os.path.join(out, "data")) == expected_files(N_ENTRIES, False)
        assert "rank_images" not in s and "gather_s" not in s and s["images"] == N_ENTRIES
