"""GPU: the record all-gather over peer memory (csrc/peer.cu: sb_peer_put_record, sb_peer_wait_records) held bit for
bit to a word-exact prediction of every mailbox, and parallel.RecordGather's peer path across processes.

One process emulates W ranks on one GPU: rank r's mailbox is row r of one zeroed int32 tensor (16-byte aligned rows,
no CUDA IPC needed), and `Layout` (tests/test_peer_exchange_args.py) predicts every word of every mailbox after each
put.  Every schedule is legal: a wait for step t is enqueued only after every rank's put of step t, on the one stream
all ranks share, so no wait spins.  The one exception is the timeout case, a single bounded 2 ms wait.  Records are
random 32-bit patterns (NaNs and denormals included): the exchange moves words and must not change one."""
import ctypes
import os
import random
import socket
import time

import pytest
import torch

from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import parallel as P
from test_peer_exchange_args import PARITIES, Layout

pytestmark = pytest.mark.gpu

SENT = 0x7FC0DEAD                  # a quiet-NaN pattern the records are not expected to contain
GUARD = 64                         # sentinel words on each side of a gathered buffer (keeps it 16-byte aligned)
TIMEOUT_S = 2e-3                   # no legal wait spins; a broken one costs at most this much
WORLDS = (1, 2, 3, 5, 8, 16)
# both sides of one float4, of the wait's 128-thread stride (512 floats) and of the put's 256-thread stride (1024)
REC_FLOATS = (4, 8, 508, 512, 516, 1020, 1028, 9900)


def i32(v):
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v >= 1 << 31 else v


def vp(t):
    return ctypes.c_void_p(t.data_ptr())


def random_words(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(-2 ** 31, 2 ** 31, shape, dtype=torch.int32, generator=g).cuda()


class Ring(object):
    """W ranks' mailboxes on one device.  `pred` is the predicted content of every word of `boxes` (words past the
    mailbox, up to the 16-byte row stride, must stay 0), `seq[r][slot]` rank r's step counter on the host.  A put is
    checked against `pred` right after it, a wait against the sentinel-guarded expected gather; both checks stay on the
    device until `verify()`."""

    def __init__(self, n_slots, world, rec_floats, mirror=True):
        self.lib = L.load()
        self.n_slots, self.world, self.rec_floats = n_slots, world, rec_floats
        nb = self.lib.sb_peer_mailbox_bytes(n_slots, world, rec_floats)
        self.m = Layout(n_slots, world, rec_floats) if mirror else None
        assert nb > 0 and (not mirror or nb == self.m.bytes)
        self.boxes = torch.zeros(world, (nb // 4 + 3) // 4 * 4, dtype=torch.int32, device="cuda")
        self.pred = torch.zeros_like(self.boxes) if mirror else None
        self.ptrs = (ctypes.c_void_p * world)(*[self.boxes[r].data_ptr() for r in range(world)])
        self.seq = [[0] * n_slots for _ in range(world)]
        self.err = torch.zeros(world, 4, dtype=torch.int32, device="cuda")
        self.gath = torch.empty(GUARD + world * rec_floats + GUARD, dtype=torch.int32, device="cuda")
        self.exp = torch.empty_like(self.gath)
        self.checks = []

    def put(self, r, slot, rec, what=""):
        assert rec.dtype == torch.int32 and rec.numel() == self.rec_floats and rec.data_ptr() % 16 == 0
        assert self.lib.sb_peer_put_record(vp(rec), self.ptrs, self.n_slots, self.world, self.rec_floats, r, slot,
                                           L.stream_ptr()) == 0
        seq = (self.seq[r][slot] + 1) & 0xFFFFFFFF
        self.seq[r][slot] = seq
        if self.pred is not None:
            o = self.m.data_off(slot, seq % PARITIES, r)
            self.pred[:, o:o + self.rec_floats] = rec                         # row (slot, seq % 4, r) of every peer
            self.pred[:, self.m.flag_off(slot, r)] = i32(seq)                 # flag (slot, r) of every peer
            self.pred[r, self.m.seq_off(slot)] = i32(seq)                     # own counter; own ticket stays 0
            self.checks.append(("put rank %d slot %d seq %d %s" % (r, slot, seq, what),
                                (self.boxes != self.pred).any()))

    def wait(self, r, slot, lag, out, timeout_s=TIMEOUT_S):
        assert self.lib.sb_peer_wait_records(vp(self.boxes[r]), self.n_slots, self.world, self.rec_floats, slot, lag,
                                             vp(out), vp(self.err[r]), timeout_s, L.stream_ptr()) == 0

    def wait_check(self, r, slot, lag, expect, what=""):
        """one wait into the guarded buffer; `expect` [world, rec_floats] words, or None: `out` left untouched"""
        self.gath.fill_(SENT)
        self.wait(r, slot, lag, self.gath[GUARD:])
        self.exp.fill_(SENT)
        if expect is not None:
            self.exp[GUARD:GUARD + self.world * self.rec_floats] = expect.reshape(-1)
        self.checks.append(("wait rank %d slot %d lag %d %s" % (r, slot, lag, what), (self.gath != self.exp).any()))

    def verify(self, tag):
        if self.pred is not None:
            self.checks.append(("mailboxes at the end", (self.boxes != self.pred).any()))
        bad = torch.stack([c for _, c in self.checks]).cpu() if self.checks else torch.zeros(0, dtype=torch.bool)
        first = [w for (w, _), b in zip(self.checks, bad.tolist()) if b][:3]
        assert not first, "%s: %d of %d checks fail, first %s" % (tag, int(bad.sum()), len(bad), first)
        assert int(self.err.abs().sum()) == 0, "%s: a wait timed out: %s" % (tag, self.err[:, 0].tolist())
        self.checks = []


def slot_order(n_slots, steps_per_slot, seed):
    order = [s for s in range(n_slots) for _ in range(steps_per_slot)]
    random.Random(seed).shuffle(order)                       # uneven interleaving of the slots
    return order


@pytest.mark.parametrize("lag", [0, 1])
def test_exchange_grid_bit_exact_with_guard_bands(lag):
    """world x n_slots x rec_floats, 9 steps per slot (every parity reused twice), slots unevenly interleaved, puts and
    waits in shuffled rank order; every mailbox word after every put, and every gathered word plus guard bands after
    every wait.  Lag 1: the first wait of a slot leaves `out` untouched, later ones return the previous step, and a
    final lag-0 wait (RecordGather.drain) returns the last step."""
    steps, n = 9, 0
    t0 = time.time()
    for world in WORLDS:
        for n_slots in (1, 3):
            for rec_floats in REC_FLOATS:
                seed = ((world * 10 + n_slots) * 10 + REC_FLOATS.index(rec_floats)) * 2 + lag
                ring = Ring(n_slots, world, rec_floats)
                recs = random_words((n_slots, steps, world, rec_floats), seed)
                done = [0] * n_slots
                rs = random.Random(seed)
                for slot in slot_order(n_slots, steps, seed):
                    t = done[slot]
                    done[slot] += 1
                    for r in rs.sample(range(world), world):
                        ring.put(r, slot, recs[slot, t, r], "step %d" % t)
                    for r in rs.sample(range(world), world):
                        ring.wait_check(r, slot, lag, recs[slot, t - lag] if t >= lag else None, "step %d" % t)
                if lag:
                    for slot in range(n_slots):
                        for r in range(world):
                            ring.wait_check(r, slot, 0, recs[slot, steps - 1], "drain")
                ring.verify("world %d n_slots %d rec_floats %d lag %d" % (world, n_slots, rec_floats, lag))
                n += 1
    print("%d configurations at lag %d in %.1f s" % (n, lag, time.time() - t0))


@pytest.mark.parametrize("world", [2, 3])
def test_tightest_lag1_schedule_keeps_four_live_records(world):
    """The legal interleaving the four parities exist for: rank A puts step s+1 before rank B copies out step s-2.
        B.put(s-1); A.put(s-1), A.wait(s-2); A.put(s), A.wait(s-1); A.put(s+1); B.wait(s-2) ...
    B must still read step s-2's records (three parities would hand it step s+1's row of A).  The other ranks (world
    3) move with B.  Rounds alternate A between rank 0 and rank 1 and cover every parity.  Uses only the library's
    mailbox size, not the Layout mirror, so a different parity count is caught here by its content alone."""
    rf, slot, rounds = 516, 1, 8
    ring = Ring(2, world, rf, mirror=False)
    recs = random_words((3 * rounds, world, rf), 77 + world)
    rec = lambda step, r: recs[step - 1, r]                   # steps are 1-based, like the counters
    n_checks = 0

    def wait_expect(r, step):
        nonlocal n_checks
        ring.wait_check(r, slot, 1, recs[step - 1] if step >= 1 else None, "collect step %d" % step)
        n_checks += 1
    n = 0                                                     # every rank has put n and collected n - 1
    for k in range(rounds):
        a = k % 2
        rest = [r for r in range(world) if r != a]
        for b in rest:
            ring.put(b, slot, rec(n + 1, b))
        ring.put(a, slot, rec(n + 1, a))
        wait_expect(a, n)
        ring.put(a, slot, rec(n + 2, a))
        wait_expect(a, n + 1)
        ring.put(a, slot, rec(n + 3, a))                      # A is now at s+1 = n+3 while B still owes s-2 = n
        for b in rest:
            wait_expect(b, n)
        for step in (n + 2, n + 3):
            for b in rest:
                ring.put(b, slot, rec(step, b))
                wait_expect(b, step - 1)
        wait_expect(a, n + 2)
        n += 3
    for r in range(world):
        ring.wait_check(r, slot, 0, recs[n - 1], "drain")
        n_checks += 1
    ring.verify("tightest lag-1 schedule, world %d" % world)
    print("world %d: %d rounds, %d gathered buffers checked" % (world, rounds, n_checks))


def copies(counter, lag):
    """the documented counter rule (csrc/peer.cu): a wait copies unless the slot's 32-bit counter, after this rank's
    put, is below 1 + lag -- "nothing that old has been put yet", which a counter past 2^32 - 1 also reads as"""
    return (counter & 0xFFFFFFFF) >= 1 + lag


@pytest.mark.parametrize("lag", [0, 1])
@pytest.mark.parametrize("start", [2 ** 31 - 6, 2 ** 32 - 6])
def test_step_counters_across_2_31_and_2_32(start, lag):
    """Every mailbox seeded to "everyone has put step S" (seq and every flag S, tickets 0, step S's records in parity
    S % 4), then 12 steps per slot.  Across 2^31 the exchange is continuous.  Across 2^32 the counter reaches the
    "never put" value 0: exactly that step's wait (and at lag 1 the next one's) returns without copying, every other
    step gathers the right records, and the parity ring carries on (2^32 is a multiple of 4)."""
    world, n_slots, rf, steps = 3, 2, 516, 12
    ring = Ring(n_slots, world, rf)
    m = ring.m
    recs = random_words((n_slots, steps + 1, world, rf), start % 1000 + lag)      # index 0: the seeded step S
    for slot in range(n_slots):
        for q in range(world):
            o = m.data_off(slot, start % PARITIES, q)
            ring.pred[:, o:o + rf] = recs[slot, 0, q]
            ring.pred[:, m.flag_off(slot, q)] = i32(start)
        ring.pred[:, m.seq_off(slot)] = i32(start)
        for r in range(world):
            ring.seq[r][slot] = start
    ring.boxes.copy_(ring.pred)
    skipped = 0
    for j in range(1, steps + 1):
        for slot in (j % n_slots, (j + 1) % n_slots):
            for r in range(world):
                ring.put(r, slot, recs[slot, j, r], "step S+%d" % j)
            c = start + j
            for r in range(world):
                ring.wait_check(r, slot, lag, recs[slot, j - lag] if copies(c, lag) else None, "step S+%d" % j)
            skipped += not copies(c, lag)
    if lag:
        for slot in range(n_slots):
            for r in range(world):
                ring.wait_check(r, slot, 0, recs[slot, steps], "drain")
    ring.verify("counters from %d, lag %d" % (start, lag))
    # the rule itself: continuous across 2^31, one (lag 0) or two (lag 1) skipped steps per slot across 2^32
    assert skipped == (0 if start < 2 ** 32 - steps else n_slots * (1 + lag))
    print("S = %d, lag %d: %d steps per slot, %d waits left out untouched by the wrap" % (start, lag, steps, skipped))


@pytest.mark.parametrize("lag", [0, 1])
def test_graph_replay_advances_device_counters(lag):
    """One step of all W puts and waits of a slot captured in a CUDA graph and replayed 10 times, the records changed
    in place between replays: each replay gathers that replay's records (lag 0) or the previous replay's (lag 1; the
    first leaves `out` untouched), because the step counters live on the device."""
    world, n_slots, slot, rf, replays = 4, 2, 1, 1028, 10
    ring = Ring(n_slots, world, rf)
    m = ring.m
    recs = torch.empty(world, rf, dtype=torch.int32, device="cuda")
    outs = torch.empty(world, GUARD + world * rf + GUARD, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        for r in range(world):
            assert ring.lib.sb_peer_put_record(vp(recs[r]), ring.ptrs, n_slots, world, rf, r, slot, L.stream_ptr()) == 0
        for r in range(world):
            ring.wait(r, slot, lag, outs[r, GUARD:])
    assert int(ring.boxes.abs().sum()) == 0                                 # capturing ran nothing
    values = random_words((replays, world, rf), 5 + lag)
    for k in range(replays):
        recs.copy_(values[k])
        outs.fill_(SENT)
        graph.replay()
        exp = torch.full_like(outs[0], SENT)
        if k >= lag:
            exp[GUARD:GUARD + world * rf] = values[k - lag].reshape(-1)
        torch.cuda.synchronize()
        for r in range(world):
            assert torch.equal(outs[r], exp), "replay %d, rank %d" % (k, r)
        words = ring.boxes[:, m.seq_off(slot)].tolist()
        assert words == [k + 1] * world, (k, words)
    if lag:
        ring.gath.fill_(SENT)
        ring.wait(2, slot, 0, ring.gath[GUARD:])
        assert torch.equal(ring.gath[GUARD:GUARD + world * rf], values[-1].reshape(-1))
    assert int(ring.boxes[:, m.seq_off(0)].abs().sum()) == 0                # the other slot never moved
    assert int(ring.boxes[:, m.ticket_off(slot)].abs().sum()) == 0
    for r in range(world):                                  # the newest two steps sit in their parities everywhere
        for k in (replays - 1, replays - 2):
            for q in range(world):
                o = m.data_off(slot, (k + 1) % PARITIES, q)
                assert torch.equal(ring.boxes[r, o:o + rf], values[k, q])
    assert int(ring.err.abs().sum()) == 0
    print("lag %d: %d replays of %d puts + %d waits" % (lag, replays, world, world))


def test_wait_times_out_on_a_rank_that_never_puts():
    """One bounded wait: world 2, rank 0 puts and waits with a 2 ms timeout, rank 1 never puts.  The call returns
    with err = 1 + 1 (rank 1 missing), row 0 is copied and row 1 keeps its sentinels."""
    world, rf = 2, 8
    ring = Ring(1, world, rf)
    rec = random_words((rf,), 9)
    ring.put(0, 0, rec)
    assert torch.equal(ring.boxes, ring.pred)
    ring.gath.fill_(SENT)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    ring.wait(0, 0, 0, ring.gath[GUARD:], timeout_s=2e-3)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1)
    g = ring.gath
    assert int(ring.err[0, 0]) == 2 and int(ring.err[1].abs().sum()) == 0
    assert torch.equal(g[GUARD:GUARD + rf], rec)
    assert bool((g[:GUARD] == SENT).all()) and bool((g[GUARD + rf:] == SENT).all())
    assert ms >= 1.9, ms                                    # it did wait out the timeout (device clock)
    print("timed-out wait returned after %.2f ms, err %d" % (ms, int(ring.err[0, 0])))


# ------------------------------------------------------------------ RecordGather across processes (CUDA IPC)
SHAPES = ((300, 33), (7, 33), (1, 5), (301, 33))
LAYOUTS = ("contiguous", "transposed", "offset by one float")


def _record(shape, step, slot, rank):
    g = torch.Generator().manual_seed(100000 * SHAPES.index(shape) + 1000 * step + 10 * slot + rank)
    return torch.rand(shape, generator=g)


def _laid_out(x, layout, dev):
    if layout == "transposed":                              # a non-contiguous view
        return x.t().contiguous().to(dev).t()
    if layout == "offset by one float":                     # contiguous but 4 bytes past 16-byte alignment
        buf = torch.zeros(x.numel() + 1, device=dev)
        buf[1:].copy_(x.reshape(-1))
        return buf[1:].view(x.shape)
    return x.to(dev)


def _record_gather_worker(rank, world, port, q):
    import torch.distributed as dist
    bad, n = [], 0
    try:
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
        dev = torch.device("cuda", rank % torch.cuda.device_count())
        torch.cuda.set_device(dev)
        dist.init_process_group("gloo", rank=rank, world_size=world)
        for shape in SHAPES:
            for lag in (0, 1):
                gat = P.RecordGather(world, rank, dev, dist, n_slots=2, mode="peer", rec_shape=shape, lag=lag,
                                     timeout_s=10.0)
                if gat.mode != "peer":
                    bad.append("%s: %s" % (shape, gat.describe()))
                    continue
                steps = 6
                for step in range(steps):
                    for slot in (0, 1):
                        layout = LAYOUTS[(step + slot) % len(LAYOUTS)]
                        out = gat(slot, _laid_out(_record(shape, step, slot, rank), layout, dev))
                        torch.cuda.synchronize()
                        got = out.cpu()
                        what = "shape %s lag %d step %d slot %d (%s)" % (shape, lag, step, slot, layout)
                        # the wait writes world x rec_floats floats from out's first element: all inside out's storage
                        st = out.untyped_storage()
                        if out.data_ptr() - st.data_ptr() + 4 * world * gat.rec_floats > st.nbytes():
                            bad.append("%s: the gather writes past the end of out" % what)
                        if tuple(out.shape) != (world,) + shape:
                            bad.append("%s: out has shape %s" % (what, tuple(out.shape)))
                        if step >= lag:
                            for r in range(world):
                                if not torch.equal(got[r], _record(shape, step - lag, slot, r)):
                                    bad.append("%s: out[%d] differs" % (what, r))
                        n += 1
                for slot in (0, 1):
                    out = gat.drain(slot)
                    torch.cuda.synchronize()
                    for r in range(world):
                        if not torch.equal(out[r].cpu(), _record(shape, steps - 1, slot, r)):
                            bad.append("shape %s lag %d drain slot %d: out[%d] differs" % (shape, lag, slot, r))
                gat.check()
    except Exception as e:                                  # reported, not lost in the child's stderr
        bad.append("%s: %s" % (type(e).__name__, e))
    finally:
        q.put((rank, bad, n))
        if dist.is_initialized():
            dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_record_gather_peer_padded_and_staged_records_across_processes():
    """Two ranks in two processes (gloo control plane, records over CUDA IPC mailboxes) at the bench's 300 x 33, at
    R*C not a multiple of 4 (7 x 33, 1 x 5, 301 x 33), at lag 0 and at lag 1 with drain, with records contiguous,
    transposed and misaligned (the last two take the staging copy): out[r] is rank r's record, and nothing the wait
    writes lies past out's storage."""
    import queue

    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_record_gather_worker, args=(r, world, port, q)) for r in range(world)]
    deadline = time.time() + 300
    try:
        for p in procs:
            p.start()
        res = []
        while len(res) < world and time.time() < deadline:
            try:
                res.append(q.get(timeout=1))
            except queue.Empty:
                if not any(p.is_alive() for p in procs):
                    break
        for p in procs:
            p.join(max(deadline - time.time(), 1))
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(10)
            if p.is_alive():
                p.kill()
                p.join(10)
    assert len(res) == world, "only %d of %d ranks reported: %s" % (len(res), world, res)
    assert all(p.exitcode == 0 for p in procs), [p.exitcode for p in procs]
    for rank, bad, n in sorted(res):
        assert not bad, "rank %d: %d failures, first %s" % (rank, len(bad), bad[:4])
    print("%d ranks x %d gathers (%d shapes x lag 0/1 x 2 slots x 6 steps)" % (world, res[0][2], len(SHAPES)))
