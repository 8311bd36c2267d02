"""CPU: the record exchange over peer memory (csrc/peer.cu) refuses every invalid argument with SB_EINVAL before any
launch, and sb_peer_mailbox_bytes agrees with `Layout`, the Python mirror of the mailbox that
tests/test_gpu_peer_exchange.py uses to predict every word of every mailbox."""
import ctypes

import pytest

from stereo_rcnn_b200 import lib as L

SB_EINVAL = -22
FAKE = 1 << 20                                            # never dereferenced: every refusal precedes the first launch
MAX_PEERS, PARITIES = 16, 4


class Layout(object):
    """one rank's mailbox, in 32-bit words: data [n_slots][4 parities][world][rec_floats], then flags [n_slots][world],
    seq [n_slots], ticket [n_slots], then 64 spare bytes"""

    def __init__(self, n_slots, world, rec_floats):
        self.n_slots, self.world, self.rec_floats = n_slots, world, rec_floats
        self.data_words = n_slots * PARITIES * world * rec_floats

    def data_off(self, slot, par, rank):
        return ((slot * PARITIES + par) * self.world + rank) * self.rec_floats

    def flag_off(self, slot, rank):
        return self.data_words + slot * self.world + rank

    def seq_off(self, slot):
        return self.data_words + self.n_slots * self.world + slot

    def ticket_off(self, slot):
        return self.data_words + self.n_slots * self.world + self.n_slots + slot

    @property
    def bytes(self):
        return 4 * (self.data_words + self.n_slots * self.world + 2 * self.n_slots) + 64


@pytest.fixture(scope="module")
def lib():
    from stereo_rcnn_b200 import build
    build.build()
    return L.load()


def boxes(world, null_at=None, offset_at=None):
    n = max(world, 1)
    return (ctypes.c_void_p * n)(*[None if i == null_at else FAKE + 4096 * i + 4 * (i == offset_at) for i in range(n)])


def test_put_record_rejections(lib):
    def put(rec=FAKE, mailboxes="ok", n_slots=3, world=4, rec_floats=512, rank=1, slot=2):
        mb = boxes(world) if mailboxes == "ok" else mailboxes
        return lib.sb_peer_put_record(rec, mb, n_slots, world, rec_floats, rank, slot, None)
    n0 = lib.sb_launch_count()
    bad = {"null rec": put(rec=None), "null mailboxes": put(mailboxes=None),
           "null mailbox 0": put(mailboxes=boxes(4, null_at=0)), "null mailbox 3": put(mailboxes=boxes(4, null_at=3)),
           "misaligned mailbox 2": put(mailboxes=boxes(4, offset_at=2)), "world 0": put(world=0, rank=0),
           "world 17": put(world=MAX_PEERS + 1, mailboxes=boxes(MAX_PEERS + 1)), "world -1": put(world=-1),
           "rank -1": put(rank=-1), "rank == world": put(rank=4), "slot -1": put(slot=-1),
           "slot == n_slots": put(slot=3), "n_slots 0": put(n_slots=0, slot=0), "rec_floats 0": put(rec_floats=0),
           "rec_floats 3": put(rec_floats=3), "rec_floats 6": put(rec_floats=6), "rec_floats -4": put(rec_floats=-4),
           "misaligned rec": put(rec=FAKE + 4), "rec off by 8": put(rec=FAKE + 8)}
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}


def test_wait_records_rejections(lib):
    def wait(mailbox=FAKE, n_slots=3, world=4, rec_floats=512, slot=2, lag=1, gathered=FAKE, err=FAKE, timeout_s=20.0):
        return lib.sb_peer_wait_records(mailbox, n_slots, world, rec_floats, slot, lag, gathered, err, timeout_s, None)
    n0 = lib.sb_launch_count()
    inf, nan = float("inf"), float("nan")
    bad = {"null mailbox": wait(mailbox=None), "null gathered": wait(gathered=None), "null err": wait(err=None),
           "misaligned mailbox": wait(mailbox=FAKE + 4), "world 0": wait(world=0),
           "world 17": wait(world=MAX_PEERS + 1),
           "slot -1": wait(slot=-1), "slot == n_slots": wait(slot=3), "n_slots 0": wait(n_slots=0, slot=0),
           "lag -1": wait(lag=-1), "lag 2": wait(lag=2), "rec_floats 0": wait(rec_floats=0),
           "rec_floats 3": wait(rec_floats=3), "rec_floats 6": wait(rec_floats=6),
           "misaligned gathered": wait(gathered=FAKE + 4), "gathered off by 12": wait(gathered=FAKE + 12),
           "timeout nan": wait(timeout_s=nan), "timeout -nan": wait(timeout_s=-nan), "timeout inf": wait(timeout_s=inf),
           "timeout -inf": wait(timeout_s=-inf), "timeout -1e-9": wait(timeout_s=-1e-9),
           "timeout -1": wait(timeout_s=-1.0), "timeout past u64 ns": wait(timeout_s=1.9e10)}
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}


def test_alloc_rejections(lib):
    p = ctypes.c_void_p()
    n0 = lib.sb_launch_count()
    assert lib.sb_peer_alloc(0, ctypes.byref(p)) == SB_EINVAL
    assert lib.sb_peer_alloc(4096, None) == SB_EINVAL
    assert lib.sb_peer_alloc(0, None) == SB_EINVAL
    assert lib.sb_launch_count() == n0 and p.value is None


def test_mailbox_bytes_match_the_layout_mirror(lib):
    for n_slots, world, rec_floats in [(0, 2, 4), (-1, 2, 4), (1, 0, 4), (1, MAX_PEERS + 1, 4), (1, -2, 4), (1, 2, 0),
                                       (1, 2, 3), (1, 2, 6), (1, 2, -4), (3, 16, 9902)]:
        assert lib.sb_peer_mailbox_bytes(n_slots, world, rec_floats) == 0, (n_slots, world, rec_floats)
    for n_slots in (1, 2, 3, 7):
        for world in (1, 2, 3, 5, 8, 16):
            for rec_floats in (4, 8, 508, 512, 516, 1020, 1028, 9900):
                got = lib.sb_peer_mailbox_bytes(n_slots, world, rec_floats)
                assert got == Layout(n_slots, world, rec_floats).bytes, (n_slots, world, rec_floats)
    # the control words sit right after the data, in the order flags, seq, ticket, and nothing overlaps
    m = Layout(3, 5, 12)
    words = [m.data_off(s, p, r) + i for s in range(3) for p in range(PARITIES) for r in range(5) for i in range(12)]
    words += [m.flag_off(s, r) for s in range(3) for r in range(5)] + [m.seq_off(s) for s in range(3)]
    words += [m.ticket_off(s) for s in range(3)]
    assert sorted(words) == list(range(len(words))) and 4 * len(words) + 64 == m.bytes
