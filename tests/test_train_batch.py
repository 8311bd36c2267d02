"""CPU: the batches of train.fit at several pairs per step and several ranks (train.epoch_batches: one frame shape per
batch, the short tails dropped, the epoch sharded over the ranks) and the argument checks of sb_prep_stereo_pairs
(SB_EINVAL before any CUDA call)."""
import pytest
import torch

from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import train as TR

SB_EINVAL = -22
FAKE = 1 << 20                                            # never dereferenced: every refusal precedes the first call


def roidb():
    """22 entries over three frame shapes, interleaved so that first appearance differs from the sorted order"""
    order = [1, 0, 2, 0, 0, 1, 0, 2, 1, 0, 0, 1, 2, 0, 1, 0, 2, 1, 0, 0, 1, 0]
    shapes = [(370, 1224), (375, 1242), (374, 1238)]
    return [{"height": shapes[s][0], "width": shapes[s][1], "index": i} for i, s in enumerate(order)]


def shape_of(e):
    return e["height"], e["width"]


@pytest.mark.parametrize("B", [1, 2, 3])
@pytest.mark.parametrize("world", [1, 2, 3])
def test_epoch_batches_group_drop_and_shard(B, world):
    db = roidb()
    sizes = {}
    for e in db:
        sizes[shape_of(e)] = sizes.get(shape_of(e), 0) + 1
    assert sorted(sizes.values()) == [4, 7, 11]
    n_batches = len(db) if B == 1 else sum(c // B for c in sizes.values())
    steps = n_batches // world
    g = torch.Generator().manual_seed(7)
    for _epoch in range(3):
        state = g.get_state()
        whole = TR.epoch_batches(db, B, g)                           # the epoch as one rank would see it
        after = g.get_state()
        assert len(whole) == n_batches and all(len(b) == B for b in whole)
        flat = [i for b in whole for i in b]
        assert len(set(flat)) == len(flat)                          # no entry twice in an epoch
        assert all(len({shape_of(db[i]) for i in b}) == 1 for b in whole)
        if B > 1:                                                   # the drop per shape is its count mod B
            for hw, c in sizes.items():
                assert sum(shape_of(db[i]) == hw for i in flat) == c - c % B
        ranks = []
        for r in range(world):
            g.set_state(state)
            ranks.append(TR.epoch_batches(db, B, g, rank=r, world=world))
            assert torch.equal(g.get_state(), after)                # every rank draws the same amount
        assert all(len(rb) == steps for rb in ranks)
        assert all(ranks[r][k] == whole[k * world + r] for r in range(world) for k in range(steps))
        seen = [i for rb in ranks for b in rb for i in b]
        assert len(set(seen)) == len(seen)                          # the ranks' batches are disjoint
        assert sorted(seen) == sorted(i for b in whole[:world * steps] for i in b)
        g.set_state(state)
        assert TR.epoch_batches(db, B, g) == whole                  # same generator state, same epoch


def test_epoch_batches_at_one_pair_and_one_rank_is_epoch_order():
    db = roidb()
    g, h = torch.Generator().manual_seed(3), torch.Generator().manual_seed(3)
    for _ in range(3):
        assert TR.epoch_batches(db, 1, g) == [[i] for i in TR.epoch_order(len(db), h)]
    # at one pair per step the frame shape is not needed
    assert len(TR.epoch_batches([{}] * 5, 1, g)) == 5


def test_epoch_batches_groups_in_order_of_first_appearance():
    """the group permutations are drawn in the order in which the shapes first appear, then the batch permutation"""
    db = roidb()
    g, h = torch.Generator().manual_seed(1), torch.Generator().manual_seed(1)
    got = TR.epoch_batches(db, 2, g)
    groups = {}
    for i, e in enumerate(db):
        groups.setdefault(shape_of(e), []).append(i)
    assert list(groups) == [(375, 1242), (370, 1224), (374, 1238)]
    cut = []
    for members in groups.values():
        perm = torch.randperm(len(members), generator=h).tolist()
        cut += [[members[j] for j in perm[k:k + 2]] for k in range(0, len(perm) - 1, 2)]
    assert got == [cut[j] for j in torch.randperm(len(cut), generator=h).tolist()]


def test_epoch_batches_need_the_frame_shape_and_valid_ranks():
    db = roidb()
    for key in ("height", "width"):
        bad = [dict(e) for e in db]
        del bad[5][key]
        with pytest.raises(ValueError):
            TR.epoch_batches(bad, 2, torch.Generator())
    g = torch.Generator()
    for B, rank, world in ((0, 0, 1), (2, 2, 2), (2, -1, 2), (2, 0, 0)):
        with pytest.raises(ValueError):
            TR.epoch_batches(db, B, g, rank=rank, world=world)


@pytest.fixture(scope="module")
def lib():
    from stereo_rcnn_b200 import build
    build.build()
    return L.load()


def test_prep_stereo_pairs_rejects_bad_arguments(lib):
    def pairs(left=FAKE, right=FAKE, B=2, H=375, W=1242, scale=1.6, flip=FAKE, ol=FAKE, orr=FAKE):
        return lib.sb_prep_stereo_pairs(left, right, B, H, W, scale, 1, flip, ol, orr, None)
    n0 = lib.sb_launch_count()
    bad = {"null left": pairs(left=None), "null right": pairs(right=None), "null flip": pairs(flip=None),
           "null out_left": pairs(ol=None), "null out_right": pairs(orr=None), "B 0": pairs(B=0), "B -1": pairs(B=-1),
           "B 32768": pairs(B=32768), "H 0": pairs(H=0), "W 0": pairs(W=0), "scale 0": pairs(scale=0.0),
           "scale < 0": pairs(scale=-1.6), "scale nan": pairs(scale=float("nan")),
           "rounds to no rows": pairs(H=1, scale=0.25)}
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}
