"""GPU: sb_kitti_annotations bit for bit against oracle/kitti_annotations.py on every output and status -- the
reference golden's boundary and seeded cases, and a seeded split of the size of KITTI train run twice -- the host's
ValueError for an image the reference stops on, and train_roidb feeding one epoch of train.fit from a KITTI folder."""
import os

import numpy as np
import pytest
import torch

from oracle import kitti_annotations as OA
from oracle import train_input as TI
from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200 import kitti_data as KD
from stereo_rcnn_b200 import ops
from stereo_rcnn_b200 import synth
from stereo_rcnn_b200 import train as TR

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "kitti_annotations.npz")


def golden_folder(root, g, which):
    d = os.path.join(root, "training")
    for sub in ("label_2", "calib", "image_2", "image_3"):
        os.makedirs(os.path.join(d, sub), exist_ok=True)
    ids = []
    for i in which:
        idx = "%06d" % i
        ids.append(idx)
        with open(os.path.join(d, "label_2", idx + ".txt"), "w") as f:
            f.write(str(g["labels"][i]))
        with open(os.path.join(d, "calib", idx + ".txt"), "w") as f:
            f.write(str(g["calibs"][i]))
        h, w = (int(v) for v in g["image_hw"][i])
        head = synth.png_bytes(np.zeros((1, 1, 3), np.uint8))[:16] + w.to_bytes(4, "big") + h.to_bytes(4, "big")
        for sub in ("image_2", "image_3"):
            with open(os.path.join(d, sub, idx + ".png"), "wb") as f:
                f.write(head + b"\x08\x02\x00\x00\x00")
    return ids


def same(split, dev_out):
    out, n_kept, status = dev_out
    o_out, o_n, o_st = OA.split(*split.arrays())
    assert np.array_equal(status, o_st)
    assert np.array_equal(n_kept, o_n)
    assert np.array_equal(out.view(np.uint32), o_out.view(np.uint32))


def test_device_equals_the_oracle_on_the_golden_cases(tmp_path):
    g = dict(np.load(GOLD))
    ids = golden_folder(str(tmp_path), g, range(len(g["names"])))
    split = KD.Split(str(tmp_path), ids)
    res = KD.run(split, "cuda")
    same(split, res)
    assert np.array_equal(res[2], g["status"]) and np.array_equal(res[1], g["n_kept"])


def test_every_golden_case_alone(tmp_path):
    """one image per launch: the CSR offsets start at 0, the image is the whole split"""
    g = dict(np.load(GOLD))
    for i in range(len(g["names"])):
        d = str(tmp_path / str(i))
        split = KD.Split(d, golden_folder(d, g, [i]))
        same(split, KD.run(split, "cuda"))


def test_non_positive_image_size_gives_status_minus_one(tmp_path):
    """H or W not positive (a caller packing its own split; kitti_data refuses such PNG headers): status -1, nothing
    kept, the image's rows zeroed, and the other images of the launch unaffected"""
    g = dict(np.load(GOLD))
    names = list(g["names"])
    which = [names.index(n) for n in ("chain_far_first", "tie", "kp_left_vl5", "hundred")]
    split = KD.Split(str(tmp_path), golden_folder(str(tmp_path), g, which))
    split.image_hw[1] = (0, 1242)
    split.image_hw[2] = (375, -3)
    dev = torch.device("cuda")
    buf, out = split.outputs(dev)
    buf.fill_(7.0)                                        # the zeroed rows are written, not left as they were
    ops.kitti_annotations(*split.to_device(dev), out=out)
    res = tuple(t.cpu().numpy() for t in out)
    assert res[2].tolist()[:3] == [0, -1, -1] and res[1][1] == res[1][2] == 0 and res[1][0] == 3
    a, b = int(split.obj_off[1]), int(split.obj_off[3])
    assert not res[0][a:b].any()
    same(split, res)


def test_kitti_train_sized_split_twice_identical(tmp_path):
    ids = synth.kitti_folder(str(tmp_path), 3712, seed=21)
    split = KD.Split(str(tmp_path), ids)
    a = KD.run(split, "cuda")
    b = KD.run(split, "cuda")
    for x, y in zip(a, b):
        assert x.tobytes() == y.tobytes()
    same(split, a)
    assert int(a[1].sum()) > 3712


def test_host_raises_for_an_image_the_reference_stops_on(tmp_path):
    g = dict(np.load(GOLD))
    names = list(g["names"])
    ids = golden_folder(str(tmp_path), g, [names.index("tie"), names.index("past_1259")])
    with pytest.raises(ValueError, match=r"image %s: the box of the object on line 1 of .* reaches past column 1259"
                                         r".*the reference raises IndexError here" % ids[1]):
        KD.annotations(str(tmp_path), ids, "cuda")
    entries = KD.annotations(str(tmp_path), ids[:1], "cuda")
    assert len(entries) == 1 and len(entries[0]["gt_classes"]) == 2


def test_workspace_and_argument_refusals():
    L = __import__("stereo_rcnn_b200.lib", fromlist=["load"]).load()
    assert L.sb_kitti_annotations_workspace_bytes(0, 5) == 0
    assert L.sb_kitti_annotations_workspace_bytes(1, 0) > 0
    off = torch.zeros(2, dtype=torch.int64, device="cuda")
    cal = torch.zeros(1, 25, dtype=torch.float64, device="cuda")
    hw = torch.tensor([[375, 1242]], dtype=torch.int32, device="cuda")
    n, st = torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(1, dtype=torch.int32, device="cuda")
    ws = torch.zeros(1024, dtype=torch.uint8, device="cuda")
    p = lambda t: ops.ptr(t)
    base = L.sb_launch_count()
    assert L.sb_kitti_annotations(None, None, p(off), p(cal), p(hw), 1, 0, p(ws), 0, None, p(n), p(st), None) == -22
    assert L.sb_kitti_annotations(None, None, p(off), p(cal), p(hw), 0, 0, p(ws), 1024, None, p(n), p(st), None) == -22
    assert L.sb_kitti_annotations(None, None, None, p(cal), p(hw), 1, 0, p(ws), 1024, None, p(n), p(st), None) == -22
    assert L.sb_kitti_annotations(None, None, p(off), p(cal), p(hw), 1, 3, p(ws), 1024, None, p(n), p(st), None) == -22
    assert L.sb_launch_count() == base
    assert L.sb_kitti_annotations(None, None, p(off), p(cal), p(hw), 1, 0, p(ws), 1024, None, p(n), p(st), None) == 0
    torch.cuda.synchronize()
    assert n.item() == 0 and st.item() == 0


# ------------------------------------------------------------------------------------------------------ end to end
FH, FW = 375, 1242


def frame(seed):
    rs = np.random.RandomState(seed)
    base = rs.randint(0, 256, (FH // 16 + 2, FW // 16 + 2, 3)).astype(np.float32)
    im = np.kron(base, np.ones((16, 16, 1), np.float32))[:FH, :FW] + rs.randn(FH, FW, 3) * 6
    return np.clip(im, 0, 255).astype(np.uint8)


def test_train_roidb_feeds_one_epoch_of_fit(tmp_path):
    from stereo_rcnn_b200.synth import make_state_dict
    pixels = {k: (frame(100 + k), frame(200 + k)) for k in range(2)}
    ids = synth.kitti_folder(str(tmp_path / "kitti"), 2, seed=8, sizes=((FH, FW),), frames=lambda k: pixels[k])
    roidb = KD.train_roidb(str(tmp_path / "kitti"), ids, "cuda")
    assert len(roidb) == 4 and [e["flipped"] for e in roidb] == [False, False, True, True]
    assert all(e["width"] == FW and e["height"] == FH for e in roidb)
    frames = lambda e: pixels[ids.index(e["image_id"])]
    # the ground truth of a step equals the oracle's on the oracle's roidb entry
    split = KD.Split(str(tmp_path / "kitti"), ids)
    o_out, o_n, _st = OA.split(*split.arrays())
    oracle_entries = split.entries(o_out, o_n)
    sd = make_state_dict(3)
    tr = TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, grad_scale=2.0 ** 12, seed=5)
    scale = 600.0 / FH
    inp = TR.StepInputs((FH, FW), scale, "cuda", max_rows=64)
    e = roidb[0]
    inp.load(e, *frames(e))
    tr.step_from_frames(inp)
    torch.cuda.synchronize()
    n = len(e["gt_classes"])
    words = TI.random_words(5, 0, 0, 64)
    pad = {k: np.concatenate([oracle_entries[0][k], np.zeros((64 - n,) + oracle_entries[0][k].shape[1:], np.float32)])
           for k in ("boxes_left", "boxes_right", "boxes_merge", "dim_orien", "kpts")}
    pad["gt_classes"] = np.concatenate([np.ones(n, np.int32), np.zeros(64 - n, np.int32)])
    want = TI.train_gt(pad, scale, inp.im_left.shape[3], words, n)
    for got, w in zip(inp.gt[:5], want[:5]):
        assert np.array_equal(got[0].cpu().numpy().view(np.uint32), w.view(np.uint32))
    assert int(inp.gt[5][0]) == want[5] > 0
    # one epoch of fit over the two images and their flips
    tr2 = TR.Trainer(E.StereoRCNNEngine(sd, "cuda", precision="fp16"), sd, grad_scale=2.0 ** 12, seed=5)
    save = tmp_path / "ck"
    save.mkdir()
    totals = TR.fit(tr2, roidb, frames, epochs=1, save_dir=str(save), log=lambda s: None)
    assert len(totals) == 4 and all(np.isfinite(totals))
    assert sorted(os.listdir(save)) == ["stereo_rcnn_1_3.pth"]
