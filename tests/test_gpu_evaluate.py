"""GPU: the test loop over a split with the calibration in device memory.

* sb_box_solve_devcalib / sb_dense_align_n_devcalib / sb_box_rectify_devcalib equal their host-calibrated siblings bit
  for bit at three calibrations (the goldens of tests/golden/calibration.npz), including the rows >= n and the
  workspace, which they leave as the siblings do;
* one capture of the three calls, replayed after each new calibration is written into the device buffer, equals the
  eager host-calibrated calls for that calibration;
* StereoPipeline.step_from_frames equals step_with_solver on prep_stereo_pair's blobs with host P2 / P3, at two frame
  shapes whose blobs have one shape but two scales;
* pipeline.evaluate writes the same files eagerly, from graphs at inflight 1 and at inflight 2, equal to
  kitti_result_lines of per-entry eager step_with_solver, captures one graph per (frame shape, slot) and refuses a
  directory that already holds results before any launch."""
import os

import numpy as np
import pytest
import torch

from stereo_rcnn_b200 import engine as E
from stereo_rcnn_b200 import ops as G
from stereo_rcnn_b200 import pipeline as PL
from stereo_rcnn_b200.synth import gen_rois, make_state_dict, synth_pair

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
CAL = np.load(os.path.join(HERE, "golden", "calibration.npz"))
NCAL = len(CAL["texts"])
TARGET = 160                                               # blob height of the small frames below
SHAPES = ((100, 330), (101, 333))                          # both -> 160x528 blobs, at scales 1.6 and 1.5842


def calib(i, div=1.0):
    """calibration i of the golden; div scales the image axes (f, cx, cy, tx) for frames `div` times smaller"""
    s = np.array([[1.0 / div], [1.0 / div], [1.0]])
    p = {k: CAL[k][i] * s for k in ("p0", "p1", "p2", "p3")}
    return G.Calibration(t_cam2_cam0_x=(p["p2"][0, 3] - p["p0"][0, 3]) / p["p2"][0, 0], **p)


def bits(t):
    t = t.detach().contiguous()
    return t.view(torch.int64) if t.element_size() == 8 else t.view(torch.int32)


def same(a, b):
    return a.shape == b.shape and torch.equal(bits(a), bits(b))


def c(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ------------------------------------------------------------------------------------- the _devcalib entry points
def solver_inputs():
    """the detections of tests/golden/box_solver.npz scattered over 80 RoI rows, as test_gpu_round2 builds them"""
    g = np.load(os.path.join(HERE, "golden", "box_solver.npz"))
    n, R, nc = len(g["alpha"]), 80, 2
    rs = np.random.RandomState(11)
    scores = np.zeros((R, nc), np.float32)
    pbl, pbr = np.zeros((R, 8), np.float32), np.zeros((R, 8), np.float32)
    do, pk = np.zeros((R, 10), np.float32), np.zeros((R, 5), np.float32)
    rows = rs.permutation(R)[:n]
    sc = np.sort(rs.rand(n).astype(np.float32) * 0.9 + 0.06)[::-1]
    for j, r in enumerate(rows):
        scores[r, 1] = sc[j]
        pbl[r, 4:8], pbr[r, 4:8] = g["box_left"][j], g["box_right"][j]
        do[r, 5:8] = g["dim"][j]
        do[r, 8], do[r, 9] = np.sin(g["alpha"][j]), np.cos(g["alpha"][j])
        pk[r] = g["kpts"][j]
    keep = np.zeros(R, np.int32)
    keep[:n] = rows
    shape = tuple(int(v) for v in g["im_shape"])[:2]
    args = (c(scores), c(pbl), c(pbr), c(do), c(pk), c(keep), c(np.array([n], np.int32)))
    return args, shape, g["disparity"]


def solve_chain(args, shape, p2, p3, iml, imr, scale):
    """box_solve -> dense_align_n -> box_rectify, host (p2, p3) or device (p2 = [24], p3 = None) calibration"""
    inferred = G.infer_boundary(args[1], args[5], args[6], shape[1], col_offset=4)
    boxes_all, kpts_all, poses_all, src, n = G.box_solve(*args, shape, p2, p3, inferred=inferred)
    c4 = p2 if p3 is None else G.calib_vec(p2, p3)
    st, dis = G.dense_align_n(c4, scale, iml, imr, boxes_all, kpts_all, poses_all, n)
    final = G.box_rectify(boxes_all, kpts_all, poses_all, st, dis, n, shape, p2, p3)
    return dict(boxes_all=boxes_all, kpts_all=kpts_all, poses_all=poses_all, src=src, n=n, status=st, best_dis=dis,
                final=final)


@pytest.mark.parametrize("i", range(NCAL))
def test_box_solve_and_rectify_devcalib_bit_identical(i):
    args, shape, disparity = solver_inputs()
    cal = calib(i)
    dc = G.device_calib(cal.p2, cal.p3, "cuda")
    host = G.box_solve(*args, shape, cal.p2, cal.p3)
    dev = G.box_solve(*args, shape, dc, None)
    for k, a, b in zip(("boxes_all", "kpts_all", "poses_all", "src_index", "n"), host, dev):
        assert same(a, b), k
    n = int(host[4][0])
    assert n >= 8
    succ = torch.ones(80, device="cuda")
    succ[3] = 0.0
    dis = torch.zeros(80, device="cuda")
    dis[:n] = c(disparity[:n].astype(np.float32))
    fh = G.box_rectify(*host[:3], succ, dis, host[4], shape, cal.p2, cal.p3)
    fd = G.box_rectify(*dev[:3], succ, dis, dev[4], shape, dc, None)
    assert same(fh, fd)
    assert (fh[:n, 0] == 1).sum() == n - 1 and (fh[n:, 0] == 0).all()


def _dense_case(cap, seed, p2):
    H0, W0, scale = 375, 1242, 0.8                         # rows in original-image units, 300x994 network blobs
    iml, imr = synth_pair(300, 994, seed, shift=9)
    box, kp, pose = gen_rois(cap, seed, p2=p2)
    boxes_all = np.zeros((cap, 5), np.float32)
    poses_all = np.zeros((cap, 8), np.float32)
    boxes_all[:, :4], poses_all[:, :7] = box, pose
    return c(iml), c(imr), c(boxes_all), c(kp), c(poses_all), scale


@pytest.mark.parametrize("cap", [24, 300])
@pytest.mark.parametrize("i", range(NCAL))
def test_dense_align_n_devcalib_bit_identical(cap, i):
    """strip path (cap 24) and materialised path (cap 300); n_dev 0, partial and full; the workspace of both calls,
    primed with one byte pattern, ends byte-identical (untouched at n_dev 0)"""
    cal = calib(i)
    dc = G.device_calib(cal.p2, cal.p3, "cuda")
    iml, imr, boxes_all, kp, poses_all, scale = _dense_case(cap, 40 + i, cal.p2)
    for n in (0, cap // 3, cap):
        n_dev = torch.tensor([n], dtype=torch.int32, device="cuda")
        outs, wss = [], []
        for c4 in (G.calib_vec(cal.p2, cal.p3), dc):
            own = G.WorkspaceOwner()
            with G.workspace_owner(own):
                nb = G._l.load().sb_dense_align_workspace_bytes(300, 994, cap)
                ws = G.workspace(nb, iml.device, "dense_align")
                ws.fill_(0x5A)
                outs.append(G.dense_align_n(c4, scale, iml, imr, boxes_all, kp, poses_all, n_dev))
            wss.append(ws)
        torch.cuda.synchronize()
        (sh, bh), (sd, bd) = outs
        assert same(sh, sd) and same(bh, bd), n
        assert torch.equal(wss[0], wss[1]), n
        assert (sh[n:] == 0).all() and (bh[n:] == 0).all()
        if n == 0:
            assert (wss[1] == 0x5A).all()
        else:
            assert (sh[:n] > 0).any()


def test_captured_chain_replayed_with_new_calibrations():
    """one graph of box_solve -> dense_align_n -> box_rectify on a device calibration; before each replay another
    calibration is written into the buffer; every replay equals the eager host-calibrated chain"""
    args, shape, _ = solver_inputs()
    iml, imr = (c(a) for a in synth_pair(300, 994, 7, shift=9))
    dc = torch.zeros(24, dtype=torch.float64, device="cuda")
    own = G.WorkspaceOwner()
    with G.workspace_owner(own):
        cal = calib(0)
        dc.copy_(G.device_calib(cal.p2, cal.p3, "cuda"))
        runner = E.GraphRunner(lambda: solve_chain(args, shape, dc, None, iml, imr, 0.8), [], warmup=1)
    seen = set()
    for i in (1, 2, 0, 2):
        cal = calib(i)
        dc.copy_(G.device_calib(cal.p2, cal.p3, "cuda"))
        got = runner()
        with G.workspace_owner(G.WorkspaceOwner()):
            ref = solve_chain(args, shape, cal.p2, cal.p3, iml, imr, 0.8)
        torch.cuda.synchronize()
        for k in ref:
            assert same(got[k], ref[k]), (i, k)
        assert int(ref["n"][0]) > 0
        seen.add(float(ref["final"][:, 8].sum()))
    assert len(seen) == NCAL                               # the calibrations give different depths


# ---------------------------------------------------------------------------------- pipeline and the test loop
def frame(h, w, seed):
    rs = np.random.RandomState(seed)
    base = rs.randint(0, 256, (h // 8 + 2, w // 8 + 2, 3)).astype(np.float32)
    im = np.kron(base, np.ones((8, 8, 1), np.float32))[:h, :w] + rs.randn(h, w, 3) * 6
    return np.clip(im, 0, 255).astype(np.uint8)


def frame_pair(h, w, seed, shift=5):
    left = frame(h, w + shift, seed)
    return np.ascontiguousarray(left[:, shift:]), np.ascontiguousarray(left[:, :w])


@pytest.fixture(scope="module")
def pipe():
    sd = make_state_dict(3)
    b = sd["RCNN_cls_score.bias"].clone()
    b[1] += 4.0                                            # Car scores well above eval_thresh
    sd["RCNN_cls_score.bias"] = b
    return PL.StereoPipeline(sd, torch.device("cuda"), throughput=True)


def eager_reference(pipe, left, right, cal, hw):
    """step_with_solver on prep_stereo_pair's blobs with host P2 / P3 and the fp32 scale of the frame shape"""
    scale = PL.frame_scale(hw, TARGET)
    flip = torch.zeros(1, dtype=torch.int32, device="cuda")
    bl, br = G.prep_stereo_pair(c(left), c(right), scale, flip, rgb_input=True)
    with G.workspace_owner(G.WorkspaceOwner()):
        return pipe.step_with_solver(bl[None], br[None], cal.p2, cal.p3, hw, scale=np.float32(scale))


def test_step_from_frames_equals_step_with_solver(pipe):
    keys = ("record", "nkeep", "keep", "n_solved", "poses_all", "status", "best_dis", "final")  # keep: first nkeep
    blobs = set()
    for j, hw in enumerate(SHAPES):
        left, right = frame_pair(*hw, seed=60 + j)
        cal = calib(j, div=3.75)
        inp = PL.EvalInputs(hw, PL.frame_scale(hw, TARGET), "cuda")
        inp.load(left, right, cal)
        with G.workspace_owner(G.WorkspaceOwner()):
            got = pipe.step_from_frames(inp)
        ref = eager_reference(pipe, left, right, cal, hw)
        torch.cuda.synchronize()
        for k in keys:
            assert same(got[k], ref[k]) if k != "keep" else same(got[k][:got["nkeep"][0]], ref[k][:ref["nkeep"][0]]), (hw, k)
        assert int(ref["n_solved"][0]) > 0
        blobs.add(tuple(inp.im_left.shape))
    assert len(blobs) == 1                                 # one blob shape, two scales: im_info keyed by scale


def split(n=8):
    """entries over two frame shapes (A A B B ...: each shape meets both slots at inflight 2) and three
    calibrations"""
    entries = []
    for k in range(n):
        hw = SHAPES[(k // 2) % 2]
        entries.append(dict(image_id="%06d" % (3 * k), hw=hw, seed=100 + k, cal=k % NCAL))
    return entries


def read_dir(d):
    return {f: open(os.path.join(d, f)).read() for f in sorted(os.listdir(d))}


def test_evaluate_eager_and_graphs_write_the_reference_files(pipe, tmp_path):
    entries = split(8)
    frames = lambda e: frame_pair(*e["hw"], seed=e["seed"])
    cal = lambda e: calib(e["cal"], div=3.75)
    runs = {}
    for tag, inflight, use_graph in (("eager", 1, False), ("graph1", 1, True), ("graph2", 2, True)):
        out = str(tmp_path / tag)
        summary = PL.evaluate(pipe, entries, frames, cal, out, inflight=inflight, use_graph=use_graph,
                              target_size=TARGET, log=lambda s: None)
        assert summary["images"] == len(entries)
        assert summary["graphs"] == (len(SHAPES) * inflight if use_graph else 0), (tag, summary)
        runs[tag] = read_dir(os.path.join(out, "data"))
        assert summary["files"] == len(runs[tag]) and summary["lines"] == sum(
            v.count("\n") for v in runs[tag].values())
    assert runs["eager"] == runs["graph1"] == runs["graph2"]
    expect, with_lines = {}, 0
    for e in entries:
        left, right = frames(e)
        ce = cal(e)
        ref = eager_reference(pipe, left, right, ce, e["hw"])
        lines = G.kitti_result_lines(ref["final"], ce.t_cam2_cam0_x)
        if lines:
            expect[e["image_id"] + ".txt"] = "".join(lines)
            with_lines += 1
    assert runs["eager"] == expect
    assert 2 * with_lines >= len(entries), with_lines
    # every image gets a file with empty_files, the same text where there are lines
    out = str(tmp_path / "all")
    PL.evaluate(pipe, entries, frames, cal, out, target_size=TARGET, empty_files=True, log=lambda s: None)
    got = read_dir(os.path.join(out, "data"))
    assert sorted(got) == sorted(e["image_id"] + ".txt" for e in entries)
    assert all(got[k] == expect.get(k, "") for k in got)
    # a second run into a directory with results is refused before any launch or read
    n0 = G.launch_count()

    def boom(e):
        raise AssertionError("an entry was read")
    with pytest.raises(FileExistsError):
        PL.evaluate(pipe, entries, boom, boom, str(tmp_path / "graph2"), target_size=TARGET)
    assert G.launch_count() == n0
    assert read_dir(os.path.join(str(tmp_path / "graph2"), "data")) == runs["graph2"]
