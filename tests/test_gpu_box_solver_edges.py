"""GPU: the box solver stage (csrc/box_solver.cu) at its edges, through the C ABI.

* `sb_infer_boundary` on every occlusion pattern of tests/golden/box_solver_edges.npz (minted from the reference's own
  kitti_utils.infer_boundary), bit for bit, through scattered `keep` rows, with column offsets 4 and 8;
* the keypoint border fix-up of test_net.py:263-266 at, just below and just above its float32 threshold;
* the status rules and the score test against the reference's decisions in the golden, plus two rejections: z > 100
  and a non-finite solve;
* the ordered compaction: num from 0 to 512 and beyond, a cap below the solved count, several classes;
* the solver's branches (viewpoints, keypoint types, border switches) on generated problems, against the oracle's
  restatement of the reference's gradient and objective and against the host-compiled solver core;
* `sb_box_rectify`: several CTAs, rows it must skip, the fixed depth;
* the `_devcalib` entry points, bit-identical to the host-calibrated ones on the same cases.

Output buffers are filled with NaN bit patterns and have guard rows past `cap`, so a row the kernel must not write is
checked to be untouched.
"""
import ctypes
import math as m
import os
import subprocess

import numpy as np
import pytest
import torch

from oracle import box_solver as BS
from stereo_rcnn_b200 import lib as _l
from stereo_rcnn_b200 import ops as G
from stereo_rcnn_b200.lib import check, ptr, stream_ptr

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
F32 = np.float32
SENT32 = 0x7FBADBAD                    # a NaN bit pattern: a row the kernel must not write
SENT64 = 0x7FF4DEADBEEF7777
H, W = 375, 1242
GUARD = 8                              # output rows past `cap`


@pytest.fixture(scope="module")
def gold():
    return np.load(os.path.join(HERE, "golden", "box_solver_edges.npz"))


@pytest.fixture(scope="module")
def cal():
    return np.load(os.path.join(HERE, "golden", "calibration.npz"))


@pytest.fixture(scope="module")
def host_lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("boxhost") / "libboxhost.so")
    subprocess.check_call(["g++", "-O2", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests/tools/box_solver_host.cpp")])
    return ctypes.CDLL(so)


def c(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def sent_f32(*shape):
    return torch.full(shape, SENT32, dtype=torch.int32, device="cuda").view(torch.float32)


def sent_i32(*shape):
    return torch.full(shape, SENT32, dtype=torch.int32, device="cuda")


def sent_f64(*shape):
    return torch.full(shape, SENT64, dtype=torch.int64, device="cuda").view(torch.float64)


def bits(a):
    a = np.ascontiguousarray(a)
    return a.view({4: np.uint32, 8: np.uint64}[a.dtype.itemsize])


def untouched(a):
    return (bits(a) == (SENT32 if a.dtype.itemsize == 4 else SENT64)).all()


def alpha_of(sc):
    """test_net.py:292: math.atan2 of the two float32 elements; the kernel's atan2 of the same values in double"""
    return m.atan2(float(sc[0]), float(sc[1]))


# ------------------------------------------------------------------ detections and raw launches
def det(box_l, box_r, kp, sc, dim, score=0.9):
    return dict(bl=np.asarray(box_l, F32), br=np.asarray(box_r, F32), kp=np.asarray(kp, F32), sc=np.asarray(sc, F32),
                dim=np.asarray(dim, F32), score=F32(score))


def golden_det(g, name, **edit):
    i = [str(n) for n in g["st_name"]].index(name)
    d = det(g["st_box_left"][i], g["st_box_right"][i], g["st_kpts"][i], g["st_sincos"][i], g["st_dim"][i],
            g["st_score"][i])
    for k, v in edit.items():
        d[k] = v
    return d


def layout(cls_dets, R, nc=2, seed=0):
    """RoI-layout tensors with the detections of each class in `cls_dets` ({cls: [det]}, equal lengths) on scattered
    rows; every value the kernel must not read is NaN.  -> tensors, keep (device, the full permutation), rows"""
    rs = np.random.RandomState(seed)
    n = len(next(iter(cls_dets.values())))
    perm = rs.permutation(R).astype(np.int32)
    rows = perm[:n]
    t = dict(scores=np.full((R, nc), np.nan, F32), bl=np.full((R, 4 * nc), np.nan, F32),
             br=np.full((R, 4 * nc), np.nan, F32), do=np.full((R, 5 * nc), np.nan, F32), kp=np.full((R, 5), np.nan, F32))
    for cls, dets in cls_dets.items():
        for j, r in enumerate(rows):
            d = dets[j]
            t["scores"][r, cls] = d["score"]
            t["bl"][r, 4 * cls:4 * cls + 4] = d["bl"]
            t["br"][r, 4 * cls:4 * cls + 4] = d["br"]
            t["do"][r, 5 * cls:5 * cls + 3] = d["dim"]
            t["do"][r, 5 * cls + 3:5 * cls + 5] = d["sc"]
            t["kp"][r] = d["kp"]            # keypoints are class-agnostic [R,5]
    return {k: c(v) for k, v in t.items()}, c(perm), rows


def solve_raw(lay, keep, num, cls, calib, cap, inferred=None, eval_thresh=0.05):
    """sb_box_solve (calib = (p2, p3)) or sb_box_solve_devcalib (calib = device tensor [24]) into sentinel-filled
    buffers of cap + GUARD rows -> numpy dict"""
    L = _l.load()
    R, nc = lay["scores"].shape
    o = dict(boxes=sent_f32(cap + GUARD, 5), kpts=sent_f32(cap + GUARD, 5), poses=sent_f32(cap + GUARD, 8),
             src=sent_i32(cap + GUARD), n=sent_i32(2))
    head = [ptr(lay[k]) for k in ("scores", "bl", "br", "do", "kp")] + [ptr(keep), ptr(c(np.array([num], np.int32))),
                                                                         ptr(inferred), nc, cls, H, W]
    tail = [eval_thresh, cap] + [ptr(o[k]) for k in ("boxes", "kpts", "poses", "src", "n")] + [stream_ptr()]
    if torch.is_tensor(calib):
        check(L.sb_box_solve_devcalib(*head, ptr(calib), *tail), "sb_box_solve_devcalib")
    else:
        check(L.sb_box_solve(*head, G._p34(calib[0]), G._p34(calib[1]), *tail), "sb_box_solve")
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}


def solve_both(lay, keep, num, cls, p2, p3, cap, **kw):
    """host-calibrated and _devcalib launches must agree bit for bit -> the host-calibrated result"""
    a = solve_raw(lay, keep, num, cls, (p2, p3), cap, **kw)
    b = solve_raw(lay, keep, num, cls, G.device_calib(p2, p3, "cuda"), cap, **kw)
    for k in a:
        assert np.array_equal(bits(a[k]), bits(b[k])), "devcalib differs in %s" % k
    return a


def check_compacted(out, expect_rows, cap, dets_by_row=None):
    """n_out, src_index in kept order, rows past the written ones untouched"""
    k = min(len(expect_rows), cap)
    assert int(out["n"][0]) == k and untouched(out["n"][1:])
    np.testing.assert_array_equal(out["src"][:k], np.asarray(expect_rows[:k], np.int32))
    for key in ("boxes", "kpts", "poses", "src"):
        assert untouched(out[key][k:]), key
    if dets_by_row is not None:
        for q in range(k):
            d = dets_by_row[int(out["src"][q])]
            np.testing.assert_array_equal(out["boxes"][q], np.r_[d["bl"], d["score"]].astype(F32))
            np.testing.assert_array_equal(out["poses"][q, 3:6], d["dim"])
            assert out["poses"][q, 7] == F32(alpha_of(d["sc"]))
            assert np.isfinite(out["poses"][q]).all() and out["poses"][q, 2] <= 100


# ------------------------------------------------------------------ infer_boundary
def ib_raw(buf, coff, keep, num, im_w, out):
    L = _l.load()
    check(L.sb_infer_boundary(ptr(buf), buf.shape[1], coff, ptr(keep), ptr(c(np.array([num], np.int32))), im_w,
                              ptr(out), stream_ptr()), "sb_infer_boundary")
    torch.cuda.synchronize()
    return out.cpu().numpy()


def test_infer_boundary_golden_patterns(gold):
    g = gold
    off = g["ib_offsets"]
    for p, name in enumerate(g["ib_names"]):
        b, ref = g["ib_boxes"][off[p]:off[p + 1]], g["ib_left_right"][off[p]:off[p + 1]]
        n, im_w = len(b), int(g["ib_im_w"][p])
        for seed, coff in ((p, 4), (p + 1000, 8)):
            rs = np.random.RandomState(seed)
            R = n + 5
            buf = (rs.rand(R, coff + 5) * 50).astype(F32)            # other rows / columns hold unrelated boxes
            perm = rs.permutation(R).astype(np.int32)
            buf[perm[:n], coff:coff + 4] = b
            got = ib_raw(c(buf), coff, c(perm), n, im_w, sent_f32(R, 2))
            assert np.array_equal(bits(got[:n]), bits(ref)), "%s (col_offset %d)" % (name, coff)
            assert untouched(got[n:]), name
    buf = c(np.ones((4, 8), F32))
    assert untouched(ib_raw(buf, 4, c(np.arange(4, dtype=np.int32)), 0, W, sent_f32(4, 2)))


# ------------------------------------------------------------------ border fix-up
def test_border_fixup_threshold(gold, cal):
    """kp4 - kp3 < 0.5 * (i1 - i0), all in float32 as torch computes it: equal does not replace, one float below does"""
    g = gold
    p2, p3 = cal["p2"][0], cal["p3"][0]
    base = golden_det(g, "kp_at")
    dets, inf = [], []
    for i0, i1, k3 in ((100.0, 140.0, 50.0), (1.8082901, 8.0, 1.0), (300.25, 351.0, 7.5)):
        half = F32(0.5) * (F32(i1) - F32(i0))
        k4_at = F32(F32(k3) + half)
        while F32(k4_at - F32(k3)) >= half:          # the smallest kp4 whose float32 difference reaches the bound
            k4_at = np.nextafter(k4_at, F32(0))
        while not F32(k4_at - F32(k3)) >= half:
            k4_at = np.nextafter(k4_at, F32(1e9))
        for k4 in (np.nextafter(k4_at, F32(0)), k4_at, np.nextafter(k4_at, F32(1e9))):
            kp = base["kp"].copy()
            kp[3], kp[4] = F32(k3), k4
            dets.append(golden_det(g, "kp_at", kp=kp))
            inf.append([i0, i1])
    n, R = len(dets), len(dets) + 3
    lay, keep, rows = layout({1: dets}, R)
    inferred = np.full((R, 2), np.nan, F32)
    inferred[:n] = np.asarray(inf, F32)                # indexed by kept position, as sb_infer_boundary writes it
    for with_inf in (True, False):
        out = solve_both(lay, keep, n, 1, p2, p3, R, inferred=c(inferred) if with_inf else None)
        check_compacted(out, list(rows), R)
        for q in range(n):
            kp = dets[q]["kp"].copy()
            i0, i1 = F32(inferred[q, 0]), F32(inferred[q, 1])
            replaced = with_inf and F32(kp[4] - kp[3]) < F32(0.5) * F32(i1 - i0)
            assert replaced == (with_inf and q % 3 == 0), q
            if replaced:
                kp[3:5] = (i0, i1)
            assert np.array_equal(bits(out["kpts"][q]), bits(kp)), q


# ------------------------------------------------------------------ status rules and score
def test_status_rules_and_score_vs_reference(gold, cal):
    """every golden status case in one launch: solved exactly where the reference solves.  On top: the score test at
    float32(0.05), a far box (z > 100) and a detection with identical left and right boxes (disparity 0, so the start
    point and the solve are not finite).  The reference would append a NaN pose for the last one; the kernel drops it
    (DESIGN.md §(f)1)."""
    g = gold
    p2, p3 = cal["p2"][0], cal["p3"][0]
    names = [str(n) for n in g["st_name"]]
    dets = [golden_det(g, nm) for nm in names]
    solved = [int(s) == 1 for s in g["st_status"]]
    for v, ok in zip(g["score_values"], g["score_pass"]):
        dets.append(golden_det(g, "kp_at", score=F32(v)))
        solved.append(bool(ok))
        names.append("score_%r" % float(v))
    d0 = golden_det(g, "kp_at")
    dets.append(golden_det(g, "kp_at", br=d0["bl"].copy()))
    solved.append(False)
    names.append("zero_disparity")
    n = len(dets)
    for R, cap in ((n + 6, n), (n, 3)):
        lay, keep, rows = layout({1: dets}, R, seed=R)
        out = solve_both(lay, keep, n, 1, p2, p3, cap)
        expect = [int(rows[j]) for j in range(n) if solved[j]]
        got = [names[list(rows).index(int(r))] for r in out["src"][:int(out["n"][0])]]
        exp_names = [names[j] for j in range(n) if solved[j]][:cap]
        assert got == exp_names, "solved %s, the reference solves %s" % (got, exp_names)
        check_compacted(out, expect, cap, {int(r): dets[j] for j, r in enumerate(rows)})


# ------------------------------------------------------------------ ordered compaction
def compaction_dets(g, n, seed):
    """n detections, a random third of them rejected by the score or by the box height rule (both per class; the
    keypoints are shared by the classes) -> dets, solved flags"""
    rs = np.random.RandomState(seed)
    dets, solved = [], []
    for j in range(n):
        mode = rs.randint(6)
        d = golden_det(g, "kp_at", score=F32(0.06 + 0.9 * rs.rand()))
        if mode == 0:
            d["score"] = F32(0.05)
        elif mode == 1:
            d["bl"] = d["bl"].copy(); d["bl"][3] = d["bl"][1] + F32(9.5)
        dets.append(d)
        solved.append(mode > 1)
    return dets, solved


@pytest.mark.parametrize("num", [0, 1, 31, 32, 33, 64, 300, 511, 512])
def test_ordered_compaction(gold, cal, num):
    g = gold
    p2, p3 = cal["p2"][1], cal["p3"][1]
    n = max(num, 1)
    dets, solved = compaction_dets(g, n, num)
    R = n + 7
    lay, keep, rows = layout({1: dets}, R, seed=num)
    by_row = {int(r): dets[j] for j, r in enumerate(rows)}
    expect = [int(rows[j]) for j in range(num) if solved[j]]
    full = solve_both(lay, keep, num, 1, p2, p3, R)
    check_compacted(full, expect, R, by_row)
    if expect:          # every solved row solves the same problem: the same bits
        assert (bits(full["poses"][:len(expect)]) == bits(full["poses"][0])).all()
    for cap in sorted({1, len(expect) // 2, len(expect) - 1}):
        if not 1 <= cap < len(expect):             # cap >= 1 is an argument check of the entry points
            continue
        out = solve_both(lay, keep, num, 1, p2, p3, cap)
        check_compacted(out, expect, cap, by_row)
        for key in ("boxes", "kpts", "poses", "src"):
            assert np.array_equal(bits(out[key][:cap]), bits(full[key][:cap])), key


def test_compaction_beyond_512_detections(gold, cal):
    """one CTA of 512 threads: of num > 512 kept detections only the first 512 are considered (DESIGN.md §(f)1)"""
    g = gold
    p2, p3 = cal["p2"][0], cal["p3"][0]
    n = 600
    dets, solved = compaction_dets(g, n, 5)
    lay, keep, rows = layout({1: dets}, n + 4, seed=3)
    out = solve_both(lay, keep, n, 1, p2, p3, n)
    check_compacted(out, [int(rows[j]) for j in range(512) if solved[j]], n,
                    {int(r): dets[j] for j, r in enumerate(rows)})


@pytest.mark.parametrize("cls", [1, 2])
def test_compaction_multi_class(gold, cal, cls):
    """n_classes = 3: each class reads its own columns of scores, boxes and dim_orien"""
    g = gold
    p2, p3 = cal["p2"][2], cal["p3"][2]
    n = 70
    d1, s1 = compaction_dets(g, n, 11)
    d2, s2 = compaction_dets(g, n, 12)
    lay, keep, rows = layout({1: d1, 2: d2}, n + 9, nc=3, seed=4)
    dets, solved = (d1, s1) if cls == 1 else (d2, s2)
    out = solve_both(lay, keep, n, cls, p2, p3, n)
    check_compacted(out, [int(rows[j]) for j in range(n) if solved[j]], n, {int(r): dets[j] for j, r in enumerate(rows)})


# ------------------------------------------------------------------ solver branches
def gen_problems(p2, p3, seed, n_cand=6000, per_bin=3):
    """generated problems that reach every branch of the solver set-up, `per_bin` of each -> dets, tags"""
    rs = np.random.RandomState(seed)
    f, cx, cy = p2[0, 0], p2[0, 2], p2[1, 2]
    bl = (p2[0, 3] - p3[0, 3]) / f
    counts, dets, tags = {}, [], []
    for _ in range(n_cand):
        z = rs.uniform(4, 50); x = rs.uniform(-0.8 * z, 0.8 * z); y = rs.uniform(-0.5, 2.2)
        w, h, l = rs.uniform([1.4, 1.2, 3.0], [2.0, 3.0, 5.0]); th = rs.uniform(-np.pi, np.pi); kt = rs.randint(4)
        cs, sn = np.cos(th), np.sin(th)
        xs = np.array([-w / 2, -w / 2, w / 2, w / 2] * 2); ys = np.array([0, 0, 0, 0, -h, -h, -h, -h])
        zs = np.array([-l / 2, l / 2, l / 2, -l / 2] * 2)
        X, Y, Z = cs * xs + sn * zs + x, ys + y, -sn * xs + cs * zs + z
        if Z.min() < 1:
            continue
        u, v, ur = f * X / Z + cx, f * Y / Z + cy, f * (X - bl) / Z + cx
        box_l = np.array([u.min(), v.min(), u.max(), v.max()]) + rs.randn(4) * 0.3
        box_r = np.array([ur.min(), v.min(), ur.max(), v.max()]) + rs.randn(4) * 0.3
        box_l = np.clip(box_l, 0, [W - 1, H - 1, W - 1, H - 1]).astype(F32)
        box_r = np.clip(box_r, 0, [W - 1, H - 1, W - 1, H - 1]).astype(F32)
        vw, vl = [(-w, -l), (-w, l), (w, l), (w, -l)][kt]
        uk = f * (x + cs * vw / 2 + sn * vl / 2) / (z - sn * vw / 2 + cs * vl / 2) + cx + rs.randn() * 0.3
        kp = np.array([uk, kt, 0.9, box_l[0], box_l[2]], F32)
        alpha = th - m.pi / 2 + m.atan2(-x, z)
        sc = np.array([np.sin(alpha), np.cos(alpha)], F32)
        dim = (np.array([w, h, l]) + rs.randn(3) * 0.05).astype(F32)
        if BS.rejected(box_l, kp) or box_l[0] - box_r[0] < 1:
            continue
        pb = BS.Problem((H, W), p2, p3, alpha_of(sc), dim.astype(np.float64), box_l.astype(np.float64),
                        box_r.astype(np.float64), kp.astype(np.float64))
        t = {("trunc" if pb.truncation else "kpt", BS.bb2viewpoint(pb.alpha))}
        if not pb.truncation:
            t.add(("kpt_type", kt))
        if pb.truncation and box_l[2] > W - 20 and pb.on["urr"]:
            t.add("right_trunc_r7")
        if pb.truncation and pb.on["ulr"]:
            t.add("r6_live")
        if not pb.on["vt"]:
            t.add("vt<10")
        if not pb.on["vb"]:
            t.add("vb>h-10")
        if abs(pb.alpha) > m.pi:
            t.add("|alpha|>180")
        if not any(counts.get(k, 0) < per_bin for k in t):
            continue
        for k in t:
            counts[k] = counts.get(k, 0) + 1
        dets.append(det(box_l, box_r, kp, sc, dim))
        tags.append(t)
    return dets, tags


def host_solve(host_lib, p2, p3, d):
    P = lambda a: np.ascontiguousarray(a, np.float64)
    args = [P(p2), P(p3), P(d["dim"]), P(d["bl"]), P(d["br"]), P(d["kp"])]
    s, info = np.zeros(4), np.zeros(4)
    dp = lambda a: a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))
    host_lib.box_solve_host(H, W, dp(args[0]), dp(args[1]), ctypes.c_double(alpha_of(d["sc"])), dp(args[2]), dp(args[3]),
                            dp(args[4]), dp(args[5]), 0, ctypes.c_double(0.0), dp(s), dp(info))
    return s


def test_solver_branches_vs_oracle(cal, host_lib):
    all_tags, worse, n_tot, dstate = {}, 0, 0, []
    for ci in range(len(cal["p2"])):
        p2, p3 = cal["p2"][ci], cal["p3"][ci]
        dets, tags = gen_problems(p2, p3, 100 + ci)
        for t in tags:
            for k in t:
                all_tags[k] = all_tags.get(k, 0) + 1
        n = len(dets)
        assert n <= 512
        lay, keep, rows = layout({1: dets}, n + 3, seed=ci)
        out = solve_both(lay, keep, n, 1, p2, p3, n)
        check_compacted(out, list(rows), n, {int(r): dets[j] for j, r in enumerate(rows)})
        for q in range(n):
            d = dets[q]
            pb = BS.Problem((H, W), p2, p3, alpha_of(d["sc"]), d["dim"].astype(np.float64), d["bl"].astype(np.float64),
                            d["br"].astype(np.float64), d["kp"].astype(np.float64))
            s = out["poses"][q, [0, 1, 2, 6]].astype(np.float64)
            assert np.abs(pb.gradient(s)).max() < 1e-5, (ci, q, tags[q], pb.gradient(s))
            st, sref = BS.solve_x_y_z_theta_from_kpt((H, W), p2, p3, alpha_of(d["sc"]), d["dim"], d["bl"], d["br"], d["kp"])

            def f_eff(st_):
                r, _ = pb.residuals(st_)
                r = r.copy(); r[2] /= np.sqrt(2.0)
                return float(np.dot(r, r))
            worse += f_eff(s) > f_eff(np.asarray(sref)) * (1 + 1e-6) + 1e-12
            n_tot += 1
            hs = host_solve(host_lib, p2, p3, d)
            dstate.append(np.abs(s - hs.astype(F32).astype(np.float64)) / np.maximum(np.abs(hs), 1.0))
    dstate = np.array(dstate)
    print("branch counts:", sorted(((str(k), v) for k, v in all_tags.items())))
    print("problems %d; objective above Newton-CG's in %d" % (n_tot, worse))
    print("|device - float32(host)| / max(|host|, 1) per state: median %.3g, 99th pct %.3g, max %.3g; exact in %.1f %%"
          % (np.median(dstate), np.percentile(dstate, 99), dstate.max(), 100.0 * (dstate == 0).mean()))
    for path in ("kpt", "trunc"):
        for vp in range(8):
            assert all_tags.get((path, vp), 0) > 0, (path, vp)
    for kt in range(4):
        assert all_tags.get(("kpt_type", kt), 0) > 0, kt
    for k in ("right_trunc_r7", "r6_live", "vt<10", "vb>h-10", "|alpha|>180"):
        assert all_tags.get(k, 0) > 0, k
    assert worse <= 0.1 * n_tot
    # H100 80GB HBM3: 99.1 % of the states are bit-identical to the host core's, the rest one float32 ulp apart
    # (max 1.18e-7 relative), from the last bit of the device's fp64 math functions; the bar is two ulps
    assert dstate.max() <= 2.4e-7


# ------------------------------------------------------------------ rectify
def rectify_raw(t, n, cap, calib, alloc):
    L = _l.load()
    out = sent_f64(alloc, 13)
    head = [ptr(t[k]) for k in ("boxes", "kpts", "poses", "succ", "dis")] + [ptr(c(np.array([n], np.int32))), cap, H, W]
    if torch.is_tensor(calib):
        check(L.sb_box_rectify_devcalib(*head, ptr(calib), ptr(out), stream_ptr()), "sb_box_rectify_devcalib")
    else:
        check(L.sb_box_rectify(*head, G._p34(calib[0]), G._p34(calib[1]), ptr(out), stream_ptr()), "sb_box_rectify")
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("n", [0, 300])
def test_rectify(cal, n):
    p2, p3 = cal["p2"][1], cal["p3"][1]
    cap = 400
    dets, _ = gen_problems(p2, p3, 7, per_bin=12)
    rs = np.random.RandomState(n)
    pick = rs.randint(len(dets), size=cap)
    boxes = np.stack([np.r_[dets[j]["bl"], F32(0.1 + 0.8 * rs.rand())] for j in pick]).astype(F32)
    kpts = np.stack([dets[j]["kp"] for j in pick])
    f = p2[0, 0]
    bl = (p2[0, 3] - p3[0, 3]) / f
    poses = np.zeros((cap, 8), F32)
    dis = np.zeros(cap, F32)
    for q, j in enumerate(pick):
        d = dets[j]
        z = f * bl / max(float(d["bl"][0] + d["bl"][2] - d["br"][0] - d["br"][2]) / 2, 1.0)
        poses[q, 3:6], poses[q, 7] = d["dim"], F32(alpha_of(d["sc"]))
        dis[q] = F32(f * bl / z + rs.randn() * 0.3)
    succ = np.ones(cap, F32)
    succ[rs.rand(cap) < 0.3] = 0.0
    succ[rs.rand(cap) < 0.1] = -1.0
    succ[rs.rand(cap) < 0.1] = np.nan
    t = dict(boxes=c(boxes), kpts=c(kpts), poses=c(poses), succ=c(succ), dis=c(dis))
    out = rectify_raw(t, n, cap, (p2, p3), cap + GUARD)
    assert np.array_equal(bits(out), bits(rectify_raw(t, n, cap, G.device_calib(p2, p3, "cuda"), cap + GUARD)))
    assert untouched(out[n:])
    for q in range(n):
        if not succ[q] > 0:
            assert out[q, 0] == 0 and untouched(out[q, 1:]), q
            continue
        assert out[q, 0] == 1 and out[q, 1] == float(boxes[q, 4])
        np.testing.assert_array_equal(out[q, 2:6], boxes[q, :4].astype(np.float64))
        assert out[q, 8] == f * ((p2[0, 3] - p3[0, 3]) / f) / float(dis[q])
        np.testing.assert_array_equal(out[q, 9:12], poses[q, 3:6].astype(np.float64))
        pr = BS.Problem((H, W), p2, p3, float(poses[q, 7]), poses[q, 3:6].astype(np.float64),
                        boxes[q, :4].astype(np.float64), None, kpts[q].astype(np.float64), z_fixed=out[q, 8])
        assert np.abs(pr.gradient(out[q, [6, 7, 12]])).max() < 1e-8, q
    if n:
        assert (succ[:n] > 0).sum() > 100 and (~(succ[:n] > 0)).sum() > 50
