"""dense_align (csrc/dense_align.cu) hypothesis by hypothesis against the CPU oracle.

The kernel's per-pixel arithmetic is the oracle's (every fp32 step an _rn intrinsic in the oracle's order, the oracle
built with -ffp-contract=off), so each pixel's three |L - R| terms are bit-identical and the 70 costs of a RoI differ
from the oracle's float64 sums only by the order of the kernel's fp32 additions.  The tests read the kernel's per-slice
partial sums out of its workspace (part0 [D][S][51] = 50 coarse costs + valid-pixel count, part1 [D][S][21] = 20 fine
costs + count) and hold every cost to the bound that order implies:

    |c_gpu - c_ora| <= (n_chain + 3) * 2^-24 * c_ora

n_chain is the longest chain of fp32 adds a term passes through (per-thread accumulation over the rows or pixels of a
slice, 5 shuffle levels, the cross-warp sum, the S slice adds in argmin_partials); the + 3 covers the two adds of a
pixel's three channel terms and the second-order part of the bound.  The costs are sums of non-negative terms, so the
bound is relative to the cost itself.  Pixel counts, status and best_dis (at the argmins recomputed from the partials)
are exact; an argmin that differs from the oracle's must be a tie within the two costs' bounds.

A CPU census (no GPU) mirrors the strip kernel's reach logic on the oracle's valid pixels and checks that the case
matrix reaches every branch of the kernel: both lattice widths, strip rows that fit in and overflow kStripMax columns,
taps inside and outside the strip, hypotheses through the d = 1 / (zf + rdis) pole, clamping at both image edges,
lattice rows without valid pixels, and every slice count.
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import ops as O
from stereo_rcnn_b200.synth import DEMO_P2, DEMO_P3, gen_rois, synth_pair

F32 = np.float32
SCALE = float(F32(1.6))
STRIP_MAX_D = 48           # kStripMaxD: up to this many RoIs the strip kernel, beyond it the materialised 2x pair
STRIP_MAX = 2048           # kStripMax: columns of the 2x right image one strip holds
MAX_SLICES = 16            # kMaxSlices


def cu(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


# ----------------------------------------------------------------------------------------- host mirrors of the kernel
class Consts(object):
    """dense_align_impl's constants: python doubles rounded to fp32 where they meet a tensor"""

    def __init__(self, c4, scale, H, W):
        s2 = scale * 2.0
        fd = c4[0] * s2
        bld = c4[3] * s2 / fd
        self.s2f, self.f32, self.bl32, self.fb32 = F32(s2), F32(fd), F32(bld), F32(fd * bld)
        self.FH, self.FW = 2 * H, 2 * W
        self.fw2 = F32((self.FW - 1.0) / 2.0)
        self.fh2 = F32((self.FH - 1.0) / 2.0)


def py_slice(start, stop, step, size):
    if start < 0:
        start = max(start + size, 0)
    start = min(start, size)
    if stop < 0:
        stop = max(stop + size, 0)
    stop = min(stop, size)
    return start, (0 if stop <= start else (stop - start + step - 1) // step)


def lattice(k, box_in, kp):
    """setup_roi's pixel lattice -> (u0, nu, su, v0, nv, sv), fp32 arithmetic in the kernel's order"""
    box = np.asarray(box_in, F32) * k.s2f
    b0, b1 = F32(kp[3]) * k.s2f, F32(kp[4]) * k.s2f
    su = max(int((b1 - b0) / F32(56.0)), 1)
    sv = max(int((box[3] - box[1]) / F32(56.0)), 1)
    vs = int((box[1] + box[3]) / F32(2.0) + F32(0.5))
    ve = int(box[3] - (box[3] - box[1]) * F32(0.1) + F32(0.5))
    us, ue = int(b0 + F32(0.5)), int(b1 + F32(0.5))
    v0, nv = py_slice(vs, ve, sv, k.FH)
    u0, nu = py_slice(us, ue, su, k.FW)
    return u0, nu, su, v0, nv, sv


def n_slices(D):
    mat = D > STRIP_MAX_D
    return mat, min(max((296 if mat else 592) // D, 1), MAX_SLICES)


def da_layout(H, W, D):
    """da_layout: byte offsets of upL, upR, part0, part1 and the total, each region rounded up to 256 bytes"""
    off, out = 0, []
    px = 4 * H * W if D > STRIP_MAX_D else 0
    d = max(D, 1)
    for nbytes in (px * 16, px * 16, d * MAX_SLICES * 51 * 4, d * MAX_SLICES * 21 * 4):
        out.append(off)
        off += (nbytes + 255) & ~255
    return out + [off]


def n_chain(lat, D):
    """longest chain of fp32 adds a pixel's term passes through on its way into a slice-summed cost"""
    u0, nu, su, v0, nv, sv = lat
    mat, S = n_slices(D)
    if mat:     # stage_costs_up: pixels per thread, 5 shuffle levels, 8 warps, S slices
        return -(-nu * nv // (256 * S)) + 5 + 8 + S
    wpg = (64 if nu <= 64 else 128) // 32      # stage_costs<NH, PB>: rows per slice, 5 levels, PB / 32 warps, S
    return -(-nv // S) + 5 + wpg + S


def coarse_depth(z0, h):
    d = (z0 - F32(12.5)) + F32(0.5 * h)
    return F32(1.5) if d < F32(1.5) else d


def final_dis(k, pose, ci, fj):
    """dense_final_kernel's best_dis at coarse index ci and fine index fj"""
    dis_init = k.fb32 / F32(pose[2])
    z0 = ((F32(1.0) / dis_init) * k.f32) * k.bl32
    bd = (coarse_depth(z0, ci) - F32(0.5)) + F32(0.05 * fj)
    return k.fb32 / (bd * k.s2f) + F32(0.5)


def rdis_of(k, depths):
    depths = np.asarray(depths, F32)
    return F32(1.0) / ((F32(1.0) / depths) * k.fb32)


def coarse_depths(k, pose):
    dis_init = k.fb32 / F32(pose[2])
    z0 = ((F32(1.0) / dis_init) * k.f32) * k.bl32
    return np.array([coarse_depth(z0, h) for h in range(50)], F32)


def fine_depths(best):
    return np.array([(F32(best) - F32(0.5)) + F32(0.05 * j) for j in range(20)], F32)


def tap_x(k, u, zf, rdis):
    """(xi0, unclamped ix, zf + rdis) of the right-image taps of pixels (u, zf) [P] x hypotheses rdis [NH]"""
    den = zf[:, None] + rdis[None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        d = F32(1.0) / den
        gx = ((u[:, None] - d) - k.fw2) / k.fw2
        ix = ((gx + F32(1.0)) * F32(0.5)) * F32(k.FW - 1)
    xi0 = np.floor(np.minimum(np.maximum(ix, F32(0.0)), F32(k.FW - 1))).astype(np.int64)
    return xi0, ix, den


# --------------------------------------------------------------------------------------------------- case geometry
def calib_for(H, W):
    """DEMO_P2/P3 rescaled so that the original-size frame (H, W) / 1.6 sees the same field of view"""
    kx, ky = (W / SCALE) / 1242.0, (H / SCALE) / 375.0
    p2, p3 = DEMO_P2.copy(), DEMO_P3.copy()
    for p in (p2, p3):
        p[0, :] *= kx           # fx, cx, baseline term
        p[1, 1] = p[0, 0]       # one focal length, as the kernel's ray test uses
        p[1, 2] *= ky
    return p2, p3


FAMILIES = ("near", "narrow", "wide", "near_wide", "left", "right", "border_out", "border_neg", "border_negneg",
            "thin", "tall", "bottom", "invalid")


def family_rois(fams, seed, H, W):
    """one RoI per entry of `fams`: a car projected with calib_for(H, W), box / keypoint border / pose shaped so
    that the RoI exercises one branch of the kernel"""
    p2, _ = calib_for(H, W)
    f, cx, cy = p2[0, 0], p2[0, 2], p2[1, 2]
    Wo, Ho = W / SCALE, H / SCALE
    boxes, kps, poses = [], [], []
    for i, fam in enumerate(fams):
        r = np.random.RandomState(seed * 1009 + i)
        while True:
            z = {"near": (4.0, 14.0), "left": (5.0, 20.0), "right": (5.0, 20.0), "bottom": (4.0, 9.0),
                 "near_wide": (4.0, 10.0), "narrow": (10.0, 60.0), "wide": (6.0, 30.0)}.get(fam, (6.0, 40.0))
            z = r.uniform(*z)
            x = {"left": -r.uniform(0.45, 0.7) * z, "right": r.uniform(0.45, 0.7) * z}.get(fam, r.uniform(-0.3, 0.3) * z)
            y = 1.65
            w, h, l = r.normal([1.6, 1.5, 3.9], 0.1)
            th = r.uniform(-np.pi, np.pi)
            c, s = np.cos(th), np.sin(th)
            xs = np.array([-w / 2, -w / 2, w / 2, w / 2] * 2)
            ys = np.array([0, 0, 0, 0, -h, -h, -h, -h])
            zs = np.array([-l / 2, l / 2, l / 2, -l / 2] * 2)
            X, Y, Z = c * xs + s * zs + x, ys + y, -s * xs + c * zs + z
            if Z.min() < 1:
                continue
            u, v = f * X / Z + cx, f * Y / Z + cy
            x1, x2 = np.clip([u.min(), u.max()], 0, Wo - 1)
            y1, y2 = np.clip([v.min(), v.max()], 0, Ho - 1)
            if x2 - x1 >= 4 and y2 - y1 >= 4:
                break
        b0, b1 = x1, x2
        xc = (x1 + x2) / 2
        if fam == "narrow":                   # lattice <= 64 columns: PB = 64
            half = r.uniform(2.0, 9.5)
            b0, b1 = xc - half, xc + half
        elif fam in ("wide", "near_wide"):    # 64 < nu <= 112: PB = 128 with su = 1
            half = r.uniform(10.8, 17.2)
            b0, b1 = xc - half, xc + half
        elif fam == "border_out":             # the border runs past the box and the frame
            b0, b1 = x1 - r.uniform(5, 40), x2 + r.uniform(5, 40)
        elif fam == "border_neg":             # negative start: python's slice wraps it, nu = 0
            b0 = -r.uniform(1, 30)
        elif fam == "border_negneg":          # both ends negative: a lattice at the right edge of the frame
            b0, b1 = -r.uniform(20, 60), -r.uniform(1, 15)
        elif fam == "left":
            b0 = min(b0, 0.0)
        elif fam == "right":
            b1 = max(b1, Wo - 1)
        if fam == "thin":                     # one or two lattice rows
            yc = (y1 + y2) / 2
            hh = r.uniform(0.4, 0.75)
            y1, y2 = yc - hh, yc + hh
        elif fam == "tall":                   # the box runs below the car: lattice rows without a valid pixel
            y2 = y2 + r.uniform(0.5, 1.5) * (y2 - y1)
        elif fam == "bottom":                 # sv = 1 rows down to the last row of the 2x frame
            y2 = Ho + r.uniform(1, 20)
            y1 = y2 - r.uniform(10, 34)
        pose = [x, y, z, w, h, l, th]
        if fam == "invalid":                  # the rays of its lattice miss the car: no valid pixel
            pose[0] = x + 8.0 + 2 * w
        boxes.append([x1, y1, x2, y2])
        kps.append([xc, 1, 0.9, b0, b1])
        poses.append(pose)
    return np.array(boxes, F32), np.array(kps, F32), np.array(poses, F32)


SIZES = {"bench": (600, 1987), "small": (160, 256), "odd": (75, 1001)}


def _mix(D, offset=0):
    return [FAMILIES[(i + offset) % len(FAMILIES)] for i in range(D)]


# (id, image size, D, families); seeds follow the id
CASES = [
    ("bench-D1-near", "bench", ["near"]),
    ("bench-D1-narrow", "bench", ["narrow"]),
    ("bench-D47-mix", "bench", _mix(47)),
    ("bench-D48-mix", "bench", _mix(48, 3)),
    ("bench-D49-mix", "bench", _mix(49, 5)),
    ("bench-D128-gen", "bench", None),              # gen_rois(128): the bench's own RoI sampler
    ("bench-D300-mix", "bench", _mix(300, 1)),
    ("small-D24-mix", "small", _mix(24, 2)),
    ("small-D48-mix", "small", _mix(48, 7)),
    ("small-D49-mix", "small", _mix(49, 4)),
    ("small-D3-none", "small", ["invalid", "border_neg", "invalid"]),   # no valid pixel anywhere: the early-out
    ("small-D60-none", "small", ["invalid"] * 60),                        # ... on the materialised path
    ("odd-D24-mix", "odd", _mix(24, 6)),
    ("odd-D128-mix", "odd", _mix(128, 8)),
]


def case_inputs(cid):
    """-> images (left, right), calib4, box_left, keypoints, poses of one case"""
    _, size, fams = next(c for c in CASES if c[0] == cid)
    H, W = SIZES[size]
    seed = sum(map(ord, cid))
    left, right = synth_pair(H, W, seed % 97, 40 if size == "bench" else 9)
    if fams is None:
        b, k, p = gen_rois(int(cid.split("-")[1][1:]), seed=5)
        c4 = O.calib_vec(DEMO_P2, DEMO_P3)
    else:
        b, k, p = family_rois(fams, seed, H, W)
        c4 = O.calib_vec(*calib_for(H, W))
    return left, right, c4, b, k, p


# -------------------------------------------------------------------------------------------------------- census
def census_case(cnt, left, right, c4, b, k, p, D=None):
    """mirror of stage_costs' strip reach (a)-(c) on the oracle's valid pixels: counts the branches one call takes"""
    H, W = left.shape[-2:]
    D = b.shape[0] if D is None else D
    kc = Consts(c4, SCALE, H, W)
    mat, S = n_slices(D)
    cnt["S=%d" % S] += 1
    cnt["materialised" if mat else "strip"] += 1
    uvz, npix = O.dense_sample(c4, SCALE, H, W, b, k, p)
    if mat:
        return
    _, _, dg = O.dense_align(c4, SCALE, left, right, b, k, p, diagnostics=True)
    for i in range(b.shape[0]):
        lat = lattice(kc, b[i], k[i])
        if npix[i] == 0:
            continue
        P = int(npix[i])
        u, v, dz = (uvz[i, :P, j].astype(F32) for j in range(3))
        zf = dz / kc.fb32
        pb = 64 if lat[1] <= 64 else 128
        rows = np.unique(v)
        cnt["rows without valid pixels"] += lat[4] - rows.size
        cnt["single-row lattice"] += lat[4] == 1
        cnt["nv < S"] += lat[4] < S
        best = coarse_depths(kc, p[i])[dg["idx"][i, 0]]
        for stage, depths in ((0, coarse_depths(kc, p[i])), (1, fine_depths(best))):
            cnt["PB%d stage %d RoIs" % (pb, stage)] += 1
            xi0, ix, den = tap_x(kc, u, zf, rdis_of(kc, depths))
            cnt["zf + rdis <= 0"] += int((den <= 0).sum())
            cnt["tap clamped at column 0"] += int((ix < 0).sum())
            cnt["tap clamped at FW-1"] += int((ix > kc.FW - 1).sum())
            for vr in rows:
                m = v == vr
                ends = np.concatenate([xi0[m, 0], xi0[m, -1]])
                lo, s_hi = int(ends.min()), int(ends.max()) + 1
                hi = min(s_hi, kc.FW - 1, lo + STRIP_MAX - 1)
                ln = hi - lo + 1
                cnt["strip rows that fit"] += min(s_hi, kc.FW - 1) - lo + 1 <= STRIP_MAX
                cnt["strip rows that overflow"] += min(s_hi, kc.FW - 1) - lo + 1 > STRIP_MAX
                o = xi0[m] - lo
                inside = (o >= 0) & (o + 1 < ln + (xi0[m] + 1 > kc.FW - 1))
                cnt["taps inside the strip"] += int(inside.sum())
                cnt["taps outside the strip (fallback)"] += int((~inside).sum())
                cnt["fallback taps PB%d stage %d" % (pb, stage)] += int((~inside).sum())


def test_dense_align_branch_census(golden_dir):
    """CPU: the case matrix of the GPU tests reaches every branch of the strip kernel and of the dispatch"""
    from collections import Counter
    cnt = Counter()
    g = np.load(os.path.join(golden_dir, "dense_align.npz"))
    left, right = synth_pair(int(g["H"]), int(g["W"]), int(g["seed"]), int(g["shift"]))
    census_case(cnt, left, right, O.calib_vec(g["p2"], g["p3"]), g["box_left"], g["keypoints"], g["poses"])
    for cid, _, _ in CASES:
        census_case(cnt, *case_inputs(cid))
    for cap in N_CAPS:
        cnt["S=%d" % n_slices(cap)[1]] += 1
    for key in sorted(cnt):
        print("census: %-40s %d" % (key, cnt[key]))
    for key in ("PB64 stage 0 RoIs", "PB64 stage 1 RoIs", "PB128 stage 0 RoIs", "PB128 stage 1 RoIs",
                "strip rows that fit", "strip rows that overflow", "taps inside the strip",
                "taps outside the strip (fallback)", "fallback taps PB64 stage 0", "fallback taps PB128 stage 0",
                "zf + rdis <= 0", "tap clamped at column 0", "tap clamped at FW-1", "rows without valid pixels",
                "single-row lattice", "nv < S", "S=16", "S=12", "S=6", "S=1", "strip", "materialised"):
        assert cnt[key] > 0, key


# ------------------------------------------------------------------------------------------------ the GPU contract
N_CAPS = (32, 300)          # sb_dense_align_n: a strip-path capacity and the solver's (materialised, S = 1)


def oracle(left, right, c4, b, k, p):
    st, dis, dg = O.dense_align(c4, SCALE, left, right, b, k, p, diagnostics=True)
    return dict(st=st, dis=dis, **dg)


def nan_workspace(own, H, W, D):
    from stereo_rcnn_b200 import lib
    nb = lib.load().sb_dense_align_workspace_bytes(H, W, D)
    lay = da_layout(H, W, D)
    assert lay[-1] == nb, (lay, nb)
    ws = own.get(nb, torch.device("cuda", torch.cuda.current_device()), "dense_align")   # ops.workspace()'s key
    ws.fill_(0xFF)                                       # every float a NaN
    return ws, nb


def partials(ws, H, W, D, rows):
    """-> part0 [rows, S, 51], part1 [rows, S, 21] of a workspace, after checking that nothing else of the part0 /
    part1 regions was written: rows >= `rows` and the slices the launch did not have are still NaN"""
    _, S = n_slices(D)
    lay = da_layout(H, W, D)
    out = []
    for off, w in ((lay[2], 51), (lay[3], 21)):
        a = ws[off:off + max(D, 1) * MAX_SLICES * w * 4].cpu().numpy().view(F32)
        used = a[:rows * S * w].reshape(rows, S, w)
        assert np.isfinite(used).all(), "unwritten partials"
        assert np.isnan(a[rows * S * w:]).all(), "partials written past row %d x %d slices" % (rows, S)
        out.append(used)
    return out


def run_dense(left, right, c4, b, k, p, own=None):
    """ops.dense_align in a NaN-filled private workspace -> status, best_dis, part0, part1, workspace"""
    from stereo_rcnn_b200 import ops
    H, W = left.shape[-2:]
    D = b.shape[0]
    own = own or ops.WorkspaceOwner()
    ws, _ = nan_workspace(own, H, W, D)
    with ops.workspace_owner(own):
        st, dis = ops.dense_align(c4, SCALE, cu(left), cu(right), cu(b), cu(k), cu(p))
    torch.cuda.synchronize()
    p0, p1 = partials(ws, H, W, D, D)
    return st.cpu().numpy(), dis.cpu().numpy(), p0, p1, ws


def slice_sums(part):
    """argmin_partials' costs: fp32 sums over the slices in slice order"""
    c = np.zeros(part.shape[::2], F32)
    for s in range(part.shape[1]):
        c = c + part[:, s, :]
    return c


def check_contract(tag, c4, H, W, b, k, p, st, dis, p0, p1, ora, D):
    """the per-RoI contract of rows b/k/p (launched with D rows): exact counts, status and best_dis, costs within
    their summation-order bound, argmins equal to the oracle's or a tie within the bounds.  -> stats"""
    kc = Consts(c4, SCALE, H, W)
    n = b.shape[0]
    eps = 2.0 ** -24
    for part, w in ((p0, 50), (p1, 20)):
        cnt = part[:, :, w].astype(np.float64).sum(1)
        np.testing.assert_array_equal(cnt, ora["npix"], err_msg="%s: valid-pixel counts" % tag)
    any_valid = bool((ora["npix"] > 0).any())
    np.testing.assert_array_equal(st, (ora["npix"] > 0).astype(F32) if any_valid else np.zeros(n, F32))
    bound = np.array([(n_chain(lattice(kc, b[i], k[i]), D) + 3) * eps for i in range(n)])[:, None]
    cg, fg = slice_sums(p0[:, :, :50]), slice_sums(p1[:, :, :20])
    worst, ties = 0.0, dict(coarse=0, fine=0, fine_unchecked=0)
    exp = np.empty(n, F32)
    for i in range(n):
        ci, oi = int(np.argmin(cg[i])), int(ora["idx"][i, 0])
        co = ora["cost_coarse"][i]
        err = np.abs(cg[i].astype(np.float64) - co)
        assert (err <= bound[i] * co).all(), (tag, i, "coarse", np.max(err / np.maximum(bound[i] * co, 1e-300)))
        worst = max(worst, float(np.max(err / np.maximum(bound[i] * co, 1e-300))))
        if ci != oi:
            assert co[ci] - co[oi] <= bound[i, 0] * (co[ci] + co[oi]), (tag, i, "coarse argmin", ci, oi)
            ties["coarse"] += 1
        fj = int(np.argmin(fg[i]))
        if ci == oi:
            fo, oj = ora["cost_fine"][i], int(ora["idx"][i, 1])
            err = np.abs(fg[i].astype(np.float64) - fo)
            assert (err <= bound[i] * fo).all(), (tag, i, "fine", np.max(err / np.maximum(bound[i] * fo, 1e-300)))
            worst = max(worst, float(np.max(err / np.maximum(bound[i] * fo, 1e-300))))
            if fj != oj:
                assert fo[fj] - fo[oj] <= bound[i, 0] * (fo[fj] + fo[oj]), (tag, i, "fine argmin", fj, oj)
                ties["fine"] += 1
        else:
            ties["fine_unchecked"] += 1
        exp[i] = final_dis(kc, p[i], ci, fj) if any_valid else kc.fb32 / F32(p[i, 2])
        if any_valid and ci == oi and fj == int(ora["idx"][i, 1]):
            assert exp[i] == ora["dis"][i], (tag, i, "host mirror of dense_final_kernel")
    np.testing.assert_array_equal(dis.view(np.uint32), exp.view(np.uint32), err_msg="%s: best_dis" % tag)
    if not any_valid:
        np.testing.assert_array_equal(dis, ora["dis"])
    return dict(worst=worst, **ties)


def report(tag, stats):
    print("%-22s worst |dc|/bound %.3f, argmin ties justified: coarse %d, fine %d (fine not comparable: %d)"
          % (tag, stats["worst"], stats["coarse"], stats["fine"], stats["fine_unchecked"]))


def check_upsampled(ws, left, right, D):
    """the materialised path's 2x pair in the workspace equals the oracle's F.upsample, bit for bit"""
    H, W = left.shape[-2:]
    lay = da_layout(H, W, D)
    for off, im in ((lay[0], left), (lay[1], right)):
        up = ws[off:off + 4 * H * W * 16].cpu().numpy().view(F32).reshape(2 * H, 2 * W, 4)
        ref = O.upsample2x(im).transpose(1, 2, 0)
        assert np.array_equal(up[..., :3].view(np.uint32), np.ascontiguousarray(ref).view(np.uint32))
        assert not up[..., 3].any()


@pytest.mark.gpu
def test_dense_align_golden(golden_dir):
    """the golden minted by the reference's own align_parallel: status and its valid-pixel counts, plus the contract"""
    g = np.load(os.path.join(golden_dir, "dense_align.npz"))
    left, right = synth_pair(int(g["H"]), int(g["W"]), int(g["seed"]), int(g["shift"]))
    c4 = O.calib_vec(g["p2"], g["p3"])
    assert float(g["scale"]) == SCALE
    b, k, p = g["box_left"], g["keypoints"], g["poses"]
    st, dis, p0, p1, _ = run_dense(left, right, c4, b, k, p)
    ora = oracle(left, right, c4, b, k, p)
    np.testing.assert_array_equal(st, g["status"])
    np.testing.assert_array_equal(ora["npix"], g["npix"])
    np.testing.assert_array_equal(p0[:, :, 50].sum(1), g["npix"])
    np.testing.assert_allclose(ora["dis"], g["best_dis"], rtol=1e-6)
    report("golden", check_contract("golden", c4, int(g["H"]), int(g["W"]), b, k, p, st, dis, p0, p1, ora,
                                    b.shape[0]))


@pytest.mark.gpu
@pytest.mark.parametrize("cid", [c[0] for c in CASES])
def test_dense_align_sweep_vs_oracle(cid):
    """every case of the matrix: the contract, a bit-identical repeat, and the materialised 2x pair"""
    left, right, c4, b, k, p = case_inputs(cid)
    H, W = left.shape[-2:]
    D = b.shape[0]
    st, dis, p0, p1, ws = run_dense(left, right, c4, b, k, p)
    ora = oracle(left, right, c4, b, k, p)
    if cid.endswith("none"):
        assert ora["npix"].sum() == 0
    else:
        assert (ora["npix"] > 0).sum() >= D // 2, "the case should be mostly valid RoIs"
    report(cid, check_contract(cid, c4, H, W, b, k, p, st, dis, p0, p1, ora, D))
    if n_slices(D)[0]:
        check_upsampled(ws, left, right, D)
    st2, dis2, q0, q1, _ = run_dense(left, right, c4, b, k, p)
    for x, y in ((st, st2), (dis, dis2), (p0, q0), (p1, q1)):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


@pytest.mark.gpu
def test_dense_align_no_valid_pixel_early_out_and_module_api():
    from stereo_rcnn_b200.model.dense_align.dense_align import align_parallel

    class Calib:
        p2 = np.array([[100., 0, 100, 4], [0, 100., 60, 0], [0, 0, 1, 0]])
        p3 = np.array([[100., 0, 100, -50], [0, 100., 60, 0], [0, 0, 1, 0]])
    left, right = synth_pair(120, 200, 5, 4)
    b = np.array([[5, 5, 30, 30], [6, 6, 28, 33]], np.float32)
    k = np.array([[17, 1, .9, 5, 30], [17, 1, .9, 6, 28]], np.float32)
    p = np.array([[30., 1.6, 20., 1.6, 1.5, 3.9, 0.3], [-30., 1.6, 25., 1.6, 1.5, 3.9, 1.0]], np.float32)
    st, dis = align_parallel(Calib, 1.0, cu(left)[None], cu(right)[None], cu(b), cu(k), cu(p))
    st_o, dis_o = O.dense_align(O.calib_vec(Calib.p2, Calib.p3), 1.0, left, right, b, k, p)
    assert st_o.sum() == 0
    np.testing.assert_array_equal(st.cpu().numpy(), st_o)
    np.testing.assert_array_equal(dis.cpu().numpy(), dis_o)          # dis_init, bit-exact
    st, dis = align_parallel(Calib, 1.0, cu(left)[None], cu(right)[None], cu(b[:0]), cu(k[:0]), cu(p[:0]))
    assert st.numel() == 0 and dis.numel() == 0


def n_inputs(cap):
    """bench-size pair and `cap` RoIs as the solver lays them out: boxes [cap,5], poses [cap,8]; the extra columns
    hold NaN, which the kernel must not read"""
    H, W = SIZES["bench"]
    left, right = synth_pair(H, W, 11, 40)
    b, k, p = family_rois(_mix(cap, 9), 700 + cap, H, W)
    b5 = np.concatenate([b, np.full((cap, 1), np.nan, F32)], 1)
    p8 = np.concatenate([p, np.full((cap, 1), np.nan, F32)], 1)
    return left, right, O.calib_vec(*calib_for(H, W)), b, k, p, b5, p8


def call_n(L, tl, tr, c4, tb5, tk, tp8, cap, n_dev, status, best, ws, nb):
    from stereo_rcnn_b200.lib import check, ptr, stream_ptr
    H, W = tl.shape[-2:]
    c4p = (ctypes.c_double * 4)(*[float(v) for v in c4])
    check(L.sb_dense_align_n(ptr(tl), ptr(tr), H, W, c4p, SCALE, ptr(tb5), 5, ptr(tk), ptr(tp8), 8, cap, ptr(n_dev),
                             ptr(status), ptr(best), ptr(ws), nb, stream_ptr()), "sb_dense_align_n")


@pytest.mark.gpu
@pytest.mark.parametrize("cap", N_CAPS)
def test_dense_align_n_vs_oracle(cap):
    """sb_dense_align_n with a device-resident count and the solver's strided rows: rows < n meet the contract, rows
    >= n and their partials stay untouched (n = 0: the whole workspace), and n = cap equals sb_dense_align"""
    from stereo_rcnn_b200 import lib, ops
    L = lib.load()
    left, right, c4, b, k, p, b5, p8 = n_inputs(cap)
    H, W = left.shape[-2:]
    ora = oracle(left, right, c4, b, k, p)
    assert (ora["npix"] > 0).sum() >= cap // 2
    tl, tr, tb5, tk, tp8 = cu(left), cu(right), cu(b5), cu(k), cu(p8)
    own = ops.WorkspaceOwner()
    for n in (0, 1, cap // 2 + 1, cap):
        ws, nb = nan_workspace(own, H, W, cap)
        status = torch.full((cap,), float("nan"), device="cuda")
        best = torch.full((cap,), float("nan"), device="cuda")
        n_dev = torch.tensor([n], dtype=torch.int32, device="cuda")
        call_n(L, tl, tr, c4, tb5, tk, tp8, cap, n_dev, status, best, ws, nb)
        torch.cuda.synchronize()
        st, dis = status.cpu().numpy(), best.cpu().numpy()
        assert np.isnan(st[n:]).all() and np.isnan(dis[n:]).all(), "rows >= n written"
        if n == 0:
            assert bool(torch.isnan(ws[:nb].view(torch.float32)).all()), "n = 0 wrote the workspace"
            continue
        p0, p1 = partials(ws, H, W, cap, n)
        rows = {key: v[:n] for key, v in ora.items()}
        if not (rows["npix"] > 0).any():          # the early-out of a call whose live rows have no valid pixel
            rows["dis"] = Consts(c4, SCALE, H, W).fb32 / p[:n, 2]
        report("n %d/%d" % (n, cap), check_contract("n=%d cap=%d" % (n, cap), c4, H, W, b[:n], k[:n], p[:n],
                                                    st[:n], dis[:n], p0, p1, rows, cap))
        if n == cap:
            st_e, dis_e, e0, e1, _ = run_dense(left, right, c4, b, k, p)
            for x, y in ((st, st_e), (dis, dis_e), (p0, e0), (p1, e1)):
                assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


@pytest.mark.gpu
def test_dense_align_n_graph_replay_with_changing_count():
    """one capture of sb_dense_align_n, replayed with the device count changed between replays: each replay equals
    the eager sb_dense_align on its live rows and leaves the rest untouched"""
    from stereo_rcnn_b200 import lib, ops
    L = lib.load()
    cap = N_CAPS[0]
    left, right, c4, b, k, p, b5, p8 = n_inputs(cap)
    H, W = left.shape[-2:]
    st_e, dis_e, _, _, _ = run_dense(left, right, c4, b, k, p)
    tl, tr, tb5, tk, tp8 = cu(left), cu(right), cu(b5), cu(k), cu(p8)
    own = ops.WorkspaceOwner()
    ws, nb = nan_workspace(own, H, W, cap)
    status = torch.full((cap,), float("nan"), device="cuda")
    best = torch.full((cap,), float("nan"), device="cuda")
    n_dev = torch.tensor([cap], dtype=torch.int32, device="cuda")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                   # warm-up outside the capture (attribute setup, module load)
        call_n(L, tl, tr, c4, tb5, tk, tp8, cap, n_dev, status, best, ws, nb)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call_n(L, tl, tr, c4, tb5, tk, tp8, cap, n_dev, status, best, ws, nb)
    for n in (5, 0, cap, 1, cap - 3):
        status.fill_(float("nan"))
        best.fill_(float("nan"))
        n_dev.fill_(n)
        graph.replay()
        torch.cuda.synchronize()
        st, dis = status.cpu().numpy(), best.cpu().numpy()
        assert np.isnan(st[n:]).all() and np.isnan(dis[n:]).all(), n
        exp = dis_e[:n] if st_e[:n].any() else Consts(c4, SCALE, H, W).fb32 / p[:n, 2]     # the early-out
        np.testing.assert_array_equal(st[:n], st_e[:n])
        np.testing.assert_array_equal(dis[:n].view(np.uint32), exp.view(np.uint32))
