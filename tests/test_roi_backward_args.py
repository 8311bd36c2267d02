"""CPU: sb_roi_align_pyramid_backward refuses every invalid argument with SB_EINVAL before any CUDA call (so without a
GPU, and without a launch), a call with no RoI returns SB_OK without a launch, the workspace query states the fixed-point
accumulators' size, sb_roi_grad_source has the same layout in C and in the ctypes mirror, and the GPU file's kernel
cases cover every routing, edge and layout family."""
import collections
import ctypes
import os
import shutil
import subprocess
import zlib

import numpy as np
import pytest

from stereo_rcnn_b200 import lib as L
from test_gpu_roi_backward import CASES, tiny_rois
from test_gpu_roi_heads import IMAGE, boundary_sweep, level_sets, mixed_rois

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SB_EINVAL = -22
BENCH = ((150, 497), (75, 249), (38, 125), (19, 63))      # P2..P5 of a 600x1987 image


@pytest.fixture(scope="module")
def lib():
    from stereo_rcnn_b200 import build
    build.build()
    return L.load()


def ints(v):
    return (ctypes.c_int * len(v))(*v)


def test_workspace_of_the_benchmark_pair(lib):
    """P2..P5 of one 600x1987 pair: 99172 pixels x 2 images x 256 channels of int64, plus 16 bytes"""
    hs, ws = ints([h for h, _ in BENCH]), ints([w for _, w in BENCH])
    assert sum(h * w for h, w in BENCH) == 99172
    nb = lib.sb_roi_align_pyramid_backward_workspace(hs, ws, 2, 256)
    assert nb == 99172 * 2 * 256 * 8 + 16
    print("RoIAlign backward workspace at 600x1987, B=1: %.1f MB" % (nb / 1e6))
    assert lib.sb_roi_align_pyramid_backward_workspace(hs, ws, 0, 256) == 0
    assert lib.sb_roi_align_pyramid_backward_workspace(ints([150, 75, 38, 1]), ws, 2, 256) == 0


def test_rejections_before_any_launch(lib):
    fake = 1 << 20                                          # never dereferenced: every refusal precedes the first call
    hs0, ws0 = [h for h, _ in BENCH], [w for _, w in BENCH]
    nb = lib.sb_roi_align_pyramid_backward_workspace(ints(hs0), ints(ws0), 2, 256)

    def call(R=512, P=7, ld=512, coff=0, boff=0, grad=fake, rois=fake, n_src=1, N=2, C=256, hs=None, ws=None,
             feats=(fake,) * 4, work=fake, nbytes=nb, src_null=False, n_sources_arr=1):
        srcs = (L.RoiGradSource * max(n_src, 1))()
        for s in srcs:
            s.grad, s.rois, s.R, s.pooled, s.ld, s.coff, s.batch_offset = grad, rois, R, P, ld, coff, boff
        fp = (ctypes.c_void_p * 4)(*feats)
        return lib.sb_roi_align_pyramid_backward(None if src_null else srcs, n_src, fp, ints(hs or hs0),
                                                 ints(ws or ws0), N, C, 600.0, None, work, nbytes, None)
    n0 = lib.sb_launch_count()
    bad = {"slice past ld": call(coff=260), "C % 4": call(C=254, ld=508), "ld % 4": call(ld=514),
           "coff % 4": call(coff=2), "coff < 0": call(coff=-4), "C = 0": call(C=0),
           "level 1 row": call(hs=[150, 75, 38, 1]), "level 1 column": call(ws=[497, 1, 125, 63]),
           "batch offset < 0": call(boff=-1), "batch offset = N": call(boff=2),
           "short workspace": call(nbytes=nb - 1), "misaligned workspace": call(work=fake + 4),
           "null workspace": call(work=None), "null grad": call(grad=None), "null rois": call(rois=None),
           "null level": call(feats=(fake, fake, None, fake)), "null sources": call(src_null=True),
           "no source": call(n_src=0), "five sources": call(n_src=5), "N = 0": call(N=0),
           "R < 0": call(R=-1), "pooled 0": call(P=0), "shared memory > 48 KB": call(P=64)}
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}
    # no RoI in any source: nothing to add, nothing launched (null gradients are then allowed, as in the forward)
    assert call(R=0, grad=None, rois=None, n_src=3) == 0
    assert lib.sb_launch_count() == n0


def test_source_struct_layout_matches_c(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "stereo_b200.h"', "int main(void) {",
             'printf("size %zu\\n", sizeof(sb_roi_grad_source));']
    for f in L.RoiGradSource._fields_:
        lines.append('printf("%s %%zu\\n", offsetof(sb_roi_grad_source, %s));' % (f[0], f[0]))
    lines += ["return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                           str(exe)])
    got = dict(l.split() for l in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(got["size"]) == ctypes.sizeof(L.RoiGradSource)
    for f in L.RoiGradSource._fields_:
        assert int(got[f[0]]) == getattr(L.RoiGradSource, f[0]).offset, f[0]


def test_case_matrix_census():
    """the kernel cases of test_gpu_roi_backward reach every level routed and clamped, the three ambiguous boundaries,
    both image edges, tiny RoIs, an empty source, a right-image offset, C/4 from 1 to 128 and P in 1, 2, 7, 8, 9, 14,
    15"""
    cnt = collections.Counter()
    for c in CASES:
        for i, s in enumerate(c.srcs):
            if s.fam == "sweep":
                rois = np.concatenate([boundary_sweep(k) for k in range(3)])
            elif s.fam == "tiny":
                rois = tiny_rois(s.R, c.pyr, zlib.crc32(c.id.encode()) + i)
            elif s.R:
                rois = mixed_rois(s.R, c.pyr, zlib.crc32(c.id.encode()) + i)
            else:
                cnt["empty source"] += 1
                continue
            lo, hi, raw = level_sets(rois)
            for l in range(4):
                cnt["P%d routed" % (l + 2)] += int(((lo == hi) & (lo == l) & (raw == l + 2)).sum())
                cnt["P%d clamped" % (l + 2)] += int(((lo == hi) & (lo == l) & (raw != l + 2)).sum())
            for l in range(3):
                cnt["ambiguous P%d|P%d" % (l + 2, l + 3)] += int(((lo == l) & (hi == l + 1)).sum())
            im_h, im_w = IMAGE[c.pyr]
            cnt["past right/bottom"] += int(((rois[:, 3] > im_w - 1) | (rois[:, 4] > im_h - 1)).sum())
            cnt["negative start"] += int(((rois[:, 1] < 0) | (rois[:, 2] < 0)).sum())
            cnt["tiny"] += int((((rois[:, 3] - rois[:, 1]) < 1) & ((rois[:, 4] - rois[:, 2]) < 1)).sum())
            cnt["right offset"] += int(s.side == 1)
    print("\nRoIAlign backward census: %s" % dict(sorted(cnt.items())))
    need = (["P%d routed" % l for l in range(2, 6)] + ["P2 clamped", "P5 clamped"] +
            ["ambiguous P%d|P%d" % (l, l + 1) for l in range(2, 5)] +
            ["past right/bottom", "negative start", "tiny", "right offset", "empty source"])
    assert not [k for k in need if not cnt[k]], [k for k in need if not cnt[k]]
    assert {c.C // 4 for c in CASES} >= {1, 128}
    assert {s.P for c in CASES for s in c.srcs} >= {1, 2, 7, 8, 9, 14, 15}
