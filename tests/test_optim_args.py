"""CPU: the optimizer step and the weight refresh (sb_sgd_step, sb_pack_plan, sb_pack_weights) refuse every invalid
argument with SB_EINVAL before any CUDA call; sb_pack_target has the header's layout; the training step's bucket plan
and parameter groups are those of trainval_net.py."""
import ctypes
import os
import shutil
import subprocess

import pytest
import torch

from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import train as TR

SB_EINVAL = -22
FAKE = 1 << 20                                            # never dereferenced: every refusal precedes the first call
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from stereo_rcnn_b200 import build
    build.build()
    return L.load()


def test_sgd_step_rejections(lib):
    n = 3

    def call(n=n, params=True, grads=True, moms=True, counts=(5, 7, 9), wd=(0.0, 1e-4, 0.0), lrm=(1.0, 2.0, 1.0),
             lr=FAKE, momentum=0.9, skip=FAKE, skipped=FAKE, null_at=None):
        arr = lambda on: (ctypes.c_void_p * 3)(*[None if null_at == i else FAKE + 64 * i for i in range(3)]) if on \
            else None
        return lib.sb_sgd_step(arr(params), arr(grads), arr(moms), (ctypes.c_size_t * 3)(*counts),
                               (ctypes.c_float * 3)(*wd), (ctypes.c_float * 3)(*lrm), n, lr, momentum, skip, skipped,
                               None)
    n0 = lib.sb_launch_count()
    inf, nan = float("inf"), float("nan")
    bad = {"null params": call(params=False), "null grads": call(grads=False), "null moms": call(moms=False),
           "null param 1": call(null_at=1), "n = 0": call(n=0), "n < 0": call(n=-1), "count 0": call(counts=(5, 0, 9)),
           "wd < 0": call(wd=(0.0, -1e-4, 0.0)), "wd nan": call(wd=(nan, 0.0, 0.0)), "wd inf": call(wd=(inf, 0, 0)),
           "lr_mult < 0": call(lrm=(1.0, -1.0, 1.0)), "lr_mult nan": call(lrm=(1.0, 1.0, nan)),
           "null lr": call(lr=None), "momentum nan": call(momentum=nan), "momentum inf": call(momentum=inf),
           "null skip": call(skip=None), "null skipped": call(skipped=None)}
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in bad.values()), {k: v for k, v in bad.items() if v != SB_EINVAL}
    assert lib.sb_sgd_step(None, None, None, None, None, None, 1, FAKE, 0.9, FAKE, FAKE, None) == SB_EINVAL


def _target(**over):
    t = L.PackTarget()
    t.src, t.dst = FAKE, FAKE
    for k, (s, ss, ds) in enumerate(zip((1, 9, 32, 64), (0, 1, 9 * 64, 9), (0, 64, 9 * 64, 1))):
        t.shape[k], t.src_stride[k], t.dst_stride[k] = s, ss, ds
    t.transform = L.PACK_TF32
    for k, v in over.items():
        if k in ("shape", "src_stride", "dst_stride"):
            for i, x in enumerate(v):
                getattr(t, k)[i] = x
        else:
            setattr(t, k, v)
    return t


def _plan(lib, ts):
    tab = (L.PackTarget * len(ts))(*ts)
    n = ctypes.c_longlong(-1)
    return lib.sb_pack_plan(tab, len(ts), ctypes.byref(n)), tab, n.value


def test_pack_plan_tiles(lib):
    """a plain copy runs straight through in 4096-element tiles; a transposed target gets 288-row x 32-column tiles,
    the reads walking i1 first and then the nearer of i2 / i3"""
    flat = _target(shape=(1, 1, 1, 10000), src_stride=(0, 0, 0, 1), dst_stride=(0, 0, 0, 1))
    fwd3 = _target()                                                      # [co][ci][tap] -> [co][tap][ci]
    dgrad3 = _target(shape=(1, 9, 64, 32), src_stride=(0, -1, 9, 9 * 64), dst_stride=(0, 32, 9 * 32, 1),
                     src_offset=8, transform=L.PACK_SCALE_F16, scale=FAKE)
    rc, tab, n = _plan(lib, [flat, fwd3, dgrad3])
    assert rc == 0
    assert (list(tab[0].tile), tab[0].tiled, tab[0].tile0) == ([1, 1, 4096], 0, 0)
    assert (list(tab[1].tile), tab[1].tiled, tab[1].tile0) == ([9, 32, 32], 2, 3)
    assert (list(tab[2].tile), tab[2].tiled, tab[2].tile0) == ([9, 32, 32], 1, 3 + 2)
    assert n == 3 + 2 + 2


def test_pack_rejections(lib):
    n0 = lib.sb_launch_count()
    bad_targets = {
        "null src": _target(src=None), "null dst": _target(dst=None), "zero extent": _target(shape=(1, 9, 0, 64)),
        "negative extent": _target(shape=(-1, 9, 32, 64)), "dst_stride[3] != 1": _target(dst_stride=(0, 64, 576, 2)),
        "transform -1": _target(transform=-1), "transform 4": _target(transform=4),
        "scale without SCALE_F16": _target(scale=FAKE), "SCALE_F16 without scale": _target(transform=L.PACK_SCALE_F16),
        "scale_dim 4": _target(transform=L.PACK_SCALE_F16, scale=FAKE, scale_dim=4),
        "scale_dim -1": _target(transform=L.PACK_SCALE_F16, scale=FAKE, scale_dim=-1),
        "dst16 with F16": _target(transform=L.PACK_F16, dst16=FAKE),
        "flip below src": _target(src_stride=(0, -1, 576, 9)),
        "flip below dst": _target(dst_stride=(0, -64, 576, 1), dst_offset=7 * 64),
    }
    got = {k: _plan(lib, [_target(), t])[0] for k, t in bad_targets.items()}
    n = ctypes.c_longlong()
    got["n_targets 0"] = lib.sb_pack_plan((L.PackTarget * 1)(_target()), 0, ctypes.byref(n))
    got["null table"] = lib.sb_pack_plan(None, 1, ctypes.byref(n))
    got["null n_tiles"] = lib.sb_pack_plan((L.PackTarget * 1)(_target()), 1, None)
    got["too many tiles"] = _plan(lib, [_target(shape=(1 << 26, 9, 32, 1 << 12))])[0]
    # sb_pack_weights: the same checks, plus tile fields that differ from the plan's
    rc, tab, _ = _plan(lib, [_target(), _target(shape=(1, 1, 1, 5000), src_stride=(0, 0, 0, 1),
                                                dst_stride=(0, 0, 0, 1))])
    assert rc == 0

    def weights(mut=None, n=2, dev=FAKE):
        t2 = (L.PackTarget * 2)(*tab)
        if mut:
            mut(t2)
        return lib.sb_pack_weights(t2, dev, n, None)
    got["weights: null device table"] = weights(dev=None)
    got["weights: n 0"] = weights(n=0)
    got["weights: null src"] = weights(lambda t: setattr(t[1], "src", None))
    got["weights: tile0 off"] = weights(lambda t: setattr(t[1], "tile0", t[1].tile0 + 1))
    got["weights: tiled flag"] = weights(lambda t: setattr(t[0], "tiled", 1))
    got["weights: tile extent"] = weights(lambda t: t[0].tile.__setitem__(1, 16))
    got["weights: unplanned"] = lib.sb_pack_weights((L.PackTarget * 1)(_target()), FAKE, 1, None)
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in got.values()), {k: v for k, v in got.items() if v != SB_EINVAL}


def test_pack_target_layout_against_the_header_compiled_as_c(tmp_path):
    if shutil.which("gcc") is None:
        pytest.skip("no gcc")
    cls = L.PackTarget
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "stereo_b200.h"', "int main(void) {",
             'printf("size %zu\\n", sizeof(sb_pack_target));']
    lines += ['printf("%s %%zu\\n", offsetof(sb_pack_target, %s));' % (f[0], f[0]) for f in cls._fields_]
    lines += ['printf("consts %d %d %d %d\\n", SB_PACK_F32, SB_PACK_TF32, SB_PACK_F16, SB_PACK_SCALE_F16);',
              "return 0;", "}"]
    src = tmp_path / "pack_layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "pack_layout"
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o",
                           str(exe)])
    got = dict(l.split(" ", 1) for l in subprocess.check_output([str(exe)], text=True).splitlines())
    assert int(got["size"]) == ctypes.sizeof(cls)
    for f in cls._fields_:
        assert int(got[f[0]]) == getattr(cls, f[0]).offset, f[0]
    assert got["consts"].split() == [str(v) for v in (L.PACK_F32, L.PACK_TF32, L.PACK_F16, L.PACK_SCALE_F16)]


@pytest.mark.parametrize("fixed_blocks", [0, 1])
def test_bucket_plan_shared_by_masters_gradients_and_momentum(fixed_blocks):
    named = TR.trainable_names(fixed_blocks)
    shapes = [s for _, s in named] + [(6,)]
    sets = TR.state_buckets(shapes, "cpu")
    assert len(named) == (139 if fixed_blocks == 1 else 139 + 3 * 3 + 1)
    for views in zip(*[s.grads for s in sets]):
        locs = []
        for s, v in zip(sets, views):
            b = [i for i, bk in enumerate(s.buckets) if bk.untyped_storage().data_ptr() == v.untyped_storage().data_ptr()]
            assert len(b) == 1
            locs.append((b[0], v.storage_offset(), tuple(v.shape)))
        assert locs[0] == locs[1] == locs[2]
    for s in sets:
        assert tuple(s.grads[-1].shape) == (6,)
        b = s.buckets[-1]
        assert s.grads[-1].storage_offset() + 6 <= b.numel()
        assert all(v.storage_offset() < s.grads[-1].storage_offset() for v in s.grads[:-1]
                   if v.untyped_storage().data_ptr() == b.untyped_storage().data_ptr())
        assert all(float(b.abs().max()) == 0.0 for b in s.buckets)
    # the clip list of a step is every view but the last: uncert is not a model parameter (net_utils.py:37-49)
    clip = sets[1].grads[:-1]
    assert len(clip) == len(named) and all(tuple(v.shape) == tuple(s) for v, (_, s) in zip(clip, named))


@pytest.mark.parametrize("double_bias", [False, True])
@pytest.mark.parametrize("bias_decay", [False, True])
def test_param_groups_match_trainval(double_bias, bias_decay):
    """trainval_net.py:158-166, restated over torch parameters and torch.optim.SGD's own group bookkeeping"""
    lr, wd = 1e-3, 1e-4
    named = TR.trainable_names(1)
    params = []
    for key, _ in named:
        value = torch.nn.Parameter(torch.zeros(1))
        if "bias" in key:
            params += [{"params": [value], "lr": lr * (double_bias + 1), "weight_decay": bias_decay and wd or 0}]
        else:
            params += [{"params": [value], "lr": lr, "weight_decay": wd}]
    params += [{"params": [torch.nn.Parameter(torch.zeros(6))], "lr": lr}]
    opt = torch.optim.SGD(params, momentum=0.9)
    ours = TR.param_groups([n for n, _ in named] + ["uncert"], wd, double_bias, bias_decay)
    assert len(ours) == len(opt.param_groups)
    for (mult, w), g in zip(ours, opt.param_groups):
        assert lr * mult == g["lr"] and w == g["weight_decay"] and g["momentum"] == 0.9
        assert g["dampening"] == 0 and not g["nesterov"]
