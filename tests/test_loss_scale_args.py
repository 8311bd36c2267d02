"""CPU: the dynamic loss scale's entry points -- the six _devscale twins of the backward entry points,
sb_fill_reciprocal and sb_loss_scale_update -- refuse every invalid argument with SB_EINVAL before any CUDA call, and
train.DynamicLossScale refuses the settings sb_loss_scale_update would."""
import ctypes

import pytest

from stereo_rcnn_b200 import lib as L
from stereo_rcnn_b200 import train as TR

SB_EINVAL = -22
FAKE = 1 << 20                                            # never dereferenced: every refusal precedes the first call
INF, NAN = float("inf"), float("nan")


@pytest.fixture(scope="module")
def lib():
    from stereo_rcnn_b200 import build
    build.build()
    return L.load()


def p(off=0):
    return ctypes.c_void_p(FAKE + off)


def refused(lib, bad):
    n0 = lib.sb_launch_count()
    got = {k: f() for k, f in bad.items()}
    assert lib.sb_launch_count() == n0
    assert all(v == SB_EINVAL for v in got.values()), {k: v for k, v in got.items() if v != SB_EINVAL}


def test_conv_wgrad_devscale_rejections(lib):
    N, H, W, Cin, Cout = 1, 4, 8, 64, 128
    nb = lib.sb_conv_wgrad_workspace(N, H, W, Cin, Cout, 3)

    def call(dy=p(), x=p(), n=N, cin=Cin, cout=Cout, k=3, gs=p(), dw=p(), dy32=None, db=None, ws=p(), nbytes=nb):
        return lambda: lib.sb_conv_wgrad_devscale(dy, x, n, H, W, cin, cout, k, None, gs, dw, dy32, db, None, ws,
                                                  nbytes, None)
    refused(lib, {"null grad_scale": call(gs=None), "null dY": call(dy=None), "null X": call(x=None),
                  "null dW": call(dw=None), "N = 0": call(n=0), "k = 2": call(k=2), "Cin % 64": call(cin=96),
                  "Cout < 64": call(cout=32), "db without dy32": call(db=p()), "misaligned dY": call(dy=p(8)),
                  "misaligned X": call(x=p(2)), "misaligned workspace": call(ws=p(4)),
                  "misaligned dy32": call(dy32=p(2), db=p()), "short workspace": call(nbytes=nb - 1)})


def test_conv_wgrad_acc_devscale_rejections(lib):
    N, H, W, Cin, Cout, k = 1, 4, 8, 64, 128, 3
    nb = lib.sb_conv_wgrad_acc_workspace(N, H, W, Cin, Cout, k)

    def call(dy=p(), dy_ld=1024, x=p(), x_ld=Cin + 8, cin=Cin, cout=Cout, gs=p(), dy32=None, dy32_ld=0, db=None,
             rows=Cout, split=Cout, dw_hi=None, db_hi=None, ws=p(), nbytes=nb):
        return lambda: lib.sb_conv_wgrad_acc_devscale(dy, dy_ld, x, x_ld, N, H, W, cin, cout, k, None, gs, dy32,
                                                      dy32_ld, 0, rows, split, p(), db, dw_hi, db_hi, None, ws, nbytes,
                                                      None)
    refused(lib, {"null grad_scale": call(gs=None), "misaligned dY": call(dy=p(8)), "misaligned X": call(x=p(2)),
                  "misaligned workspace": call(ws=p(4)), "dY ld < Cout": call(dy_ld=120), "X ld < Cin": call(x_ld=56),
                  "ld % 8": call(dy_ld=1020), "Cin % 64": call(cin=72, x_ld=72), "Cout % 64": call(cout=96),
                  "short workspace": call(nbytes=nb - 1), "split > rows": call(rows=24, split=30),
                  "rows > Cout": call(rows=Cout + 64), "split < rows without dw_hi": call(rows=24, split=6),
                  "split < rows, db without db_hi": call(rows=24, split=6, dw_hi=p(), db=p(), dy32=p(), dy32_ld=1024),
                  "dy32 ld < Cout": call(db=p(), dy32=p(), dy32_ld=120)})


def test_fpn_grad_combine_devscale_rejections(lib):
    def call(n=1, h=8, w=8, th=16, tw=16, c=256, dt=p(), dp6=None, h6=0, w6=0, scale=p(), out=p(), out16=None):
        return lambda: lib.sb_fpn_grad_combine_devscale(p(), dt, n, h, w, th, tw, c, dp6, h6, w6, scale, out, out16,
                                                        None)
    refused(lib, {"null scale": call(scale=None), "N = 0": call(n=0), "H = 0": call(h=0), "C = 0": call(c=0),
                  "no output": call(out=None), "dt with TH = 0": call(th=0), "dt with TW = 0": call(tw=0),
                  "dp6 of the wrong height": call(dp6=p(), h6=5, w6=4), "dp6 of the wrong width": call(dp6=p(), h6=4,
                                                                                                  w6=3),
                  "too many pixels": call(n=1 << 12, h=1 << 10, w=1 << 10, dt=None)})


def test_rpn_head_grad_devscale_rejections(lib):
    def call(cls=p(), box=p(), B=1, P=100, gs=p(), d16=p(), d32=None):
        return lambda: lib.sb_rpn_head_grad_devscale(cls, box, B, P, gs, d16, d32, None)
    refused(lib, {"null grad_scale": call(gs=None), "null grad_scale, empty": call(gs=None, P=0), "B < 0": call(B=-1),
                  "P < 0": call(P=-1), "null d_cls": call(cls=None), "null d_box": call(box=None),
                  "null dhead16": call(d16=None), "misaligned dhead16": call(d16=p(1)),
                  "misaligned dhead32": call(d32=p(2))})


def test_box_tail_backward_devscale_rejections(lib):
    def call(R=4, K=64, nc=2, ms=1.0, gs=p(), dz16=p(), null_at=None):
        ptrs = [None if null_at == i else p(64 * i) for i in range(15)]
        return lambda: lib.sb_box_tail_backward_devscale(*ptrs[:4], R, K, nc, *ptrs[4:7], ms, gs, *ptrs[7:13],
                                                         dz16 if null_at != 13 else None, ptrs[14], None, None)
    bad = {"null grad_scale": call(gs=None), "R = 0": call(R=0), "nc = 5": call(nc=5), "nc = 0": call(nc=0),
           "K = 0": call(K=0), "mask_scale 0": call(ms=0.0), "mask_scale inf": call(ms=INF),
           "mask_scale nan": call(ms=NAN), "misaligned dz16": call(dz16=p(1)), "R K too large": call(R=1 << 16,
                                                                                                    K=1 << 15)}
    bad.update({"null pointer %d" % i: call(null_at=i) for i in range(15)})
    refused(lib, bad)


def test_kpts_tail_backward_devscale_rejections(lib):
    nb = lib.sb_kpts_tail_backward_workspace(4, 256)

    def call(R=4, G=28, C=256, gs=p(), up=p(), nbytes=nb, ws=p(), null_at=None):
        ptrs = [None if null_at == i else p(64 * i) for i in range(10)]
        return lambda: lib.sb_kpts_tail_backward_devscale(up if null_at != 0 else None, R, G, C, *ptrs[1:5], gs,
                                                          *ptrs[5:9], None, ws if null_at != 9 else None, nbytes, None)
    bad = {"null grad_scale": call(gs=None), "R = 0": call(R=0), "odd G": call(G=27), "G = 66": call(G=66),
           "G = 0": call(G=0), "C % 32": call(C=100), "C > 1024": call(C=2048), "C < 32": call(C=0),
           "misaligned up": call(up=p(1)), "short workspace": call(nbytes=nb - 1), "misaligned workspace": call(ws=p(2))}
    bad.update({"null pointer %d" % i: call(null_at=i) for i in range(10)})
    refused(lib, bad)


def test_fill_reciprocal_rejections(lib):
    refused(lib, {"null v": lambda: lib.sb_fill_reciprocal(p(), 16, None, None),
                  "null v, n = 0": lambda: lib.sb_fill_reciprocal(p(), 0, None, None),
                  "null p": lambda: lib.sb_fill_reciprocal(None, 16, p(), None)})


def test_loss_scale_update_rejections(lib):
    def call(fi=p(), s=p(4), t=p(8), growth=2.0, backoff=0.5, interval=2000):
        return lambda: lib.sb_loss_scale_update(fi, s, t, growth, backoff, interval, None)
    refused(lib, {"null found_inf": call(fi=None), "null scale": call(s=None), "null tracker": call(t=None),
                  "interval 0": call(interval=0), "interval < 0": call(interval=-3), "growth 1": call(growth=1.0),
                  "growth 3": call(growth=3.0), "growth 0.5": call(growth=0.5), "growth inf": call(growth=INF),
                  "growth nan": call(growth=NAN), "growth 0": call(growth=0.0), "growth -2": call(growth=-2.0),
                  "backoff 1": call(backoff=1.0), "backoff 2": call(backoff=2.0), "backoff 0.3": call(backoff=0.3),
                  "backoff 0": call(backoff=0.0), "backoff -0.5": call(backoff=-0.5), "backoff nan": call(backoff=NAN),
                  "backoff 0.75": call(backoff=0.75)})


@pytest.mark.parametrize("kw", [dict(init_scale=3.0), dict(init_scale=0.0), dict(init_scale=-4.0),
                                dict(init_scale=2.0 ** 33), dict(init_scale=2.0 ** -33), dict(init_scale=INF),
                                dict(init_scale=NAN), dict(init_scale=2.0 ** 16 + 1), dict(growth_factor=1.0),
                                dict(growth_factor=3.0), dict(growth_factor=0.5), dict(growth_factor=2.0 ** 200),
                                dict(growth_factor=INF), dict(backoff_factor=1.0), dict(backoff_factor=0.3),
                                dict(backoff_factor=2.0), dict(backoff_factor=0.0), dict(backoff_factor=2.0 ** -200),
                                dict(growth_interval=0), dict(growth_interval=-1), dict(growth_interval=1.5)])
def test_dynamic_loss_scale_rejects_bad_settings(kw):
    with pytest.raises(ValueError):
        TR.DynamicLossScale(**kw)


def test_dynamic_loss_scale_accepts_the_bounds():
    for s in (2.0 ** -32, 1.0, 2.0 ** 16, 2.0 ** 32):
        d = TR.DynamicLossScale(init_scale=s, growth_factor=4.0, backoff_factor=0.25, growth_interval=1)
        assert (d.init_scale, d.growth_factor, d.backoff_factor, d.growth_interval) == (s, 4.0, 0.25, 1)
    d = TR.DynamicLossScale()
    assert (d.init_scale, d.growth_factor, d.backoff_factor, d.growth_interval) == (2.0 ** 16, 2.0, 0.5, 2000)
