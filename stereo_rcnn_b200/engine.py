"""The Stereo R-CNN test-mode forward on hand-written sm_90a kernels.

Host-side schedule of `_StereoRCNN.forward` (lib/model/stereo_rcnn/stereo_rcnn.py:141-324):
weights are packed once (NHWC / K-major, frozen BN folded to per-channel scale+shift --
resnet.py:300-309 freezes every BN), left and right images run through the trunk as one
batch of two, and every stage is a libstereo_b200 kernel launched on torch's current stream.
There is no PyTorch operator on the compute path (torch only allocates device memory).
"""
import ctypes

import torch

from . import lib as _lib
from . import ops

LAYERS = [3, 4, 23, 3]
PLANES = [64, 128, 256, 512]
STRIDES = [1, 2, 2, 2]
EPS = 1e-5


def trainable_trunk_fpn_params(fixed_blocks=1):
    """[(name, shape)] of the trunk + FPN parameters that receive a gradient (resnet.py:289-309 of the reference):
    RCNN_layer0 and every BatchNorm are frozen, cfg.RESNET.FIXED_BLOCKS = k also freezes RCNN_layer1..k, the FPN convs
    (top, lateral and smooth layers, weights and biases) always train."""
    assert 0 <= fixed_blocks < 4
    out = []
    inplanes = 64
    for li, nb in enumerate(LAYERS):
        planes = PLANES[li]
        for bi in range(nb):
            p = "RCNN_layer%d.0.%d" % (li + 1, bi)
            cin = inplanes if bi == 0 else planes * 4
            if li + 1 > fixed_blocks:
                out += [(p + ".conv1.weight", (planes, cin, 1, 1)), (p + ".conv2.weight", (planes, planes, 3, 3)),
                        (p + ".conv3.weight", (planes * 4, planes, 1, 1))]
                if bi == 0:
                    out.append((p + ".downsample.0.weight", (planes * 4, cin, 1, 1)))
        inplanes = planes * 4
    for k, cin, ks in (("RCNN_toplayer", 2048, 1), ("RCNN_smooth1", 256, 3), ("RCNN_smooth2", 256, 3),
                       ("RCNN_smooth3", 256, 3), ("RCNN_latlayer1", 1024, 1), ("RCNN_latlayer2", 512, 1),
                       ("RCNN_latlayer3", 256, 1)):
        out += [(k + ".weight", (256, cin, ks, ks)), (k + ".bias", (256,))]
    return out


def trainable_rpn_params():
    """[(name, shape)] of the stereo RPN's parameters (stereo_rpn.py:32-39 of the reference), all trainable: RPN_Conv
    (3x3, 256 -> 512, shared by both images and all five levels) and the two 1x1 heads on the 1024-channel
    concatenation"""
    return [("RCNN_rpn.RPN_Conv.weight", (512, 256, 3, 3)), ("RCNN_rpn.RPN_Conv.bias", (512,)),
            ("RCNN_rpn.RPN_cls_score.weight", (6, 1024, 1, 1)), ("RCNN_rpn.RPN_cls_score.bias", (6,)),
            ("RCNN_rpn.RPN_bbox_pred_left_right.weight", (18, 1024, 1, 1)),
            ("RCNN_rpn.RPN_bbox_pred_left_right.bias", (18,))]


def trainable_rcnn_head_params(n_classes=2):
    """[(name, shape)] of the R-CNN heads' parameters (resnet.py:256-286 of the reference), all trainable: RCNN_top
    (Conv7x7/7 512 -> 2048, Conv1x1 2048 -> 2048), the three linears on fc7, the six keypoint 3x3 convs, the keypoint
    deconv (ConvTranspose2d, weight [Cin, Cout, 2, 2]) and kpts_class"""
    out = [("RCNN_top.0.weight", (2048, 512, 7, 7)), ("RCNN_top.0.bias", (2048,)),
           ("RCNN_top.3.weight", (2048, 2048, 1, 1)), ("RCNN_top.3.bias", (2048,)),
           ("RCNN_cls_score.weight", (n_classes, 2048)), ("RCNN_cls_score.bias", (n_classes,)),
           ("RCNN_bbox_pred.weight", (6 * n_classes, 2048)), ("RCNN_bbox_pred.bias", (6 * n_classes,)),
           ("RCNN_dim_orien_pred.weight", (5 * n_classes, 2048)), ("RCNN_dim_orien_pred.bias", (5 * n_classes,))]
    for i in range(0, 12, 2):
        out += [("RCNN_kpts.%d.weight" % i, (256, 256, 3, 3)), ("RCNN_kpts.%d.bias" % i, (256,))]
    return out + [("RCNN_kpts.12.weight", (256, 256, 2, 2)), ("RCNN_kpts.12.bias", (256,)),
                  ("kpts_class.weight", (6, 256, 1, 1)), ("kpts_class.bias", (6,))]


# Dropout(p=0.2) after each ReLU of RCNN_top (resnet.py:256-263): active in training, since resnet.train() never puts
# RCNN_top back in eval mode
DROPOUT_P = 0.2


class HeadsSaved(object):
    """what StereoRCNNEngine.heads(save_for_backward=True) keeps for heads_backward, all for the R sampled RoIs: the fp16
    pooled tensors pooled_box [R,7,7,512] and pooled_kpts [R,14,14,256]; top0 [R,1,1,2048] fp16 and fc7 [R,2048] fp32,
    the outputs of RCNN_top.0 / RCNN_top.3 after ReLU and dropout (y > 0 is the combined mask); kpts, the six fp16
    outputs of RCNN_kpts.0..10 [R,14,14,256]; up [R,28,28,256] fp16, the deconv's ReLU'd output; and for
    roi_align_backward the RoIs the pooling read (rois_l, rois_r [R,5]: references, not copies), im_h and B"""
    __slots__ = ("R", "dropout", "pooled_box", "pooled_kpts", "top0", "fc7", "kpts", "up", "rois_l", "rois_r", "im_h",
                 "B")

    def __init__(self, R, dropout, pooled_box, pooled_kpts, top0, fc7, kpts, up, rois_l, rois_r, im_h, B):
        self.R, self.dropout, self.pooled_box, self.pooled_kpts = R, dropout, pooled_box, pooled_kpts
        self.top0, self.fc7, self.kpts, self.up = top0, fc7, kpts, up
        self.rois_l, self.rois_r, self.im_h, self.B = rois_l, rois_r, im_h, B


class RpnSaved(object):
    """what StereoRCNNEngine.rpn(save_for_backward=True) keeps for rpn_backward: per level the fp16 `cat` buffer
    [B,h,w,1024] (the ReLU'd RPN_Conv outputs of L | R: the heads' input and the ReLU mask) and the fp16 P level
    [2B,h,w,256] it read, plus the raw fused head output [B,P,32]"""
    __slots__ = ("B", "shapes", "offs", "cats", "levels", "head")

    def __init__(self, B, shapes, offs, cats, levels, head):
        self.B, self.shapes, self.offs, self.cats, self.levels, self.head = B, shapes, offs, cats, levels, head


_LEVELS = ("p2", "p3", "p4", "p5", "p6")
_FC = ("RCNN_cls_score.weight", "RCNN_cls_score.bias", "RCNN_bbox_pred.weight", "RCNN_bbox_pred.bias",
       "RCNN_dim_orien_pred.weight", "RCNN_dim_orien_pred.bias")


# which lateral conv reads the input of RCNN_layer<li+1> (li = 1..3): c2 -> latlayer3, c3 -> latlayer2, c4 -> latlayer1
_LATERAL_OF_INPUT = {1: ("RCNN_latlayer3", "dt2"), 2: ("RCNN_latlayer2", "dt3"), 3: ("RCNN_latlayer1", "dt4")}


def _alloc(shape, dtype, device, zeroed=False):
    """a device tensor for sb_pack_weights to fill; zeroed ones (padding the table never writes) are host zeros
    copied over, so that building an engine launches no torch kernel"""
    if zeroed:
        return torch.zeros(shape, dtype=dtype).to(device)
    return torch.empty(shape, dtype=dtype, device=device)


class _DgradConv(object):
    """conv weights for the data gradient (the forward conv Cin -> Cout run backwards, Cout -> Cin here):
    w16 [Cout][kh][kw][Cin] fp16, written by sb_pack_weights (StereoRCNNEngine._pack_targets)"""
    __slots__ = ("w16", "Cin", "Cout", "kh", "kw", "pad")

    def __init__(self, Cin, Cout, kh, kw, pad, device, zeroed=False):
        self.Cin, self.Cout, self.kh, self.kw, self.pad = Cin, Cout, kh, kw, pad
        self.w16 = _alloc((Cout, kh, kw, Cin), torch.float16, device, zeroed)


def _numel(shape):
    n = 1
    for d in shape:
        n *= int(d)
    return n


class _PackT(object):
    """one sb_pack_target of engine.refresh_weights: the master tensor `name` -> dst (element strides, see
    include/stereo_b200.h)"""
    __slots__ = ("name", "dst", "shape", "sstr", "dstr", "transform", "src_offset", "dst_offset", "dst16", "scale")

    def __init__(self, name, dst, shape, sstr, dstr, transform, src_offset=0, dst_offset=0, dst16=None, scale=None):
        assert dst.is_contiguous() and (dst16 is None or dst16.is_contiguous())
        self.name, self.dst, self.shape, self.sstr, self.dstr = name, dst, shape, sstr, dstr
        self.transform, self.src_offset, self.dst_offset, self.dst16, self.scale = (transform, src_offset, dst_offset,
                                                                                      dst16, scale)

    def fill(self, t, src):
        t.src, t.dst = src.data_ptr(), self.dst.data_ptr()
        t.dst16 = self.dst16.data_ptr() if self.dst16 is not None else None
        t.scale = self.scale.data_ptr() if self.scale is not None else None
        t.src_offset, t.dst_offset = self.src_offset, self.dst_offset
        for k in range(4):
            t.shape[k], t.src_stride[k], t.dst_stride[k] = self.shape[k], self.sstr[k], self.dstr[k]
        t.transform, t.scale_dim = self.transform, 3


class PackedConv(object):
    """a forward conv on the device: w [Cout][kh][kw][Cin] fp32 and, in fp16 engines, its fp16 twin w16, written by
    sb_pack_weights (StereoRCNNEngine._pack_targets); scale the folded frozen-BN scale (None for a conv with a bias),
    shift the folded BN shift or the bias"""
    __slots__ = ("w", "w16", "scale", "shift", "Cin", "Cout", "kh", "kw", "pad")

    def __init__(self, Cout, Cin, kh, kw, pad, scale, shift, half, device, zeroed=False):
        self.Cout, self.Cin, self.kh, self.kw, self.pad = Cout, Cin, kh, kw, pad
        self.w = _alloc((Cout, kh, kw, Cin), torch.float32, device, zeroed)
        self.w16 = _alloc((Cout, kh, kw, Cin), torch.float16, device, zeroed) if half else None
        self.scale, self.shift = scale, shift


class StereoRCNNEngine(object):
    """state_dict uses the reference's key names (RCNN_layer1.0.0.conv1.weight, ...)"""

    def __init__(self, state_dict, device="cuda", n_classes=2, conv_impl="auto", precision=None, forks=True):
        """precision: "tf32" (fp32 storage, tf32) or "fp16" (fp16 conv operands, f16, fp32 accumulate
        and fp32 residual stream); default from $SB_PRECISION, else "fp16" (same measured accuracy as tf32 --
        both round operands to an 11-bit significand -- at twice the MMA rate and half the activation bytes).  conv_impl="simt" forces exact fp32.
        forks=True is the latency schedule: layers 3-4 of the left and the right image run as two concurrent chains,
        and the coarse RPN levels and the box head run on a side stream beside the rest.  forks=False is the
        throughput schedule, one chain with no forks: with several independent pairs in flight the SMs are already
        full and the batched chain (fewer, wider tiles) costs less SM time."""
        import os
        precision = precision or os.environ.get("SB_PRECISION", "fp16")
        assert precision in ("tf32", "fp16")
        self.half = precision == "fp16" and conv_impl != "simt"
        self.precision = "fp32-simt" if conv_impl == "simt" else precision
        self.keep32 = False
        self.forks = bool(forks)
        self.side = torch.cuda.Stream(device=torch.device(device)) if torch.device(device).type == "cuda" else None
        self.device = torch.device(device)
        self.n_classes = n_classes
        self.conv_impl = conv_impl
        self.impl_used = {}
        self.record = None        # bench: list collecting (desc, live tensors) of every conv launch of a forward
        # conv_impl="simt" is the exact-fp32 yardstick: exact weights, exact stores, no TF32 hygiene modes
        self.exact = conv_impl == "simt"
        # The BN fold is host arithmetic on frozen values; every weight layout is written by one sb_pack_weights launch
        # over the table of _pack_targets, from fp32 masters uploaded by plain copies and dropped after: no torch kernel
        # runs on the GPU for it, so a profiler's launch window of a process that builds an engine shows this library's
        # kernels only.  The host masters stay for the data-gradient copies, packed on first use.
        sd = {k: v.detach().to("cpu", torch.float32).contiguous() for k, v in state_dict.items()
              if not k.endswith("num_batches_tracked")}
        self._masters = sd
        self._trainable = dict(trainable_trunk_fpn_params(0) + trainable_rpn_params() +
                               trainable_rcnn_head_params(n_classes))
        self._bwd = None
        self._found_inf = None
        dev, h = self.device, self.half
        empty = lambda *shape: torch.empty(shape, dtype=torch.float32, device=dev)
        self.p = {}

        def bn_fold(k):
            s = sd[k + ".weight"] / torch.sqrt(sd[k + ".running_var"] + EPS)
            return s.to(dev), (sd[k + ".bias"] - sd[k + ".running_mean"] * s).to(dev)

        def conv(key, pad, bn=None):
            co, ci, kh, kw = sd[key + ".weight"].shape
            scale, shift = bn_fold(bn) if bn is not None else (None, empty(co))
            self.p[key] = PackedConv(co, ci, kh, kw, pad, scale, shift, h, dev)

        s, b = bn_fold("RCNN_layer0.1")
        self.stem = (empty(64, 7, 7, 3), s, b)
        # the stem as a GEMM over sb_stem_im2col's patch matrix (K = 147 taps padded to 160), and the fp16 K layout of
        # the fused stem sb_stem_conv_tc (padded to three 64-wide K-steps)
        self.p["stem_gemm"] = PackedConv(64, 160, 1, 1, 0, s, b, h, dev, zeroed=True)
        self.stem_w16 = _alloc((64, 192), torch.float16, dev, zeroed=True)
        for li, nb in enumerate(LAYERS):
            for bi in range(nb):
                p = "RCNN_layer%d.0.%d" % (li + 1, bi)
                conv(p + ".conv1", 0, p + ".bn1")
                conv(p + ".conv2", 1, p + ".bn2")
                conv(p + ".conv3", 0, p + ".bn3")
                if bi == 0:
                    conv(p + ".downsample.0", 0, p + ".downsample.1")
        for k in ("RCNN_toplayer", "RCNN_latlayer1", "RCNN_latlayer2", "RCNN_latlayer3"):
            conv(k, 0)
        for k in ("RCNN_smooth1", "RCNN_smooth2", "RCNN_smooth3", "RCNN_rpn.RPN_Conv"):
            conv(k, 1)
        # RPN 1x1 heads fused: rows 0..5 cls logits, 6..23 box deltas, 24..31 zero padding
        self.p["rpn_heads"] = PackedConv(32, 1024, 1, 1, 0, None, _alloc(32, torch.float32, dev, True), h, dev,
                                         zeroed=True)
        # box head: Conv2d(512,2048,k=7,s=7) on a 7x7 map == FC over (ph,pw,c) of the NHWC pooled tile
        self.p["RCNN_top.0"] = PackedConv(2048, 7 * 7 * 512, 1, 1, 0, None, empty(2048), h, dev)
        conv("RCNN_top.3", 0)
        for i in range(0, 12, 2):
            conv("RCNN_kpts.%d" % i, 1)
        # ConvTranspose2d(256,256,2,2): out[2i+a,2j+b] = W[:,:,a,b]^T x[i,j]  -> four 1x1 convs
        self.deconv = [[PackedConv(256, 256, 1, 1, 0, None, empty(256), h, dev) for b in range(2)] for a in range(2)]
        self.kpts_class = (empty(6, 256), empty(6))
        self.fc = [empty(*sd[k].shape) for k in _FC]
        self._pack_from_host(self._pack_targets()[0])

    # ------------------------------------------------------------------ helpers
    def _conv(self, x, pc, relu=False, stride=1, residual=None, up_src=None, out=None, out_coff=0,
              out_strides=None, tag=None, out_mode=ops.EXACT, res_biased=False, in_biased=False,
              f32=True, f16=False, out16=None):
        """x fp32 (tf32 / simt modes) or fp16 (fp16 mode).  Returns the fp32 output, the fp16 twin, or both."""
        N, H, W = x.shape[:3]
        Ho = (H + 2 * pc.pad - pc.kh) // stride + 1
        Wo = (W + 2 * pc.pad - pc.kw) // stride + 1
        half_in = x.dtype == torch.float16
        if out is None and f32:
            out = torch.empty(N, Ho, Wo, pc.Cout, dtype=torch.float32, device=x.device)
        if out16 is None and f16:
            out16 = torch.empty(N, Ho, Wo, pc.Cout, dtype=torch.float16, device=x.device)
        if self.exact or half_in:
            out_mode, res_biased, in_biased = ops.EXACT, False, False
        d = ops.conv_desc(x, pc.w16 if half_in else pc.w, out, pc.Cin, pc.Cout, pc.kh,
                          pc.kw, stride, pc.pad, Ho, Wo, scale=pc.scale, shift=pc.shift, residual=residual,
                          up_src=up_src, relu=relu, out_coff=out_coff, out_strides=out_strides, out_mode=out_mode,
                          res_biased=res_biased, in_biased=in_biased, out16=out16)
        if half_in and pc.kh == 3 and stride == 1 and residual is None and up_src is None:
            # fp16 3x3: flat 128-pixel tiles by TMA im2col, the same bits as the 8x16 patches of sb_conv2d_tc without
            # their MMA rows past the map edges.  Recorded as "tc": bench.py's roofline re-launches the descriptor
            # through sb_conv2d_tc, so it times these convs on patches.
            ops.conv2d_rows(d)
            impl = "tc"
        else:
            impl = ops.conv2d(d, "tc" if half_in else self.conv_impl)
        if self.record is not None:
            self.record.append((d, impl, (x, out, out16, residual, up_src)))
        if tag is not None:
            self.impl_used[tag] = impl + ("16" if half_in else "")
        if out is not None and out16 is not None:
            return out, out16
        return out if out is not None else out16

    def _bottleneck(self, x, prefix, stride, has_ds):
        """resnet.py:82-102; the stride sits on the 1x1 conv1 and on the downsample (Q1)"""
        # TF32 hygiene: the residual stream x is stored "pre-biased" (exact fp32 + 0x1000): the tensor core's
        # truncation of it is then round-to-nearest, and the residual add un-biases it exactly.  Tensors
        # read only by the next conv (o1, o2) are stored rounded to TF32.
        xin = ops.subsample2(x) if stride == 2 else x
        o = self._conv(xin, self.p[prefix + ".conv1"], relu=True, tag=prefix + ".conv1", out_mode=ops.ROUND_TF32,
                       in_biased=True)
        o = self._conv(o, self.p[prefix + ".conv2"], relu=True, tag=prefix + ".conv2", out_mode=ops.ROUND_TF32)
        if has_ds:
            res = self._conv(xin, self.p[prefix + ".downsample.0"], tag=prefix + ".ds", in_biased=True)
        else:
            res = x
        return self._conv(o, self.p[prefix + ".conv3"], relu=True, residual=res, tag=prefix + ".conv3",
                          out_mode=ops.BIASED, res_biased=not has_ds)

    def _bottleneck16(self, x32, x16, prefix, stride, has_ds, out=None, saved=None):
        """fp16-operand variant: convs read fp16 twins, the residual stream itself stays exact fp32.
        out = (fp32 view, fp16 view) to write the block output into (slices of a batched tensor).
        saved: dict that receives the conv inputs the backward needs (fp16 twins, all ReLU'd)"""
        xin = ops.subsample2(x16) if stride == 2 else x16
        o1 = self._conv(xin, self.p[prefix + ".conv1"], relu=True, tag=prefix + ".conv1", f32=False, f16=True)
        o = self._conv(o1, self.p[prefix + ".conv2"], relu=True, tag=prefix + ".conv2", f32=False, f16=True)
        res = self._conv(xin, self.p[prefix + ".downsample.0"], tag=prefix + ".ds") if has_ds else x32
        if saved is not None:
            saved[prefix] = dict(xin=xin, o1=o1, o2=o)
        if out is not None:
            return self._conv(o, self.p[prefix + ".conv3"], relu=True, residual=res, tag=prefix + ".conv3",
                              out=out[0], out16=out[1])
        return self._conv(o, self.p[prefix + ".conv3"], relu=True, residual=res, tag=prefix + ".conv3", f16=True)

    def trunk_fpn(self, im_nchw, save_for_backward=False):
        """images [N,3,H,W] NCHW -> dict of NHWC C2..C5, P2..P6 (stereo_rcnn.py:155-168).
        save_for_backward=True (fp16-operand engines) returns (feats, saved): `saved` keeps the conv inputs (the fp16
        twins the forward consumed, all ReLU'd) that trunk_fpn_backward needs.  The left and the right image then run
        layers 3-4 as one batched chain; every value computed is the same."""
        if self.half:
            return self._trunk_fpn16(im_nchw, save_for_backward)
        if save_for_backward:
            raise ValueError("the backward pass runs on fp16 conv operands: build the engine with precision='fp16'")
        if self.exact:
            c0 = ops.stem_conv(im_nchw, *self.stem, out_mode=ops.EXACT)
        else:       # patch matrix (pixels rounded to TF32) + tensor-core GEMM
            c0 = self._conv(ops.stem_im2col(im_nchw), self.p["stem_gemm"], relu=True, out_mode=ops.BIASED, tag="stem")
        c1 = ops.maxpool3x3s2_ceil(c0)                      # max() commutes with the monotone pre-bias
        feats = {"c1": c1}
        x = c1
        for li, nb in enumerate(LAYERS):
            for bi in range(nb):
                x = self._bottleneck(x, "RCNN_layer%d.0.%d" % (li + 1, bi), STRIDES[li] if bi == 0 else 1, bi == 0)
            feats["c%d" % (li + 2)] = x
        R = ops.ROUND_TF32
        p5 = self._conv(feats["c5"], self.p["RCNN_toplayer"], tag="toplayer", in_biased=True)
        t = self._conv(feats["c4"], self.p["RCNN_latlayer1"], up_src=p5, tag="lat1", out_mode=R, in_biased=True)
        p4 = self._conv(t, self.p["RCNN_smooth1"], tag="smooth1")          # lateral + upsample-add fused above
        t = self._conv(feats["c3"], self.p["RCNN_latlayer2"], up_src=p4, tag="lat2", out_mode=R, in_biased=True)
        p3 = self._conv(t, self.p["RCNN_smooth2"], tag="smooth2")
        t = self._conv(feats["c2"], self.p["RCNN_latlayer3"], up_src=p3, tag="lat3", out_mode=R, in_biased=True)
        p2 = self._conv(t, self.p["RCNN_smooth3"], tag="smooth3")
        p6 = ops.subsample2(p5)                                                           # Q5
        feats.update(p2=p2, p3=p3, p4=p4, p5=p5, p6=p6)
        return feats

    def _trunk_fpn16(self, im_nchw, save_for_backward=False):
        """fp16-operand trunk: every conv input is an fp16 tensor (half the HBM bytes, f16 = 2x the TF32
        MMA rate, same 11-bit significand); fp32 copies exist only where a non-conv consumer needs them
        (residual adds, FPN upsample source, RoIAlign, the user-visible P levels)."""
        # patches gathered inside the GEMM kernel (no 229 MB patch matrix); self.stem[1:] is the folded BN scale, shift
        c0 = ops.stem_conv_tc(im_nchw, self.stem_w16, *self.stem[1:])
        self.impl_used["stem"] = "tc16-fused"
        c1 = ops.maxpool3x3s2_ceil(c0)
        feats = {"c1": c1.float() if self.keep32 else None, "c1_16": c1}
        saved = {} if save_for_backward else None
        x32, x16 = None, c1
        for li in (0, 1):                           # layers 1-2: left and right batched (hundreds of tiles)
            for bi in range(LAYERS[li]):
                x32, x16 = self._bottleneck16(x32, x16, "RCNN_layer%d.0.%d" % (li + 1, bi),
                                              STRIDES[li] if bi == 0 else 1, bi == 0, saved=saved)
            feats["c%d" % (li + 2)], feats["c%d_16" % (li + 2)] = x32, x16
        # layers 3-4 have 38 / 10 row tiles per image: far too few to fill 132 SMs, and every launch is latency
        # bound (prologue + load latency + main loop + epilogue back to back).  The left and the right image are
        # independent, so they run as two concurrent chains on two streams (two parallel branches of the CUDA
        # graph): the chains' latencies overlap and together they still need only ~76 SMs.
        N = x16.shape[0]
        B = N // 2
        dev = x16.device

        def out_bufs(li):
            h, w = x16.shape[1], x16.shape[2]
            for _ in range(li - 1):
                h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
            c = PLANES[li] * 4
            return (torch.empty(N, h, w, c, dtype=torch.float32, device=dev),
                    torch.empty(N, h, w, c, dtype=torch.float16, device=dev))
        c4 = out_bufs(2)
        c5 = out_bufs(3)

        def chain(sl):
            y32, y16 = x32[sl], x16[sl]
            for li, dst in ((2, c4), (3, c5)):
                for bi in range(LAYERS[li]):
                    last = bi == LAYERS[li] - 1
                    y32, y16 = self._bottleneck16(y32, y16, "RCNN_layer%d.0.%d" % (li + 1, bi),
                                                  STRIDES[li] if bi == 0 else 1, bi == 0,
                                                  out=(dst[0][sl], dst[1][sl]) if last else None, saved=saved)
        if self.side is not None and self.forks and saved is None:
            main = torch.cuda.current_stream()
            self.side.wait_stream(main)
            with torch.cuda.stream(self.side):
                chain(slice(B, N))
            chain(slice(0, B))
            main.wait_stream(self.side)
        else:
            chain(slice(0, N))
        feats.update(c4=c4[0], c4_16=c4[1], c5=c5[0], c5_16=c5[1])
        p5, p5h = self._conv(feats["c5_16"], self.p["RCNN_toplayer"], tag="toplayer", f16=True)
        t4 = self._conv(feats["c4_16"], self.p["RCNN_latlayer1"], up_src=p5, tag="lat1", f32=False, f16=True)
        p4, p4h = self._conv(t4, self.p["RCNN_smooth1"], tag="smooth1", f16=True)
        t3 = self._conv(feats["c3_16"], self.p["RCNN_latlayer2"], up_src=p4, tag="lat2", f32=False, f16=True)
        p3, p3h = self._conv(t3, self.p["RCNN_smooth2"], tag="smooth2", f16=True)
        t2 = self._conv(feats["c2_16"], self.p["RCNN_latlayer3"], up_src=p3, tag="lat3", f32=False, f16=True)
        p2, p2h = self._conv(t2, self.p["RCNN_smooth3"], tag="smooth3", f16=True)
        feats.update(p2=p2, p3=p3, p4=p4, p5=p5, p6=ops.subsample2(p5), p2_16=p2h, p3_16=p3h, p4_16=p4h,
                     p5_16=p5h, p6_16=ops.subsample2(p5h))
        if saved is not None:
            saved.update(c2=feats["c2_16"], c3=feats["c3_16"], c4=feats["c4_16"], c5=feats["c5_16"], t2=t2, t3=t3,
                         t4=t4)
            return feats, saved
        return feats

    # ------------------------------------------------------------------ backward of the trunk + FPN
    def _pack_backward(self, heads=False):
        """the data-gradient copies {key: _DgradConv}, allocated and packed from the host masters on first use: those
        of the trunk, FPN and RPN convs, and with heads=True also the two of the R-CNN heads with their own layout"""
        if self._bwd is None:
            self._bwd = {}
            self._found_inf = torch.zeros(4, dtype=torch.int32, device=self.device)   # [0]; sb_fill writes 4-word units
        dev, new = self.device, {}
        if "rpn_heads" not in self._bwd:
            for k, pc in self.p.items():
                if k not in ("stem_gemm", "rpn_heads", "RCNN_top.0"):
                    new[k] = _DgradConv(pc.Cout, pc.Cin, pc.kh, pc.kw, pc.pad, dev)
            new["rpn_heads"] = _DgradConv(64, 1024, 1, 1, 0, dev, zeroed=True)   # K = 64 rows, 24..63 zero
        if heads and "deconv" not in self._bwd:
            # RCNN_top.0 as the forward's 1x1 conv over (ph, pw, c) (103 MB), and the deconv as one 1x1 conv
            # 256 -> 1024 whose output channel (a, b, co) is phase (a, b) of output channel co
            new["RCNN_top.0"] = _DgradConv(2048, 7 * 7 * 512, 1, 1, 0, dev)
            new["deconv"] = _DgradConv(1024, 256, 1, 1, 0, dev)
        if new:
            self._bwd.update(new)
            self._pack_from_host(self._pack_targets(new)[1])
        return self._bwd

    @property
    def found_inf(self):
        """int32 [1] device flag: 1 when the last backward (rpn_backward, trunk_fpn_backward) produced a non-finite
        gradient (cleared at the start of every backward unless it is told to keep it, never read on the host here --
        torch.cuda.amp.GradScaler's found_inf)"""
        self._pack_backward()
        return self._found_inf[:1]

    def _dgrad(self, dy16, key, out=None, out16=None, residual=None, mask=None, out_strides=None, f32=True,
               f16=True):
        """input gradient of conv `key` from the fp16 output gradient dy16 (stride 1; stride-2 callers scatter
        through out / out_strides)"""
        pc = self._bwd[key]
        N, H, W = dy16.shape[:3]
        if out is None and f32:
            out = torch.empty(N, H, W, pc.Cout, dtype=torch.float32, device=dy16.device)
        if out16 is None and f16:
            out16 = torch.empty(N, H, W, pc.Cout, dtype=torch.float16, device=dy16.device)
        d = ops.conv_desc(dy16, pc.w16, out, pc.Cin, pc.Cout, pc.kh, pc.kw, 1, pc.pad, H, W, residual=residual,
                          out16=out16, out_strides=out_strides)
        ops.conv2d_dgrad(d, mask)
        return out, out16

    def _wgrad(self, grads, key, dy16, x16, gs, dy32=None):
        pc = self.p[key]
        ops.conv_wgrad(dy16, x16, pc.kh, grads[key + ".weight"], scale=pc.scale if dy32 is None else None,
                       grad_scale=gs, dy32=dy32, db=grads[key + ".bias"] if dy32 is not None else None,
                       nonfinite=self._found_inf)

    def _grad_buffers(self, params, grads):
        out = {}
        for name, shape in params:
            g = grads.get(name) if grads is not None else None
            if g is None:
                g = torch.empty(shape, dtype=torch.float32, device=self.device)
            assert tuple(g.shape) == tuple(shape) and g.dtype == torch.float32 and g.is_contiguous(), name
            out[name] = g
        return out

    def trunk_fpn_backward(self, saved, d_feats, fixed_blocks=1, grads=None, grad_scale=1.0, clear_found_inf=True):
        """Backward of trunk_fpn (ResNet-101 layers 1-4 + FPN, frozen BN) for the gradients d_feats["p2".."p6"] (fp32
        NHWC, the shapes trunk_fpn returns; left and right images batched, so every weight gradient sums over both).
        Returns {state_dict name: fp32 gradient} of exactly trainable_trunk_fpn_params(fixed_blocks), in the
        reference's layout; tensors given in `grads` (e.g. GradientBuckets views) are written in place.
        grad_scale (a power of two) multiplies dP before the fp16 chain and is divided out of the results exactly; it is
        a host float, or an fp32 [1] CUDA tensor that every kernel reads on the device (a captured backward then follows
        a scale changed between replays).  found_inf is set when a result is not finite; clear_found_inf=False keeps a
        flag an earlier backward of the same step set (rpn_backward before this).  No host synchronisation:
        graph-capturable."""
        self._pack_backward()
        dev = self.device
        gs = grad_scale if ops.device_scale(grad_scale) else float(grad_scale)
        out = self._grad_buffers(trainable_trunk_fpn_params(fixed_blocks), grads)
        if clear_found_inf:
            ops.fill_(self._found_inf, 0.0)
        dp = {k: ops._f32c(d_feats[k]) for k in ("p2", "p3", "p4", "p5", "p6")}
        # ---- FPN (stereo_rcnn.py:155-168): P2 <- smooth3(lat3(c2) + up(P3)) ... P5 = toplayer(c5), P6 = P5[::2, ::2]
        g32, g16 = ops.fpn_grad_combine(dp["p2"], scale=gs)
        dt = {}
        for lvl, smooth, lat, tk, ck in ((2, "RCNN_smooth3", "RCNN_latlayer3", "t2", "c2"),
                                         (3, "RCNN_smooth2", "RCNN_latlayer2", "t3", "c3"),
                                         (4, "RCNN_smooth1", "RCNN_latlayer1", "t4", "c4")):
            self._wgrad(out, smooth, g16, saved[tk], gs, dy32=g32)
            t32, t16 = self._dgrad(g16, smooth)
            self._wgrad(out, lat, t16, saved[ck], gs, dy32=t32)
            dt["dt%d" % lvl] = t16
            g32, g16 = ops.fpn_grad_combine(dp["p%d" % (lvl + 1)], dt=t32, dp6=dp["p6"] if lvl == 4 else None,
                                            scale=gs)
        self._wgrad(out, "RCNN_toplayer", g16, saved["c5"], gs, dy32=g32)
        # gradient at the pre-ReLU sum of layer 4's last block: toplayer's input gradient masked by c5 > 0
        g32, g16 = self._dgrad(g16, "RCNN_toplayer", mask=saved["c5"])
        # ---- trunk (resnet.py:66-102, stride on conv1 and the downsample), top layer first
        for li in range(3, fixed_blocks - 1, -1):
            for bi in range(LAYERS[li] - 1, -1, -1):
                p = "RCNN_layer%d.0.%d" % (li + 1, bi)
                r = saved[p]
                self._wgrad(out, p + ".conv3", g16, r["o2"], gs)
                _, g2 = self._dgrad(g16, p + ".conv3", mask=r["o2"], f32=False)
                self._wgrad(out, p + ".conv2", g2, r["o1"], gs)
                _, g1 = self._dgrad(g2, p + ".conv2", mask=r["o1"], f32=False)
                self._wgrad(out, p + ".conv1", g1, r["xin"], gs)
                if bi > 0:      # identity shortcut: input grad = conv1's + the block's own, masked by the input's ReLU
                    g32, g16 = self._dgrad(g1, p + ".conv1", residual=g32, mask=r["xin"])
                    continue
                self._wgrad(out, p + ".downsample.0", g16, r["xin"], gs)
                if li <= fixed_blocks:      # the layer below is frozen: no gradient into its output
                    break
                # stride-2 first block: conv1 + downsample input gradients at the strided pixels, scattered into the
                # even positions of the input (subsample2's backward); the lateral conv reading the same tensor
                # adds its part and the input's ReLU mask applies
                ds32, _ = self._dgrad(g16, p + ".downsample.0", f16=False)
                lat, dtk = _LATERAL_OF_INPUT[li]
                xf = saved["c%d" % (li + 1)]
                N, Hf, Wf, C = xf.shape
                scat = ops.fill_(torch.empty(N, Hf, Wf, C, dtype=torch.float32, device=dev), 0.0)
                self._dgrad(g1, p + ".conv1", out=scat, residual=ds32, f16=False,
                            out_strides=(Hf * Wf * C, 2 * Wf * C, 2 * C))
                g32, g16 = self._dgrad(dt[dtk], lat, residual=scat, mask=xf)
        return out

    def rpn(self, feats, B, save_for_backward=False):
        """stereo_rpn.py:73-95 -> cls_prob [B,A,2], bbox_pred [B,A,6], level shapes.
        save_for_backward=True (fp16-operand engines) also returns an RpnSaved for rpn_backward and the raw class
        scores rpn_cls_score [B,A,2] the RPN loss reads; cls_prob and bbox_pred are the same bits either way."""
        if save_for_backward and not self.half:
            raise ValueError("the backward pass runs on fp16 conv operands: build the engine with precision='fp16'")
        sfx = "_16" if self.half else ""
        levels = [feats[k + sfx] for k in ("p2", "p3", "p4", "p5", "p6")]
        shapes = [[f.shape[1], f.shape[2]] for f in levels]
        P = sum(h * w for h, w in shapes)
        dev = self.device
        head = torch.empty(B, P, 32, dtype=torch.float32, device=dev)
        offs = [0]
        for h, w in shapes:
            offs.append(offs[-1] + h * w)
        # saved for the backward: allocated here on the current stream, not inside the side-stream fork below
        cats = ([torch.empty(B, h, w, 1024, dtype=torch.float16, device=dev) for h, w in shapes]
                if save_for_backward else [None] * len(shapes))

        def level(f, h, w, off, cat=None):
            if cat is None:
                cat = torch.empty(B, h, w, 1024, dtype=f.dtype, device=dev)
            kw = dict(f32=False, out16=cat) if self.half else dict(out=cat, out_mode=ops.ROUND_TF32)
            if B == 1:      # L and R in one launch: image index n = side -> channel offset n * 512
                self._conv(f, self.p["RCNN_rpn.RPN_Conv"], relu=True, out_strides=(512, w * 1024, 1024),
                           tag="rpn_conv", **kw)
            else:
                for side in range(2):   # shared RPN_Conv on L then R, channel-concatenated (Q6)
                    self._conv(f[side * B:(side + 1) * B], self.p["RCNN_rpn.RPN_Conv"], relu=True,
                               out_coff=side * 512, out_strides=(h * w * 1024, w * 1024, 1024), tag="rpn_conv", **kw)
            self._conv(cat, self.p["rpn_heads"], out=head[:, off:off + h * w],
                       out_strides=(P * 32, w * 32, 32), tag="rpn_heads")
        fork = self.side is not None and self.forks
        if fork:    # the three coarse levels are a handful of tiles each: run them beside the p2 / p3 convs
            main = torch.cuda.current_stream()
            self.side.wait_stream(main)
            with torch.cuda.stream(self.side):
                for i in (2, 3, 4):
                    level(levels[i], shapes[i][0], shapes[i][1], offs[i], cats[i])
        for i in ((0, 1) if fork else range(5)):
            level(levels[i], shapes[i][0], shapes[i][1], offs[i], cats[i])
        if fork:
            main.wait_stream(self.side)
        cls_prob, bbox = ops.rpn_head_epilogue(head, B, P)
        if save_for_backward:
            return (cls_prob, bbox, shapes, RpnSaved(B, shapes, offs, cats, levels, head),
                    ops.rpn_head_scores(head, B, P))
        return cls_prob, bbox, shapes

    def rpn_backward(self, saved, d_cls_score, d_bbox_pred, grads=None, grad_scale=1.0):
        """Backward of rpn (stereo_rpn.py:73-95) for the RPN loss gradients d_cls_score [B,A,2] (w.r.t. the raw scores
        rpn returns) and d_bbox_pred [B,A,6].  Returns ({state_dict name: fp32 gradient} of exactly
        trainable_rpn_params(), in the reference's layout; tensors given in `grads` are written in place,
        {"p2".."p6": dP fp32 [2B,h,w,256]} for trunk_fpn_backward).  Weight gradients are summed over the levels
        P2..P6 and, for RPN_Conv, left before right: a fixed order, bit-identical run to run.  grad_scale (a power of
        two; a host float or an fp32 [1] CUDA tensor, as in trunk_fpn_backward) scales the fp16 chain and is divided out
        of every result exactly; found_inf is cleared, then set when a gradient is not finite.  No host
        synchronisation: graph-capturable."""
        self._pack_backward()
        dev = self.device
        on_dev = ops.device_scale(grad_scale)
        gs = grad_scale if on_dev else float(grad_scale)
        B, offs = saved.B, saved.offs
        P = offs[-1]
        out = self._grad_buffers(trainable_rpn_params(), grads)
        ops.fill_(self._found_inf, 0.0)
        dh16, dh32 = ops.rpn_head_grad(d_cls_score, d_bbox_pred, B, P, gs)
        # the dgrad epilogue's per-channel scale divides grad_scale out of dP (exact: a power of two); a device scale
        # is inverted on the device
        if on_dev:
            unscale = ops.fill_reciprocal_(torch.empty(256, dtype=torch.float32, device=dev), gs)
        else:
            unscale = ops.fill_(torch.empty(256, dtype=torch.float32, device=dev), 1.0 / gs) if gs != 1.0 else None
        hd, cd = self._bwd["rpn_heads"], self._bwd["RCNN_rpn.RPN_Conv"]
        w_cls, w_box = out["RCNN_rpn.RPN_cls_score.weight"], out["RCNN_rpn.RPN_bbox_pred_left_right.weight"]
        b_cls, b_box = out["RCNN_rpn.RPN_cls_score.bias"], out["RCNN_rpn.RPN_bbox_pred_left_right.bias"]
        w_conv, b_conv = out["RCNN_rpn.RPN_Conv.weight"], out["RCNN_rpn.RPN_Conv.bias"]
        dps = {}
        for i, (h, w) in enumerate(saved.shapes):
            cat, f16 = saved.cats[i], saved.levels[i]
            dcat32 = torch.empty(B, h, w, 1024, dtype=torch.float32, device=dev)
            dcat16 = torch.empty(B, h, w, 1024, dtype=torch.float16, device=dev)
            for b in range(B):
                # fused 1x1 head: dW / db rows 0..5 -> RPN_cls_score, 6..23 -> RPN_bbox_pred_left_right
                dy16 = dh16[b, offs[i]:offs[i + 1]].view(1, h, w, 64)
                dy32 = dh32[b, offs[i]:offs[i + 1]].view(1, h, w, 64)
                ops.conv_wgrad_acc(dy16, cat[b:b + 1], 1, w_cls, db=b_cls, dy32=dy32, grad_scale=gs,
                                   accumulate=i > 0 or b > 0, rows=24, split=6, dw_hi=w_box, db_hi=b_box,
                                   nonfinite=self._found_inf)
                # d cat = head^T dhead where cat > 0 (the ReLU of RPN_Conv; cat has the output's layout)
                d = ops.conv_desc(dy16, hd.w16, dcat32[b:b + 1], hd.Cin, hd.Cout, 1, 1, 1, 0, h, w,
                                  out16=dcat16[b:b + 1])
                ops.conv2d_dgrad(d, cat[b:b + 1])
            dp = torch.empty(2 * B, h, w, 256, dtype=torch.float32, device=dev)
            for side in range(2):       # RPN_Conv on L then R: channel halves 0..511 and 512..1023 of d cat
                c0 = side * 512
                ops.conv_wgrad_acc(dcat16[..., c0:c0 + 512], f16[side * B:(side + 1) * B], 3, w_conv, db=b_conv,
                                   dy32=dcat32[..., c0:c0 + 512], grad_scale=gs, accumulate=i > 0 or side > 0,
                                   nonfinite=self._found_inf)
                d = ops.conv_desc(dcat16[..., c0:c0 + 512], cd.w16, dp[side * B:(side + 1) * B], cd.Cin, cd.Cout, 3, 3, 1, 1,
                                  h, w, scale=unscale, in_ld=1024)
                ops.conv2d_dgrad(d)
            dps[_LEVELS[i]] = dp
        return out, dps

    def heads(self, feats, B, rois_l, rois_r, im_h, save_for_backward=False, dropout_words=None):
        """stereo_rcnn.py:240-271 on flattened rois [R,5].
        save_for_backward=True (fp16-operand engines) returns (out, HeadsSaved) for heads_backward; out then also holds
        the raw predictions the R-CNN loss reads: cls_score [R,C], kpts_pred [R,4G], left_border_pred and
        right_border_pred [R,G].  Every other output is the same bits either way.
        dropout_words (int32 [2,R,2048], train.random_words; fp16-operand engines) applies the training-mode
        Dropout(p=0.2) after each ReLU of RCNN_top: element i of RCNN_top.0's output (words[0]) and of fc7 (words[1])
        is dropped when its word, read as uint32, is < 0.2 2^32, and scaled by 1.25 otherwise.  The explicit words
        replace torch's RNG stream, as the samplers' do (DESIGN 4.4): the one deliberate difference from the
        reference's dropout."""
        if (save_for_backward or dropout_words is not None) and not self.half:
            raise ValueError("the backward pass runs on fp16 conv operands: build the engine with precision='fp16'")
        mk = ("p2", "p3", "p4", "p5")
        fl = [feats[k][:B] for k in mk]
        fr = [feats[k][B:] for k in mk]
        R = rois_l.shape[0]
        dev = self.device
        h = self.half
        adt = torch.float16 if h else torch.float32
        rt = not self.exact and not h
        c16 = dict(f32=False, f16=True) if h else {}
        if dropout_words is not None:
            assert dropout_words.dtype == torch.int32 and dropout_words.is_contiguous()
            assert tuple(dropout_words.shape) == (2, R, 2048) and dropout_words.is_cuda
        nc = self.n_classes
        # saved for the backward and read by the loss: allocated here on the current stream, not inside the side-stream
        # fork below
        train = None
        if save_for_backward:
            f32 = lambda *sh: torch.empty(*sh, dtype=torch.float32, device=dev)
            train = dict(pooled=torch.empty(R, 7, 7, 512, dtype=adt, device=dev),
                         top0=torch.empty(R, 1, 1, 2048, dtype=adt, device=dev), fc7=f32(R, 1, 1, 2048),
                         tail=(f32(R, nc), f32(R, 6 * nc), f32(R, 5 * nc), f32(R, nc)))

        def box_head():
            pooled = train["pooled"] if train else torch.empty(R, 7, 7, 512, dtype=adt, device=dev)
            ops.roi_align_pyramid_nhwc(fl, im_h, rois_l, 7, out=pooled, out_coff=0, round_tf32=rt, half=h)
            ops.roi_align_pyramid_nhwc(fr, im_h, rois_r, 7, out=pooled, out_coff=256, round_tf32=rt, half=h)
            top0 = dict(out16=train["top0"]) if train else {}
            x = self._conv(pooled.view(R, 1, 1, 7 * 7 * 512), self.p["RCNN_top.0"], relu=True, tag="top0",
                           out_mode=ops.ROUND_TF32, **c16, **top0)
            if dropout_words is not None:
                ops.dropout_words_(x, dropout_words[0], DROPOUT_P)
            fc7 = self._conv(x, self.p["RCNN_top.3"], relu=True, tag="top3",
                             out=train["fc7"] if train else None).view(R, 2048)
            if dropout_words is not None:
                ops.dropout_words_(fc7, dropout_words[1], DROPOUT_P)
            if train:
                return (pooled, fc7, x) + ops.box_tail_scores(fc7, *self.fc, n_classes=nc, out=train["tail"])
            return (pooled, fc7, x) + tuple(ops.box_tail(fc7, *self.fc, n_classes=nc)) + (None,)
        fork = self.side is not None and self.forks
        if fork:    # the box head (two FCs with 3 row tiles) is latency-bound: run it beside the keypoint convs
            main = torch.cuda.current_stream()
            self.side.wait_stream(main)
            with torch.cuda.stream(self.side):
                pooled, fc7, top0, cls_prob, bbox, dim, score = box_head()
        else:
            pooled, fc7, top0, cls_prob, bbox, dim, score = box_head()
        pk = ops.roi_align_pyramid_nhwc(fl, im_h, rois_l, 14, round_tf32=rt, half=h)
        x = pk
        kpts = []
        for i in range(0, 12, 2):
            x = self._conv(x, self.p["RCNN_kpts.%d" % i], relu=True, tag="kpts%d" % i, out_mode=ops.ROUND_TF32, **c16)
            kpts.append(x)
        up = torch.empty(R, 28, 28, 256, dtype=adt, device=dev)
        for a in range(2):
            for b in range(2):
                kw = dict(f32=False, out16=up[:, a:, b:]) if h else dict(out=up[:, a:, b:])
                self._conv(x, self.deconv[a][b], relu=True, out_strides=(28 * 28 * 256, 2 * 28 * 256, 2 * 256),
                           tag="deconv", **kw)
        kp, lb, rb, ka = ops.kpts_tail(up, *self.kpts_class, want_pred_all=True)
        if fork:
            main.wait_stream(self.side)
        out = dict(pooled_box=pooled, pooled_kpts=pk, fc7=fc7, cls_prob=cls_prob, bbox_pred=bbox,
                   dim_orien_pred=dim, kpts_prob=kp, left_border_prob=lb, right_border_prob=rb,
                   kpts_pred_all=ka)
        if not save_for_backward:
            return out
        kpred, lpred, rpred = ops.kpts_logits(ka)
        out.update(cls_score=score, kpts_pred=kpred, left_border_pred=lpred, right_border_pred=rpred)
        return out, HeadsSaved(R, dropout_words is not None, pooled, pk, top0, fc7, kpts, up, rois_l, rois_r,
                               float(im_h), B)

    # ------------------------------------------------------------------ backward of the R-CNN heads
    def _pack_heads_backward(self):
        return self._pack_backward(heads=True)

    def heads_backward(self, saved, d_cls_score, d_bbox_pred, d_dim_orien_pred, d_kpts_pred, d_left_border_pred,
                       d_right_border_pred, grads=None, grad_scale=1.0, clear_found_inf=True):
        """Backward of heads (resnet.py:256-286, stereo_rcnn.py:252-271) for the R-CNN loss gradients w.r.t. the raw
        predictions heads(save_for_backward=True) returns: d_cls_score [R,C], d_bbox_pred [R,6C], d_dim_orien_pred
        [R,5C], d_kpts_pred [R,4G], d_left_border_pred / d_right_border_pred [R,G] (fp32).
        Returns ({state_dict name: fp32 gradient} of exactly trainable_rcnn_head_params(n_classes), in the reference's
        layout; tensors given in `grads` are written in place,
        {"pooled_box": fp32 [R,7,7,512] (channels 0..255 the left image, 256..511 the right),
         "pooled_kpts": fp32 [R,14,14,256]}: the gradients of the two pooled tensors).
        Every sum runs in a fixed order: bit-identical run to run.  grad_scale (a power of two; a host float or an fp32
        [1] CUDA tensor, as in trunk_fpn_backward) scales the fp16 chain and is divided out of every result exactly;
        found_inf is cleared, then set when a gradient is not finite;
        clear_found_inf=False keeps a flag an earlier backward of the same step set (rpn_backward before this).
        No host synchronisation: graph-capturable."""
        self._pack_heads_backward()
        dev = self.device
        on_dev = ops.device_scale(grad_scale)
        gs = grad_scale if on_dev else float(grad_scale)
        R = saved.R
        out = self._grad_buffers(trainable_rcnn_head_params(self.n_classes), grads)
        nf = self._found_inf
        if clear_found_inf:
            ops.fill_(nf, 0.0)
        f32 = lambda *sh: torch.empty(*sh, dtype=torch.float32, device=dev)
        # the dgrad epilogue's per-channel scale divides grad_scale out of the pooled gradients (exact: a power of two);
        # a device scale is inverted on the device
        if on_dev:
            unscale = ops.fill_reciprocal_(f32(2048), gs)
        else:
            unscale = ops.fill_(f32(2048), 1.0 / gs) if gs != 1.0 else None
        # ---- box head: the three linears (fp32), then RCNN_top.3 and RCNN_top.0 as 1x1 convs over the R RoIs
        keep = 1.0 / (1.0 - DROPOUT_P) if saved.dropout else 1.0
        w_cls, _, w_box, _, w_dim, _ = self.fc
        tail = [out[k + s] for k in ("RCNN_cls_score", "RCNN_bbox_pred", "RCNN_dim_orien_pred")
                for s in (".weight", ".bias")]
        dz16, dz32 = ops.box_tail_backward(d_cls_score, d_bbox_pred, d_dim_orien_pred, saved.fc7, w_cls, w_box, w_dim,
                                           tail, mask_scale=keep, grad_scale=gs, nonfinite=nf)
        dz16, dz32 = dz16.view(R, 1, 1, 2048), dz32.view(R, 1, 1, 2048)
        self._wgrad(out, "RCNN_top.3", dz16, saved.top0, gs, dy32=dz32)
        # RCNN_top.0's pre-activation: top3^T dz where the saved post-dropout output is > 0 (ReLU and dropout mask),
        # times the dropout's 1 / (1 - p)
        t3 = self._bwd["RCNN_top.3"]
        d0_32, d0_16 = f32(R, 1, 1, 2048), torch.empty(R, 1, 1, 2048, dtype=torch.float16, device=dev)
        keep_v = ops.fill_(f32(2048), keep) if saved.dropout else None
        ops.conv2d_dgrad(ops.conv_desc(dz16, t3.w16, d0_32, t3.Cin, t3.Cout, 1, 1, 1, 0, 1, 1, scale=keep_v,
                                       out16=d0_16), saved.top0)
        pooled16 = saved.pooled_box.view(R, 1, 1, 7 * 7 * 512)
        g0 = f32(2048, 7 * 7 * 512, 1, 1)       # [co][(ph, pw, c)] -> the reference's [co][c][ph][pw] below
        ops.conv_wgrad(d0_16, pooled16, 1, g0, grad_scale=gs, dy32=d0_32, db=out["RCNN_top.0.bias"], nonfinite=nf)
        ops.permute3(g0, (2048, 49, 512), (49 * 512, 1, 49), out["RCNN_top.0.weight"])
        # d pooled_box = top0^T d0, in column blocks of at most 2048 output channels (the conv kernel's widest tile row)
        t0 = self._bwd["RCNN_top.0"]
        d_pooled = f32(R, 7, 7, 512)
        K0 = 7 * 7 * 512
        for c0 in range(0, K0, 2048):
            n = min(2048, K0 - c0)
            ops.conv2d_dgrad(ops.conv_desc(d0_16, t0.w16[c0:c0 + n], d_pooled, 2048, n, 1, 1, 1, 0, 1, 1,
                                           scale=unscale, out_coff=c0, out_strides=(K0, K0, K0)))
        # ---- keypoint head: kpts_class over the height-summed deconv output (fp32), the deconv, six 3x3 convs
        dup16 = ops.kpts_tail_backward(saved.up, self.kpts_class[0], d_kpts_pred, d_left_border_pred,
                                       d_right_border_pred, out["kpts_class.weight"], out["kpts_class.bias"],
                                       out["RCNN_kpts.12.bias"], grad_scale=gs, nonfinite=nf)
        x6 = saved.kpts[5]
        gd = f32(1024, 256, 1, 1)                   # [(a, b, co)][ci] -> the reference's [ci][co][a][b] below
        ops.conv_wgrad(dup16, x6, 1, gd, grad_scale=gs, nonfinite=nf)
        ops.permute3(gd, (4, 256, 256), (1, 4, 1024), out["RCNN_kpts.12.weight"])
        g32, g16 = self._dgrad(dup16, "deconv", mask=x6)
        for i in range(5, -1, -1):
            key = "RCNN_kpts.%d" % (2 * i)
            xin = saved.kpts[i - 1] if i > 0 else saved.pooled_kpts
            self._wgrad(out, key, g16, xin, gs, dy32=g32)
            if i > 0:
                g32, g16 = self._dgrad(g16, key, mask=xin)
        pc = self._bwd["RCNN_kpts.0"]
        d_pk = f32(R, 14, 14, 256)
        ops.conv2d_dgrad(ops.conv_desc(g16, pc.w16, d_pk, pc.Cin, pc.Cout, 3, 3, 1, 1, 14, 14, scale=unscale))
        return out, {"pooled_box": d_pooled, "pooled_kpts": d_pk}

    def roi_align_backward(self, saved_heads, d_pooled, d_feats):
        """Backward of the heads' three pyramid RoIAligns (stereo_rcnn.py:110-139): adds the gradients of the pooled
        tensors, d_pooled = heads_backward's {"pooled_box": [R,7,7,512], "pooled_kpts": [R,14,14,256]} (fp32), into
        d_feats["p2".."p5"] (fp32 NHWC [2B,h,w,256], e.g. rpn_backward's dP), in place and in one deterministic call:
        box channels 0..255 with rois_l into the left images, 256..511 with rois_r into the right images, and the
        keypoint pooling with rois_l into the left images.  Sets found_inf on a non-finite gradient, never clears it.
        No host synchronisation: graph-capturable.  -> d_feats"""
        self._pack_backward()
        s = saved_heads
        dp = [d_feats[k] for k in ("p2", "p3", "p4", "p5")]
        C = dp[0].shape[3]          # heads() pools the right image into channels C..2C-1 of pooled_box
        ops.roi_align_pyramid_backward(dp, s.im_h, [(d_pooled["pooled_box"], s.rois_l, 0, 0),
                                                    (d_pooled["pooled_box"], s.rois_r, C, s.B),
                                                    (d_pooled["pooled_kpts"], s.rois_l, 0, 0)],
                                       nonfinite=self._found_inf)
        return d_feats

    # ------------------------------------------------------------------ the packed weights
    def _pack_targets(self, dgrad=()):
        """Every packed copy of the weights, as sb_pack_targets that read the masters in the reference's layout:
        ({state_dict name: [_PackT]} of the forward's copies, {state_dict name: [_PackT]} of the data-gradient copies
        of the convs in `dgrad`, keys of self._bwd).  The forward's weights are TF32-rounded fp32 with an fp16 twin in
        fp16 engines (exact fp32 with conv_impl="simt"); the data gradient's are fp16."""
        L, tf = _lib, self._fwd_transform
        fw, dg = {}, {}

        def put(tg, name, *a, **k):
            tg.setdefault(name, []).append(_PackT(name, *a, **k))

        def flat(tg, name, dst, n, transform, **k):
            put(tg, name, dst, (1, 1, 1, n), (0, 0, 0, 1), (0, 0, 0, 1), transform, **k)

        # stem [64,3,7,7]: [64][7][7][3] fp32 (i1 = tap, i2 = co, i3 = ci); as 64 rows of the 147 taps in (ci, r, s)
        # order, the GEMM's [64,160] over sb_stem_im2col's patches and the fused stem's fp16 [64,192]
        name = "RCNN_layer0.0.weight"
        put(fw, name, self.stem[0], (1, 49, 64, 3), (0, 1, 147, 49), (0, 3, 147, 1), L.PACK_F32)
        sg = self.p["stem_gemm"]
        put(fw, name, sg.w, (1, 1, 64, 147), (0, 0, 147, 1), (0, 0, 160, 1), tf, dst16=sg.w16)
        put(fw, name, self.stem_w16, (1, 1, 64, 147), (0, 0, 147, 1), (0, 0, 192, 1), L.PACK_F16)
        # trunk, FPN, RPN_Conv, RCNN_top.3, RCNN_kpts.0..10: forward [Cout][kh][kw][Cin] (i1 = tap, i2 = co,
        # i3 = ci); data gradient [Cin][kh][kw][Cout], i1 = flipped tap t' (source tap T-1-t'), i2 = ci, i3 = co,
        # the frozen-BN scale folded in for the trunk convs
        for key, pc in self.p.items():
            if key in ("stem_gemm", "rpn_heads", "RCNN_top.0"):
                continue
            name, co, ci, T = key + ".weight", pc.Cout, pc.Cin, pc.kh * pc.kw
            if T == 1:
                flat(fw, name, pc.w, co * ci, tf, dst16=pc.w16)
            else:
                put(fw, name, pc.w, (1, T, co, ci), (0, 1, T * ci, T), (0, ci, T * ci, 1), tf, dst16=pc.w16)
            if pc.scale is None:
                flat(fw, key + ".bias", pc.shift, co, L.PACK_F32)
            if key in dgrad:
                put(dg, name, self._bwd[key].w16, (1, T, ci, co), (0, -1, T, ci * T), (0, co, T * co, 1),
                    L.PACK_F16 if pc.scale is None else L.PACK_SCALE_F16, src_offset=T - 1, scale=pc.scale)
        # RPN heads: rows 0..5 / 6..23 of the fused head, columns 0..5 / 6..23 of its 64-column data-gradient copy
        ph = self.p["rpn_heads"]
        for key, r0, n in (("RCNN_rpn.RPN_cls_score", 0, 6), ("RCNN_rpn.RPN_bbox_pred_left_right", 6, 18)):
            flat(fw, key + ".weight", ph.w, n * 1024, tf, dst_offset=r0 * 1024, dst16=ph.w16)
            flat(fw, key + ".bias", ph.shift, n, L.PACK_F32, dst_offset=r0)
            if "rpn_heads" in dgrad:
                put(dg, key + ".weight", self._bwd["rpn_heads"].w16, (1, 1, 1024, n), (0, 0, 1, 1024), (0, 0, 64, 1),
                    L.PACK_F16, dst_offset=r0)
        # RCNN_top.0 [2048,512,7,7]: forward [co][(ph, pw, c)], data gradient [(ph, pw, c)][co]
        pt = self.p["RCNN_top.0"]
        put(fw, "RCNN_top.0.weight", pt.w, (1, 49, 2048, 512), (0, 1, 49 * 512, 49), (0, 512, 49 * 512, 1), tf,
            dst16=pt.w16)
        flat(fw, "RCNN_top.0.bias", pt.shift, 2048, L.PACK_F32)
        if "RCNN_top.0" in dgrad:
            put(dg, "RCNN_top.0.weight", self._bwd["RCNN_top.0"].w16, (1, 49, 512, 2048), (0, 1, 49, 49 * 512),
                (0, 512 * 2048, 2048, 1), L.PACK_F16)
        # deconv [Cin,Cout,2,2]: phase (a, b) forward [co][ci] = W[ci, co, a, b]; data gradient [ci][(a, b, co)]
        name = "RCNN_kpts.12.weight"
        for a in range(2):
            for b in range(2):
                pc = self.deconv[a][b]
                put(fw, name, pc.w, (1, 256, 1, 256), (0, 4, 0, 1024), (0, 256, 0, 1), tf, src_offset=2 * a + b,
                    dst16=pc.w16)
                flat(fw, "RCNN_kpts.12.bias", pc.shift, 256, L.PACK_F32)
        if "deconv" in dgrad:
            put(dg, name, self._bwd["deconv"].w16, (1, 4, 256, 256), (0, 1, 1024, 4), (0, 256, 1024, 1), L.PACK_F16)
        # the fp32 linears and kpts_class: plain copies
        for key, dst in zip(_FC + ("kpts_class.weight", "kpts_class.bias"), self.fc + list(self.kpts_class)):
            flat(fw, key, dst, dst.numel(), L.PACK_F32)
        return fw, dg

    @property
    def _fwd_transform(self):
        return _lib.PACK_F32 if self.exact else _lib.PACK_TF32

    def _table(self, items, srcs):
        """the planned host table of pack targets `items` reading srcs[name], and its device copy"""
        L = _lib
        for tp in items:
            shape = (64, 3, 7, 7) if tp.name == "RCNN_layer0.0.weight" else self._trainable[tp.name]
            assert srcs[tp.name].numel() == _numel(shape), tp.name
        tab = (L.PackTarget * len(items))()
        for i, tp in enumerate(items):
            tp.fill(tab[i], srcs[tp.name])
        n_tiles = ctypes.c_longlong()
        L.check(L.load().sb_pack_plan(tab, len(items), ctypes.byref(n_tiles)), "sb_pack_plan")
        return tab, torch.frombuffer(bytearray(memoryview(tab).cast("B")), dtype=torch.uint8).to(self.device)

    def _pack_from_host(self, tg):
        """pack the targets {name: [_PackT]} in one launch from the host masters, uploaded for it and then dropped"""
        L = _lib
        with torch.cuda.device(self.device):
            srcs = {n: self._masters[n].to(self.device) for n in tg}
            tab, dev = self._table([tp for ts in tg.values() for tp in ts], srcs)
            L.check(L.load().sb_pack_weights(tab, ops.ptr(dev), len(tab), L.stream_ptr()), "sb_pack_weights")

    def refresh_weights(self, params):
        """Rewrite, in place and on the device, every copy this engine holds of the parameters in `params`
        ({state_dict name: fp32 contiguous device tensor in the reference's layout}, any subset of the trainable
        names): the forward's packed weights (TF32-rounded fp32 and fp16), the data gradient's transposed fp16
        copies (taps flipped, frozen-BN scale folded in), the fused RPN head and its data-gradient copy, the
        (ph, pw, c)-ordered RCNN_top.0, the four deconv phases, biases, the linears and kpts_class.  The targets are
        the ones the constructor and the first backward pack from, so the result is bit-identical to a new engine
        built from the same values.  No tensor is reallocated, so CUDA graphs captured over the forward or backward
        stay valid.  Frozen tensors (the stem, frozen layers, the BN scale and shift) are never written.
        One launch (sb_pack_weights).  The table of a new set of (name, tensor) pairs is built and uploaded on first
        use: make that first call outside any graph capture; later calls with the same tensors are
        graph-capturable and do not synchronise."""
        L = _lib
        if not hasattr(self, "_refresh_cache"):
            self._refresh_cache = {}
            # the data-gradient copies first: packed later from the host masters, they would miss this refresh
            self._pack_heads_backward()
            fw, dg = self._pack_targets(self._bwd)
            self._refresh_tg = {n: fw[n] + dg.get(n, []) for n in self._trainable}
        for n, t in params.items():
            if n not in self._refresh_tg:
                raise KeyError("not a trainable parameter of this engine: %s" % n)
            assert t.dtype == torch.float32 and t.is_contiguous() and t.device.type == self.device.type, n
        key = tuple(sorted((n, t.data_ptr()) for n, t in params.items()))
        ent = self._refresh_cache.get(key)
        if ent is None:
            tab, dev = self._table([tp for n in sorted(params) for tp in self._refresh_tg[n]], params)
            ent = self._refresh_cache[key] = (tab, dev, [params[n] for n in sorted(params)])
        tab, dev, _keep = ent
        L.check(L.load().sb_pack_weights(tab, ops.ptr(dev), len(tab), L.stream_ptr()), "sb_pack_weights")

    @torch.no_grad()
    def forward(self, im_left, im_right, im_info, cfg_key="TEST", keep_features=False, im_h=None,
                before_proposals=None):
        """im_left/right [B,3,H,W] NCHW fp32 (BGR - means), im_info [B,3] (device) -> dict (the reference's
        tuple order is produced by model.stereo_rcnn.resnet.resnet.forward).  `im_h` (= im_info[0][0],
        stereo_rcnn.py:128) is taken from the tensor shape so that no device->host read is needed."""
        B = im_left.shape[0]
        im_h = float(im_left.shape[2]) if im_h is None else float(im_h)
        im = torch.cat((im_left, im_right), 0).contiguous()
        feats = self.trunk_fpn(im)
        cls_prob, bbox, shapes = self.rpn(feats, B)
        if before_proposals is not None:
            # the proposal stage is a chain of small, partly single-CTA kernels: callers fork independent work
            # (e.g. dense_align of the previous detections) onto a second stream here so that it fills the idle SMs
            before_proposals()
        rl, rr = ops.proposal_layer(cls_prob, bbox, im_info, cfg_key, shapes)
        out = self.heads(feats, B, rl.view(-1, 5), rr.view(-1, 5), im_h)
        n = rl.shape[1]
        out.update(rois_left=rl, rois_right=rr, rpn_cls_prob=cls_prob, rpn_bbox_pred=bbox, rpn_shapes=shapes)
        out["cls_prob"] = out["cls_prob"].view(B, n, -1)
        out["bbox_pred"] = out["bbox_pred"].view(B, n, -1)
        out["dim_orien_pred"] = out["dim_orien_pred"].view(B, n, -1)
        if keep_features:      # debugging / tests: exact-fp32 views of the pre-biased trunk tensors
            ub = not self.exact and not self.half
            out["feats"] = {k: (ops.unbias(v) if (k[0] == "c" and ub and v is not None and v.dtype == torch.float32)
                                else v) for k, v in feats.items()}
            out["feats_raw"] = feats
        return out


class GraphRunner(object):
    """Capture a launch-bound sequence of libstereo_b200 kernels once into a CUDA graph and replay it.

    `fn(*static_inputs)` must be free of host<->device syncs (every entry point of the C ABI is) and is run
    `warmup` times eagerly first so that workspaces, function attributes and TMA descriptors exist.  Inputs are
    fixed tensors: copy new data into them (`runner.inputs[i].copy_(...)`) before `runner()`.
    """

    def __init__(self, fn, inputs, warmup=2):
        self.fn, self.inputs = fn, list(inputs)
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(warmup):
                fn(*self.inputs)
        torch.cuda.current_stream().wait_stream(s)
        torch.cuda.synchronize()
        self.graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self.graph):
            self.outputs = fn(*self.inputs)

    def __call__(self):
        self.graph.replay()
        return self.outputs
