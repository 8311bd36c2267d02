/*
 * stereo_b200.h -- C ABI of libstereo_b200.so (sm_90a).
 *
 * Drop-in boundary for the Stereo R-CNN hot path.  Every entry point takes
 * plain device pointers + sizes + an explicit stream (a cudaStream_t passed
 * as void*), never allocates, never synchronises, and returns 0 on success
 * or a non-zero code (a cudaError_t value, or SB_EINVAL for a bad argument /
 * too-small workspace).  Caller allocates every output, as in the reference.
 *
 * Reference interfaces replaced (paths relative to the reference checkout):
 *   sb_nms                    <- lib/model/nms/src/nms_cuda_kernel.h:5-6  (nms_cuda_compute)
 *                                lib/model/nms/src/nms_cuda.h:4-5         (nms_cuda, THC glue)
 *   sb_roi_align_forward      <- lib/model/roi_align/src/roi_align_kernel.h:13-17 (ROIAlignForwardLaucher)
 *                                lib/model/roi_align/src/roi_align_cuda.h:1-2     (roi_align_forward_cuda)
 *   sb_roi_align_backward     <- lib/model/roi_align/src/roi_align_kernel.h:24-27 (ROIAlignBackwardLaucher)
 *                                lib/model/roi_align/src/roi_align_cuda.h:4-5     (roi_align_backward_cuda)
 *   sb_proposal_layer         <- lib/model/rpn/proposal_layer.py:42-145 (_ProposalLayer.forward)
 *   sb_dense_align            <- lib/model/dense_align/dense_align.py:240-300 (align_parallel)
 *   sb_roi_align_pyramid_nhwc <- lib/model/stereo_rcnn/stereo_rcnn.py:110-139 (PyramidRoI_Feat + RoIAlignAvg)
 *   sb_conv2d / sb_* layer ops<- torch.nn.Conv2d/BatchNorm2d/... call sites in
 *                                lib/model/stereo_rcnn/resnet.py:66-121,236-286 and
 *                                lib/model/rpn/stereo_rpn.py:32-40,73-95
 */
#ifndef STEREO_B200_H
#define STEREO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB_OK 0
#define SB_EINVAL (-22)

typedef void* sb_stream_t; /* cudaStream_t */

/* library / device info: returns the compute capability major*10+minor of device 0, <0 on error */
int sb_version(void);
int sb_device_cc(void);

/* ---------------------------------------------------------------- NMS ----
 * dets: n x 5 [x1,y1,x2,y2,score] fp32, pre-sorted by score desc.
 * keep: >= n int32 (ascending indices of kept boxes), num_out: 1 int32.
 * Suppress j>i when IoU(i,j) > thresh ("+1" areas), bit-exact with the
 * reference's bitmask + greedy scan; the scan runs on the device.            */
size_t sb_nms_workspace_bytes(int n);
int sb_nms(const float* dets, int n, float thresh, int* keep, int* num_out,
           void* workspace, size_t workspace_bytes, sb_stream_t stream);
/* the raw 64x64 bitmask, upper-triangle blocks only (blocks below the diagonal are zero) */
int sb_nms_mask(const float* dets, int n, float thresh, uint64_t* mask, sb_stream_t stream);

/* ----------------------------------------------------------- RoIAlign ----
 * Reference semantics: features NCHW fp32, rois R x 5 [batch,x1,y1,x2,y2],
 * (ah, aw) is the tap lattice (RoIAlignAvg passes pooled+1), out R x C x ah x aw.
 * SB_EINVAL unless H >= 2 and W >= 2 (the bilinear cell at hstart = min(floor(h), H-2)
 * must lie inside the map).                                                          */
int sb_roi_align_forward(const float* features, int N, int C, int H, int W,
                         const float* rois, int R, int ah, int aw, float spatial_scale,
                         float* out, sb_stream_t stream);
/* bottom_grad (N x C x H x W) must be zero-filled by the caller, as in the reference.
 * Like the reference kernel (roi_align_kernel.cu:94-143) the scatter uses four float
 * atomicAdds per tap: the summation ORDER is not deterministic, results agree with the
 * reference launcher to 1e-4 relative (tests/test_gpu_ops.py), not bit for bit.        */
int sb_roi_align_backward(const float* top_grad, int N, int C, int H, int W,
                          const float* rois, int R, int ah, int aw, float spatial_scale,
                          float* bottom_grad, sb_stream_t stream);

/* The same backward, deterministic (SURVEY 7.8): contributions are accumulated in 64-bit fixed point (scale from
 * max|top_grad|, quantum max|top| * 2^-41), so the sums do not depend on the order of the atomics or of the RoIs --
 * bit-identical run to run.  bottom_grad is OVERWRITTEN (no zero-fill needed); workspace = N*C*H*W*8 + 16 bytes. */
size_t sb_roi_align_backward_det_workspace(int N, int C, int H, int W);
int sb_roi_align_backward_det(const float* top_grad, int N, int C, int H, int W,
                              const float* rois, int R, int ah, int aw, float spatial_scale,
                              float* bottom_grad, void* workspace, size_t workspace_bytes, sb_stream_t stream);

/* Fused PyramidRoI_Feat: level routing (Q14) + per-level scale (Q15) + tap lattice +
 * 2x2/stride-1 average, NHWC features, one launch for all levels.
 * feats[l]: N x H_l x W_l x C (l = P2..P5); out[r][ph][pw][out_coff + c], row pitch out_ld elements;
 * round_tf32: 0 = exact fp32, 1 = fp32 rounded to TF32, 2 = __half output (out is then a __half*).
 * SB_EINVAL, before any launch, unless: R >= 0; C > 0 and C % 4 == 0; pooled >= 1; out_ld % 4 == 0;
 * out_coff >= 0, out_coff % 4 == 0 and out_coff + C <= out_ld; round_tf32 in {0, 1, 2}; every level
 * has a non-null pointer and H_l >= 2, W_l >= 2; rois and out non-null when R > 0; and the kernel's
 * shared memory, 8 (pooled+1) C + 40 (rb+1)(pooled+1) bytes with rb = pooled <= 8 ? pooled : (pooled+1)/2,
 * is at most 200 KB.  R == 0 launches nothing.
 * Mode 0 is bit-exact with the reference's arithmetic (fp32 lattice values rounded once from fp64, the
 * 2x2 average in fp32) except where an fp64 lattice value lies within ~2^-50 of an fp32 rounding tie;
 * modes 1 and 2 are mode 0 rounded (TF32 ties away, fp16 ties to even).  The level, round(logf(..) + 4),
 * may differ from a correctly rounded log's for a RoI within 1 ulp of a level boundary. */
int sb_roi_align_pyramid_nhwc(const float* const* feats, const int* heights, const int* widths,
                              int C, float im_h, const float* rois, int R, int pooled,
                              float* out, int out_ld, int out_coff, int round_tf32, sb_stream_t stream);

/* Backward of sb_roi_align_pyramid_nhwc (mode 0) for fp32 gradients: the exact adjoint of the forward, routing and
 * taps included, ADDED in place into fp32 NHWC level gradients dfeats[l] [N, H_l, W_l, C] (l = P2..P5).
 * A source is one forward call's gradient: grad[r][ph][pw][coff + c] (row pitch ld) of RoI r of rois [R,5], pooled =
 * P, read at image batch_offset + rois[r][0] of the levels (0 for the left images, B for the right ones).
 * Lattice point gradient gl = ((G[i-1][j-1] + G[i-1][j]) + (G[i][j-1] + G[i][j])) / 4 in fp64 over the outputs that
 * read it; each corner of its bilinear tap (the forward's fp64 weights; zero taps contribute nothing) gains
 * rint(gl 2^e w) in a 64-bit fixed-point accumulator, e = 60 - ex - k with max|G| < 2^ex over every source and
 * T = sum_s R_s (P_s+1)^2 <= 2^k the call's lattice taps (at most T contributions per element: no overflow).
 * Finally dfeats += acc 2^-e in fp64, one rounding to fp32.  Bit-identical run to run and under any permutation of
 * the RoIs of a source.  Per element, |result - exact| <= 2^-e n + ulp/2 (+ fp64 rounding), n its contributions.
 * *nonfinite (device int, may be NULL) is set to 1 when a gradient read or a result is not finite (never cleared);
 * a non-finite gradient makes every element of dfeats NaN.  A RoI whose image lies outside [0, N) contributes
 * nothing.  Workspace: sb_roi_align_pyramid_backward_workspace bytes, 8-byte aligned.
 * SB_EINVAL, before any launch, unless: 1 <= n_sources <= 4; N >= 1; C > 0 and C % 4 == 0; every level has a
 * non-null pointer and H_l >= 2, W_l >= 2; the workspace is non-null, aligned and large enough; and for each source
 * R >= 0, pooled >= 1, ld % 4 == 0, coff >= 0, coff % 4 == 0, coff + C <= ld, 0 <= batch_offset < N, grad and
 * rois non-null when R > 0, and (rb+1)(pooled+1) 40 bytes of shared memory <= 48 KB (rb as the forward's).
 * R == 0 in every source launches nothing and leaves dfeats untouched.                                        */
typedef struct {
    const float* grad;
    const float* rois;
    int R, pooled, ld, coff, batch_offset;
} sb_roi_grad_source;
size_t sb_roi_align_pyramid_backward_workspace(const int* heights, const int* widths, int N, int C);
int sb_roi_align_pyramid_backward(const sb_roi_grad_source* sources, int n_sources, float* const* dfeats,
                                  const int* heights, const int* widths, int N, int C, float im_h,
                                  int* nonfinite, void* workspace, size_t workspace_bytes, sb_stream_t stream);

/* ----------------------------------------------------- proposal layer ----
 * cls_prob [B,A,2] (column 1 = score), bbox_pred_lr [B,A,6], im_info [B,3] (device).
 * cfg: host struct (anchor pyramid + top-N / threshold constants), A = n_ratios*sum(h*w).
 * rois_left/right: [B, post_nms_top_n, 5], zero padded; fully stream-ordered.
 * Scores are ranked as torch.sort(descending=True) ranks them -- every NaN above +inf, -0.0 equal to +0.0 -- with
 * ties by ascending anchor index.  pre_nms_top_n <= 0 or >= A keeps all A anchors (K = min(pre, A) <= 16384).
 * SB_EINVAL, before any launch, unless: every level has positive h, w, scale and stride; every ratio is finite and
 * positive; A = n_ratios * sum(h*w) <= 2048 * 4096; post_nms_top_n >= 1; nms_thresh is finite; B >= 0; the five
 * tensors are non-null when B > 0; the workspace is non-null and large enough.  sb_generate_anchors applies the
 * same pyramid checks.                                                                 */
typedef struct {
    int n_levels;             /* <= 8 */
    int shapes[8][2];         /* (h, w) of each pyramid level (rpn_shapes) */
    int anchor_scales[8];     /* cfg.FPN_ANCHOR_SCALES */
    int feat_strides[8];      /* cfg.FPN_FEAT_STRIDES  */
    int n_ratios;             /* <= 4 */
    double ratios[4];         /* cfg.ANCHOR_RATIOS */
    int pre_nms_top_n;        /* cfg[key].RPN_PRE_NMS_TOP_N  (<= 16384) */
    int post_nms_top_n;       /* cfg[key].RPN_POST_NMS_TOP_N */
    float nms_thresh;         /* cfg[key].RPN_NMS_THRESH */
} sb_proposal_cfg;
size_t sb_proposal_workspace_bytes(int B, int A, int pre_nms_top_n);
int sb_proposal_layer(const float* cls_prob, const float* bbox_pred_lr, const float* im_info,
                      int B, int A, const sb_proposal_cfg* cfg,
                      float* rois_left, float* rois_right,
                      void* workspace, size_t workspace_bytes, sb_stream_t stream);
/* the whole anchor table of the pyramid (generate_anchors.py:112-173: fp64, cast to fp32), [A,4] in the proposal
 * layer's order (level, y, x, ratio); only shapes / anchor_scales / feat_strides / ratios of cfg are read.  The
 * proposal layer itself never materialises it; the train-time anchor target layer (below) needs it. */
int sb_generate_anchors(const sb_proposal_cfg* cfg, int A, float* anchors, sb_stream_t stream);
/* fused RPN head epilogue: raw head output [B, sum(h*w), ld] (cols 0..5 cls logits in the
 * reference's channel order, 6..23 the 18 box channels) -> cls_prob [B,A,2], bbox_pred [B,A,6]
 * with the reference's softmax channel pairing (stereo_rpn.py:52-60,81-83)               */
int sb_rpn_head_epilogue(const float* head, int B, int P, int ld, float* cls_prob, float* bbox_pred,
                         sb_stream_t stream);
/* the raw class scores the RPN loss reads (stereo_rpn.py:89,116-119: rpn_cls_score, each pixel's six score channels as
 * the consecutive pairs (c0,c1), (c2,c3), (c4,c5)): head [B, P, ld] -> rpn_cls_score [B, 3P, 2]; ld >= 6 */
int sb_rpn_head_scores(const float* head, int B, int P, int ld, float* rpn_cls_score, sb_stream_t stream);

/* -------------------------------------------------------- dense_align ----
 * im_left/right: 3 x H x W planar fp32 (network-scale, batch 1).
 * calib4: host {P2[0,0], P2[0,2], P2[1,2], P2[0,3]-P3[0,3]}; scale = im_info[0,2].
 * box_left D x 4, keypoints D x 5, poses D x 7 (device).  status[D], best_dis[D] (device). */
size_t sb_dense_align_workspace_bytes(int H, int W, int D);
int sb_dense_align(const float* im_left, const float* im_right, int H, int W,
                   const double* calib4, double scale,
                   const float* box_left, const float* keypoints, const float* poses, int D,
                   float* status, float* best_dis,
                   void* workspace, size_t workspace_bytes, sb_stream_t stream);

/* ----------------------------------------------------- dense layer ops ----
 * NHWC fp32 activations.  One descriptor drives both the SIMT fp32 kernel (stem, odd
 * shapes) and the wgmma TF32 / FP16 implicit-GEMM kernel (everything GEMM-shaped).          */
typedef struct {
    const float* in;        /* [N,H,W,in_ld] channels [0,Cin) used */
    const float* wgt;       /* [Cout][kh][kw][Cin] */
    const float* scale;     /* [Cout] or NULL (folded frozen BN gamma/sqrt(var+eps)); 16-byte aligned for the tensor-core path */
    const float* shift;     /* [Cout] or NULL (folded BN beta / conv bias); 16-byte aligned for the tensor-core path */
    const float* residual;  /* [N,Ho,Wo,res_ld] or NULL: added before ReLU (tensor-core path: 1x1 convs only -- conv3 of a
                             * bottleneck; sb_conv2d_tc_supported() says no otherwise and the SIMT kernel takes it) */
    const float* up_src;    /* [N,UH,UW,Cout] or NULL: bilinear(align_corners) upsample to Ho x Wo, added */
    float* out;             /* out[n*out_n_stride + ho*out_h_stride + wo*out_w_stride + out_coff + c] */
    int N, H, W, Cin, Cout, kh, kw, stride, pad, Ho, Wo;
    int in_ld, res_ld, UH, UW, relu;
    int out_coff;
    /* TF32 operand hygiene (the tf32 tensor-core MMA TRUNCATES fp32 operands to 19 bits, a biased rounding):
     *   out_mode 0: store exact fp32 (tensors read by non-conv consumers)
     *   out_mode 1: store round-to-nearest TF32 (tensors read only by convs: truncation becomes exact)
     *   out_mode 2: store exact fp32 with +0x1000 added to the bit pattern ("pre-biased"): the tensor
     *               core's truncation then IS round-to-nearest, and exact readers subtract 0x1000 back
     *               (residual stream of the trunk: conv input and exact residual from one tensor)
     *   res_biased: the residual tensor is stored pre-biased;  in_biased: the input is (SIMT kernel only) */
    int out_mode, res_biased, in_biased;
    long long out_n_stride, out_h_stride, out_w_stride;
    /* fp16 operand mode of the tensor-core kernel (f16, fp32 accumulate): in/wgt point to __half data
     * (in_dtype 1, Cin % 64 == 0); out16, when non-NULL, receives an fp16 (round-to-nearest) twin of the
     * output with the same element strides; out may be NULL when only the fp16 twin is wanted.          */
    void* out16;
    int in_dtype;
    int max_ctas;           /* 0 = one persistent CTA per SM; otherwise cap the grid (concurrent launches on
                             * other streams get the remaining SMs) */
} sb_conv_desc;

/* exact-fp32 SIMT convolution: fp32 operands (in_dtype 0) and the fp32 output only; SB_EINVAL for an fp16
 * descriptor, a non-NULL out16 or in_ld < Cin, before any launch */
int sb_conv2d_simt(const sb_conv_desc* d, sb_stream_t stream);
/* tensor-core path: requires Cin % 32 == 0 (K tile = one 128-byte swizzle row), in_ld >= Cin, stride 1.  With fp16
 * operands and a residual, the outputs leave by TMA: output pixels must be contiguous rows (h / n strides = Wo / Ho*Wo
 * pixel strides), and with a twin Cout, out_w_stride and out_coff % 8 == 0 and out16 16-byte aligned. */
int sb_conv2d_tc(const sb_conv_desc* d, sb_stream_t stream);
int sb_conv2d_tc_supported(const sb_conv_desc* d);
/* the same 3x3 convolution on flat tiles of 128 consecutive output pixels in (n, h, w) order, loaded by TMA im2col,
 * instead of 8x16 spatial patches: no MMA rows past the right or bottom edge of a map.  Bit-identical to sb_conv2d_tc
 * on the descriptors it takes: what sb_conv2d_tc_supported() accepts with fp16 operands, 3x3, pad 1, stride 1, no
 * residual and no up_src; SB_EINVAL for anything else, before any launch. */
int sb_conv2d_tc_rows(const sb_conv_desc* d, sb_stream_t stream);

/* ------------------------------------------------- backward pass of the trunk + FPN (fp16 operands, fp32 accumulate) ----
 * sb_conv2d_tc_dgrad -- data gradient of a conv (the input gradient torch.nn.Conv2d's autograd forms for the convs of
 *   lib/model/stereo_rcnn/resnet.py:66-102 and stereo_rcnn.py:91-108,155-168) as the forward implicit GEMM: d->in is the
 *   fp16 output gradient, d->wgt the weights packed [Cin][kh][kw][Cout] with the taps flipped and the frozen-BN scale
 *   folded in, Cin / Cout swapped in the descriptor.  The epilogue adds d->residual (1x1 only), then keeps an element
 *   only where mask16 (fp16, the output's element layout; NULL = no mask) is > 0: the ReLU of the saved forward tensor.
 *   d->relu, d->up_src and d->out_mode must be 0; out_strides scatter into even positions for stride-2 convs.
 * sb_conv_wgrad -- weight gradient (and optionally bias gradient) of a 1x1 or 3x3 (pad 1) stride-1 conv:
 *   dw[Cout][Cin][k][k] = scale[co] / grad_scale * sum_p dy16[p][co] x16[p + tap][ci] (NHWC fp16 operands, N x H x W),
 *   db[co] = sum_p dy32[p][co] / grad_scale.  Split over pixel ranges, partials reduced in a fixed order: bit-identical
 *   run to run.  *nonfinite (device int, may be NULL) is set to 1 when a result is not finite (never cleared).
 *   Cin, Cout multiples of 64; workspace of sb_conv_wgrad_workspace bytes.
 * sb_fpn_grad_combine -- gradient of one FPN level: out = scale * dp + up^T(dt) + scatter2(scale * dp6) over NHWC fp32
 *   [N,H,W,C]; up^T transposes the align_corners bilinear upsample of stereo_rcnn.py:91-108 from the fine [N,TH,TW,C] dt
 *   (a gather, fixed order); dp6 [N,H6,W6,C] is the gradient of P6 = P5[::2, ::2] (stereo_rcnn.py:168).  dp, dt and dp6
 *   may each be NULL; out (fp32) and/or out16 (fp16 twin) receive the result.
 * The _devscale twins of these and of the backward entry points below (sb_rpn_head_grad, sb_conv_wgrad_acc,
 *   sb_box_tail_backward, sb_kpts_tail_backward) take the gradient scale as `const float* grad_scale` (fp32 [1] in
 *   DEVICE memory, read by the kernels; sb_fpn_grad_combine_devscale's `scale` likewise) in place of the host float:
 *   sb_conv_wgrad*_devscale divide by *grad_scale as 1.0f / *grad_scale (the host passes inv_grad_scale; the two agree
 *   when the scale is a power of two).  Otherwise the same kernels, operation order and argument checks as the float
 *   entry point, plus SB_EINVAL for a NULL scale pointer; the results are bit-identical for equal values.  A captured
 *   graph then follows a scale the device changes between replays (sb_loss_scale_update).                          */
int sb_conv2d_tc_dgrad(const sb_conv_desc* d, const void* mask16, sb_stream_t stream);
size_t sb_conv_wgrad_workspace(int N, int H, int W, int Cin, int Cout, int k);
int sb_conv_wgrad(const void* dy16, const void* x16, int N, int H, int W, int Cin, int Cout, int k,
                  const float* scale, float inv_grad_scale, float* dw, const float* dy32, float* db, int* nonfinite,
                  void* workspace, size_t workspace_bytes, sb_stream_t stream);
int sb_conv_wgrad_devscale(const void* dy16, const void* x16, int N, int H, int W, int Cin, int Cout, int k,
                           const float* scale, const float* grad_scale, float* dw, const float* dy32, float* db,
                           int* nonfinite, void* workspace, size_t workspace_bytes, sb_stream_t stream);
int sb_fpn_grad_combine(const float* dp, const float* dt, int N, int H, int W, int TH, int TW, int C,
                        const float* dp6, int H6, int W6, float scale, float* out, void* out16, sb_stream_t stream);
int sb_fpn_grad_combine_devscale(const float* dp, const float* dt, int N, int H, int W, int TH, int TW, int C,
                                 const float* dp6, int H6, int W6, const float* scale, float* out, void* out16,
                                 sb_stream_t stream);

/* ------------------------------------------------- backward pass of the stereo RPN (fp16 operands, fp32 accumulate) ----
 * Together these replace the autograd of lib/model/rpn/stereo_rpn.py:73-95 (RPN_Conv, RPN_cls_score,
 * RPN_bbox_pred_left_right) that loss.backward() runs in trainval_net.py.
 * sb_rpn_head_grad -- gradient of the fused RPN head's output from the sb_rpn_loss gradients d_cls_score [B,A,2] and
 *   d_bbox_pred [B,A,6] (A = 3P): dhead16 [B,P,64] fp16 = grad_scale * d in columns 0..5 (the raw scores' channels) and
 *   6..23 (the 18 box channels), zero in 24..63; dhead32 (may be NULL) its fp32 twin.  No softmax: the loss reads the
 *   raw scores.
 * sb_conv_wgrad_acc -- sb_conv_wgrad on strided operands with accumulation: pixel p of dy16 / x16 / dy32 starts at
 *   element p * dy_ld / x_ld / dy32_ld (dy_ld, x_ld multiples of 8, >= Cout / Cin; dy16, x16 16-byte aligned).
 *   accumulate != 0 adds the results to dw / db (stream order, so a fixed call order gives bit-identical sums).
 *   Rows co < split of dW / db go to dw / db, rows split <= co < rows to dw_hi / db_hi (row co - split), rows >= rows
 *   are not stored (1 <= split <= rows <= Cout).  With dense strides, accumulate = 0 and split = rows = Cout the results
 *   are bit-identical to sb_conv_wgrad's.  Workspace of sb_conv_wgrad_acc_workspace bytes.                        */
int sb_rpn_head_grad(const float* d_cls_score, const float* d_bbox_pred, int B, int P, float grad_scale,
                     void* dhead16, float* dhead32, sb_stream_t stream);
int sb_rpn_head_grad_devscale(const float* d_cls_score, const float* d_bbox_pred, int B, int P, const float* grad_scale,
                              void* dhead16, float* dhead32, sb_stream_t stream);
size_t sb_conv_wgrad_acc_workspace(int N, int H, int W, int Cin, int Cout, int k);
int sb_conv_wgrad_acc(const void* dy16, int dy_ld, const void* x16, int x_ld, int N, int H, int W, int Cin, int Cout,
                      int k, const float* scale, float inv_grad_scale, const float* dy32, int dy32_ld, int accumulate,
                      int rows, int split, float* dw, float* db, float* dw_hi, float* db_hi, int* nonfinite,
                      void* workspace, size_t workspace_bytes, sb_stream_t stream);
int sb_conv_wgrad_acc_devscale(const void* dy16, int dy_ld, const void* x16, int x_ld, int N, int H, int W, int Cin,
                               int Cout, int k, const float* scale, const float* grad_scale, const float* dy32,
                               int dy32_ld, int accumulate, int rows, int split, float* dw, float* db, float* dw_hi,
                               float* db_hi, int* nonfinite, void* workspace, size_t workspace_bytes,
                               sb_stream_t stream);

/* ------------------------------------------------- backward pass of the R-CNN heads ----
 * Together with sb_conv2d_tc_dgrad / sb_conv_wgrad these replace the autograd of lib/model/stereo_rcnn/resnet.py:256-286
 * (RCNN_top, RCNN_kpts, kpts_class, RCNN_cls_score, RCNN_bbox_pred, RCNN_dim_orien_pred) and stereo_rcnn.py:252-271.
 * Every reduction runs in a fixed order (bit-identical run to run); *nonfinite (device int, may be NULL) is set to 1
 * when a result is not finite (never cleared).  Every argument check returns SB_EINVAL before any launch.
 * sb_box_tail_scores -- sb_box_tail that also writes the raw class scores cls_score [R,nc] the loss reads (cls_prob,
 *   bbox_pred and dim_orien are the same bits as sb_box_tail's).
 * sb_kpts_logits -- the keypoint logits [R,6,G] (sb_kpts_tail's kpts_pred_all) split into the loss's kpts_pred [R,4G]
 *   (channels 0..3), left_border_pred [R,G] (4) and right_border_pred [R,G] (5).
 * sb_dropout_words -- Dropout(p) in training mode with explicit random words instead of torch's RNG: x[i] (n fp32, or
 *   fp16 when x_is_half) becomes 0 where words[i] < p 2^32 (as uint32) and x[i] / (1 - p) elsewhere, in place;
 *   0 <= p < 1.
 * sb_box_tail_backward -- the three linears on fc7 [R,K] (the saved post-ReLU, post-dropout activation):
 *   dW / db of RCNN_cls_score [nc,K] / [nc], RCNN_bbox_pred [6nc,K] / [6nc], RCNN_dim_orien_pred [5nc,K] / [5nc] from
 *   the loss gradients d_cls_score [R,nc], d_bbox_pred [R,6nc], d_dim_orien_pred [R,5nc] (fp32 throughout), and the
 *   gradient of RCNN_top.3's pre-activation dz32 [R,K] = grad_scale * mask_scale * [fc7 > 0] * sum_o d[r][o] W[o][k]
 *   (mask_scale = 1 / (1 - p) with dropout, else 1) with its fp16 rounding dz16.  R >= 1, 1 <= n_classes <= 4.
 * sb_kpts_tail_backward -- the keypoint tail (the deconv output up16 [R,G,G,C] fp16, post-ReLU, summed over height,
 *   then kpts_class w [6][C]) from d_kpts_pred [R,4G], d_left_border_pred [R,G], d_right_border_pred [R,G]:
 *   dw [6][C] and db [6] of kpts_class, db_up [C] = the deconv bias gradient (sum over all four phases), and dup16 the
 *   gradient of the deconv output masked by up16 > 0, times grad_scale, fp16, phase-major [R,G/2,G/2,4C]: pixel (y, x)
 *   at (y/2, x/2), channels ((y%2)*2 + x%2)*C + c.  G even, 2 <= G <= 64; C % 32 == 0, 32 <= C <= 1024; workspace of
 *   sb_kpts_tail_backward_workspace bytes.
 * sb_permute3 -- dst[i0 s0 + i1 s1 + i2 s2] = src[(i0 d1 + i1) d2 + i2] (fp32, out of place): a weight gradient into the
 *   reference's layout.  The strides must lay the three dimensions out densely in some order.               */
int sb_box_tail_scores(const float* fc7, int R, int K, int n_classes, const float* w_cls, const float* b_cls,
                       const float* w_box, const float* b_box, const float* w_dim, const float* b_dim,
                       float* cls_prob, float* bbox_pred, float* dim_orien, float* cls_score, sb_stream_t stream);
int sb_kpts_logits(const float* kpts_pred_all, int R, int G, float* kpts_pred, float* left_border_pred,
                   float* right_border_pred, sb_stream_t stream);
int sb_dropout_words(void* x, int x_is_half, long long n, const unsigned* words, double p, sb_stream_t stream);
int sb_box_tail_backward(const float* d_cls_score, const float* d_bbox_pred, const float* d_dim_orien_pred,
                         const float* fc7, int R, int K, int n_classes, const float* w_cls, const float* w_box,
                         const float* w_dim, float mask_scale, float grad_scale, float* dw_cls, float* db_cls,
                         float* dw_box, float* db_box, float* dw_dim, float* db_dim, void* dz16, float* dz32,
                         int* nonfinite, sb_stream_t stream);
int sb_box_tail_backward_devscale(const float* d_cls_score, const float* d_bbox_pred, const float* d_dim_orien_pred,
                                  const float* fc7, int R, int K, int n_classes, const float* w_cls,
                                  const float* w_box, const float* w_dim, float mask_scale, const float* grad_scale,
                                  float* dw_cls, float* db_cls, float* dw_box, float* db_box, float* dw_dim,
                                  float* db_dim, void* dz16, float* dz32, int* nonfinite, sb_stream_t stream);
size_t sb_kpts_tail_backward_workspace(int R, int C);
int sb_kpts_tail_backward(const void* up16, int R, int G, int C, const float* w, const float* d_kpts_pred,
                          const float* d_left_border_pred, const float* d_right_border_pred, float grad_scale,
                          void* dup16, float* dw, float* db, float* db_up, int* nonfinite, void* workspace,
                          size_t workspace_bytes, sb_stream_t stream);
int sb_kpts_tail_backward_devscale(const void* up16, int R, int G, int C, const float* w, const float* d_kpts_pred,
                                   const float* d_left_border_pred, const float* d_right_border_pred,
                                   const float* grad_scale, void* dup16, float* dw, float* db, float* db_up,
                                   int* nonfinite, void* workspace, size_t workspace_bytes, sb_stream_t stream);
int sb_permute3(const float* src, int d0, int d1, int d2, long long s0, long long s1, long long s2, float* dst,
                sb_stream_t stream);

/* Diagnostics (tools/conv_trace.py): per-CTA phase timestamps of every following sb_conv2d_tc launch, 16 x u64
 * per CTA and 304 CTA slots per launch, into a caller-owned device buffer of sb_conv_trace_bytes(max_launches)
 * bytes.  buf = NULL switches tracing off.  sb_conv_trace_info(id) gives launch id's {Cin, Cout, kh, M, BLOCK_N, tiles,
 * K-steps, residual, upsample, variant, max_ctas, N}, variant = 1 (fp16 operands) | 2 (data gradient) | 4 (mask).
 * sb_conv_trace_epilogue(id) is 1 when launch id stored its outputs by TMA through the per-warpgroup rings, 0 when it
 * ran the register epilogue.  No counterpart in the reference. */
size_t sb_conv_trace_bytes(int max_launches);
int sb_conv_trace(void* buf, int max_launches);
int sb_conv_trace_count(void);
int sb_conv_trace_info(int id, int* out12);
int sb_conv_trace_epilogue(int id);

/* stem: NCHW image -> conv7x7/2 + frozen BN + ReLU -> NHWC (resnet.py:111-113) */
int sb_stem_conv(const float* im_nchw, int N, int H, int W, const float* wgt /*[64][7][7][3]*/,
                 const float* scale, const float* shift, float* out_nhwc, int out_mode, sb_stream_t stream);
/* stem as a TF32 tensor-core GEMM: patch matrix [N*Ho*Wo][160] (k = ci*49+r*7+s, zero padded from 147) that
 * sb_conv2d_tc then multiplies with the [64][160] stem weights (1x1 conv, Cin = 160)              */
int sb_stem_im2col(const float* im_nchw, int N, int H, int W, float* out, sb_stream_t stream);
/* the stem on the tensor cores with the patch gather INSIDE the GEMM kernel (round 2: no patch matrix in memory):
 * wgt16 = __half [64][192] ((ci, r, s) taps zero padded from 147), out16 = __half NHWC [N,Ho,Wo,64], BN + ReLU fused */
int sb_stem_conv_tc(const float* im_nchw, int N, int H, int W, const void* wgt16, const float* scale,
                    const float* shift, void* out16, sb_stream_t stream);
/* MaxPool2d(3, stride 2, pad 0, ceil_mode) NHWC (resnet.py:113) */
int sb_maxpool3x3s2_ceil(const float* in, int N, int H, int W, int C, float* out, sb_stream_t stream);
int sb_maxpool3x3s2_ceil16(const void* in_half, int N, int H, int W, int C, void* out_half, sb_stream_t stream);
/* x[:, ::2, ::2, :] (stride-2 1x1 convs of resnet.py:71 and P6 of stereo_rcnn.py:39) */
int sb_subsample2(const float* in, int N, int H, int W, int C, float* out, sb_stream_t stream);
/* keypoint tail: relu'd deconv output [R,G,G,C] -> sum over height -> 1x1 (C->6) -> [R,6,G]
 * -> softmax over 4G / G / G (stereo_rcnn.py:262-271)                                    */
int sb_kpts_tail(const void* x, int x_is_half, int R, int G, int C, const float* w /*[6][C]*/, const float* b /*[6]*/,
                 float* kpts_prob /*[R,4G]*/, float* left_prob /*[R,G]*/, float* right_prob /*[R,G]*/,
                 float* kpts_pred_all /*[R,6,G], required*/, sb_stream_t stream);
/* box-head tail: fc7 [R,K] -> cls softmax [R,nc], bbox [R,6nc], dim_orien [R,5nc] */
int sb_box_tail(const float* fc7, int R, int K, int n_classes,
                const float* w_cls, const float* b_cls, const float* w_box, const float* b_box,
                const float* w_dim, const float* b_dim,
                float* cls_prob, float* bbox_pred, float* dim_orien, sb_stream_t stream);
/* test-time decode (test_net.py:138-212), one image */
int sb_test_decode(const float* rois_left, const float* rois_right, const float* bbox_pred,
                   const float* dim_orien, const float* kpts_prob, const float* left_prob,
                   const float* right_prob, const float* im_info, int R, int n_classes, int grid,
                   float* pred_boxes_left, float* pred_boxes_right, float* dim_orien_out,
                   float* pred_kpts, sb_stream_t stream);
/* the same decode that also emits the per-image detection record which ranks all-gather (SURVEY 8e; the result
 * packing of test_net.py:233-330): record[r] = [cls_prob nc | boxes_left 4nc | boxes_right 4nc | dim_orien 5nc |
 * kpts 5], row pitch record_ld >= 14*nc + 5 floats                                                           */
int sb_test_decode_record(const float* rois_left, const float* rois_right, const float* cls_prob,
                          const float* bbox_pred, const float* dim_orien, const float* kpts_prob,
                          const float* left_prob, const float* right_prob, const float* im_info, int R,
                          int n_classes, int grid, float* pred_boxes_left, float* pred_boxes_right,
                          float* dim_orien_out, float* pred_kpts, float* record, int record_ld,
                          sb_stream_t stream);
/* per-class detection NMS (test_net.py:233-259), one image: scores [R,nc], boxes [R,4nc] (decoded left
 * boxes); keeps RoIs with score[:,cls] > score_thresh, sorted by score, NMS(nms_thresh); keep[] (>= R
 * ints) receives RoI indices in kept order, num_out the count.  R <= 512.  Equal scores (+0.0 and -0.0 are equal)
 * keep ascending RoI order; a NaN score never passes the threshold.                                   */
int sb_class_nms(const float* scores, const float* boxes, int R, int n_classes, int cls,
                 float score_thresh, float nms_thresh, int* keep, int* num_out, sb_stream_t stream);
/* input pipeline (lib/model/utils/blob.py:44-64 prep_im_for_blob + demo.py:124-128): uint8 HWC image (BGR, or RGB
 * with rgb_input = 1 as scipy's imread returns it, demo.py:106) -> fp32 (pixel - cfg.PIXEL_MEANS) ->
 * cv2.resize(fx = fy = scale, INTER_LINEAR) -> out [3, Ho, Wo] CHW, (Ho, Wo) from sb_prep_image_size            */
int sb_prep_image_size(int H, int W, double scale, int* Ho, int* Wo);
int sb_prep_image(const uint8_t* img, int H, int W, double scale, int rgb_input, float* out, sb_stream_t stream);
/* L2 flush helper for benchmarks: writes `bytes` of scratch */
int sb_fill(float* p, size_t n, float v, sb_stream_t stream);
/* p[0..n) = 1.0f / *v with v fp32 [1] in device memory (exact for a power of two): the per-channel unscale vectors of
 * the backward's data-gradient epilogues, following a loss scale that lives on the device.  SB_EINVAL for a NULL v,
 * or a NULL p with n > 0. */
int sb_fill_reciprocal(float* p, size_t n, const float* v, sb_stream_t stream);
/* number of kernel launches issued by this library since load (bench "gpu_launches") */
unsigned long long sb_launch_count(void);

/* ------------------------------------------------- 3D box solvers (SURVEY 8f-1) ----
 * The CPU stage between the network and dense_align (test_net.py:262-325), on the device.
 * sb_infer_boundary: kitti_utils.infer_boundary (kitti_utils.py:398-437) over the kept detections (keep[0..*num),
 *   in kept order); boxes [R, ld] with the box at column col_offset; left_right [>= *num, 2].
 * sb_box_solve: the keypoint border fix-up (test_net.py:263-266, inferred may be NULL) and
 *   box_estimator.solve_x_y_z_theta_from_kpt (box_estimator.py:169-385) per kept detection of class `cls` with
 *   score > eval_thresh; solved detections are appended in order to boxes_all [cap,5] (box + score), kpts_all
 *   [cap,5], poses_all [cap,8] (x,y,z,w,h,l,theta,alpha) as test_net.py:281-303 builds them; src_index [cap] = RoI
 *   index, *n_out (device) = how many.  p2 / p3: 3x4 row-major projection matrices, (im_h, im_w) the ORIGINAL image.
 * sb_dense_align_n: sb_dense_align on those device-resident rows (count read on the device).
 * sb_box_rectify: box_estimator.solve_x_y_theta_from_kpt (box_estimator.py:387-545) with the aligned disparity ->
 *   final [cap,13] doubles: valid, score, box_left[4], x, y, z, w, h, l, theta (what write_detection_results takes).
 * The reference minimises with scipy Newton-CG; here Levenberg-Marquardt in fp64 on the same residuals, to a
 * tighter stationarity than Newton-CG's own end points (tests/test_box_solver.py).                              */
int sb_infer_boundary(const float* boxes, int ld, int col_offset, const int* keep, const int* num, int im_w,
                      float* left_right, sb_stream_t stream);
int sb_box_solve(const float* scores, const float* boxes_left, const float* boxes_right, const float* dim_orien,
                 const float* kpts, const int* keep, const int* num, const float* inferred, int n_classes, int cls,
                 int im_h, int im_w, const double* p2, const double* p3, float eval_thresh, int cap,
                 float* boxes_all, float* kpts_all, float* poses_all, int* src_index, int* n_out, sb_stream_t stream);
int sb_dense_align_n(const float* im_left, const float* im_right, int H, int W, const double* calib4, double scale,
                     const float* box_left, int box_ld, const float* keypoints, const float* poses, int pose_ld,
                     int D_cap, const int* n_dev, float* status, float* best_dis, void* workspace,
                     size_t workspace_bytes, sb_stream_t stream);
int sb_box_rectify(const float* boxes_all, const float* kpts_all, const float* poses_all, const float* succ,
                   const float* best_dis, const int* n, int cap, int im_h, int im_w, const double* p2,
                   const double* p3, double* final_out, sb_stream_t stream);
/* The same three with the calibration in DEVICE memory, so that one captured CUDA graph serves every image of a
 * split, each with its own calibration file: calib = P2 then P3, 24 row-major doubles.  Every other argument is as in
 * the host-calibrated sibling.  The kernels read the calibration when they run; for equal calibration values the
 * results are bit-identical to the sibling's (sb_dense_align_n_devcalib forms calib4 and the constants derived from
 * it on the device, in the host's fp64 operations and order).  A null calib is SB_EINVAL, checked before any launch. */
int sb_box_solve_devcalib(const float* scores, const float* boxes_left, const float* boxes_right,
                          const float* dim_orien, const float* kpts, const int* keep, const int* num,
                          const float* inferred, int n_classes, int cls, int im_h, int im_w, const double* calib,
                          float eval_thresh, int cap, float* boxes_all, float* kpts_all, float* poses_all,
                          int* src_index, int* n_out, sb_stream_t stream);
int sb_dense_align_n_devcalib(const float* im_left, const float* im_right, int H, int W, const double* calib,
                              double scale, const float* box_left, int box_ld, const float* keypoints,
                              const float* poses, int pose_ld, int D_cap, const int* n_dev, float* status,
                              float* best_dis, void* workspace, size_t workspace_bytes, sb_stream_t stream);
int sb_box_rectify_devcalib(const float* boxes_all, const float* kpts_all, const float* poses_all, const float* succ,
                            const float* best_dis, const int* n, int cap, int im_h, int im_w, const double* calib,
                            double* final_out, sb_stream_t stream);

/* ------------------------------------------------- record all-gather over peer memory (SURVEY 8e) ----
 * The path's only exchange: every rank's fixed-size detection record ([300, 14nc+5] fp32, ~40 KB) to every rank of
 * one NVSwitch box.  Each rank owns a mailbox (sb_peer_alloc), exports it with CUDA IPC (sb_ipc_export, 64-byte
 * handle exchanged by the host's control plane) and maps its peers' (sb_ipc_import).  sb_peer_put_record stores the
 * local record into every mailbox (posted 128-bit NVLink writes + system-scope release of a sequence flag);
 * sb_peer_wait_records acquires the world's flags for the same step in the local mailbox and copies the records to
 * gathered[world][rec_floats].  Step counters live on the device: both calls are CUDA-graph capturable.  A peer
 * that never delivers sets *err_flag (device int) to 1 + its rank after timeout_s instead of hanging the GPU.
 * Replaces torch.distributed.all_gather / ncclAllGather on the data path; mailboxes[] is a HOST array of the
 * `world` device pointers (own allocation at index `rank`).  SB_EINVAL, before any launch, unless: 1 <= world <= 16;
 * 0 <= rank < world; 0 <= slot < n_slots; rec_floats >= 4 and a multiple of 4; rec, gathered and every mailbox are
 * non-null and 16-byte aligned; lag is 0 or 1; 0 <= timeout_s <= 1.8e10 (so never NaN).  Step counters are 32-bit:
 * the wait of a slot's 2^32nd step returns without copying (at lag 1, the next step's too), see csrc/peer.cu.    */
size_t sb_peer_mailbox_bytes(int n_slots, int world, int rec_floats);
int sb_peer_alloc(size_t bytes, void** ptr);
int sb_peer_free(void* ptr);
int sb_ipc_export(void* ptr, void* handle64);
int sb_ipc_import(const void* handle64, void** ptr);
int sb_ipc_close(void* ptr);
int sb_peer_put_record(const float* rec, void* const* mailboxes, int n_slots, int world, int rec_floats,
                       int rank, int slot, sb_stream_t stream);
/* lag = 0: collect the step just put; lag = 1: collect the PREVIOUS step of this slot (pipelined exchange: no rank
 * waits for a slower peer's current step; the first call of a slot leaves `gathered` untouched) */
int sb_peer_wait_records(void* mailbox, int n_slots, int world, int rec_floats, int slot, int lag, float* gathered,
                         int* err_flag, double timeout_s, sb_stream_t stream);

/* ------------------------------------------------- train-time target layers and losses (SURVEY A16 / 8f-4) ----
 * The label / target assignment and the losses of one training step on the device, no host round trip.
 * Every compare is bit-identical to the reference (fp32, same operation order); the regression targets differ at most
 * in the last ulp of log().  The random sampler takes explicit words instead of numpy's global stream (which the
 * reference consumes with data-dependent lengths): see oracle/train_targets.py (NumpySampler / KeySampler).
 *
 * sb_anchor_targets -- _AnchorTargetLayer.forward (lib/model/rpn/anchor_target_layer.py:42-164):
 *   anchors [A,4] fp32 (all pyramid levels, the proposal layer's order), gt_left / gt_right / gt_merge [B,K,5]
 *   (x1, y1, x2, y2, class; zero rows pad to K <= 64), im_h / im_w = int(im_info[0][0..1]) (image 0 bounds the anchors
 *   of the whole batch, :70-73), keys [B,A] uint32: one random word per anchor -- when an image has more than
 *   num_fg foreground (or more than rpn_batchsize - n_fg background) anchors, those with the SMALLEST (key, index)
 *   are disabled, i.e. "the first n - keep of a random permutation" (:109-123).
 *   -> labels [B,A] (1 / 0 / -1), targets_left / targets_right [B,A,4] (bbox_transform_batch, bbox_transform.py:38-77;
 *   zeros outside the image), inside_w / outside_w [B,A] (outside = 1 / #sampled anchors of the LAST image, :136).
 * sb_proposal_targets -- _ProposalTargetLayer.forward (lib/model/rpn/proposal_target_layer.py:36-333):
 *   rois_left / rois_right [B,R,5] (batch index first), gt_* as above, gt_dim_orien [B,K,5], gt_kpts [B,K,6];
 *   keys [B,R+K] (one word per candidate incl. the appended ground-truth boxes: foreground = the fg_rois_per_image
 *   candidates with the smallest (key, index), in that order), words [B,S] (background draw j = candidate
 *   words[j] * n_bg >> 32, i.e. floor(u * n_bg) with u = words[j] / 2^32; also the with-replacement draws of the
 *   one-sided cases :249-265) -> S = rois_per_image rows per image: rois, labels, box targets (normalised),
 *   dimension / orientation targets, keypoint / border bin targets (int32) and weights, inside / outside weights,
 *   keep_inds (index into the R+K candidates) and status [B] (1 = neither foreground nor background, the
 *   reference's ValueError :267).  R + K <= 4096, S <= 1024.
 * sb_rpn_loss -- stereo_rpn.py:114-140: losses[0] = cross entropy over the anchors with label != -1, losses[1] =
 *   _smooth_l1_loss (net_utils.py:79-99, sigma 3) on the 6-d deltas; optional gradients w.r.t. rpn_cls_score [B,A,2] and
 *   rpn_bbox_pred [B,A,6] (both or neither), scaled by exp(-uncert[0..1]) when uncert != NULL.
 * sb_rcnn_loss -- stereo_rcnn.py:201-311: losses[0..3] = RCNN_loss_cls, RCNN_loss_bbox, RCNN_loss_dim_orien,
 *   RCNN_loss_kpts; bbox_pred [R,6C] / dim_orien_pred [R,5C] are the per-class outputs (gathered by label inside);
 *   optional gradients w.r.t. all six prediction tensors (all or none), scaled by exp(-uncert[2..5]).
 * sb_multitask_loss -- trainval_net.py:214-219: total = sum_i losses[i] exp(-uncert[i]) + uncert[i]; d_uncert optional.
 * sb_clip_gradient -- net_utils.clip_gradient (net_utils.py:37-49) over n_tensors gradient tensors (HOST arrays of
 *   device pointers / element counts): one global norm, one scale; norm_out [2] (device) = total norm, applied factor.
 * Reductions are two-level in a fixed order: deterministic.                                                     */
typedef struct sb_proposal_target_cfg {
    int rois_per_image;        /* cfg.TRAIN.BATCH_SIZE = 512                         */
    int fg_rois_per_image;     /* round(FG_FRACTION * BATCH_SIZE) = 128              */
    float fg_thresh;           /* 0.5                                                */
    float bg_thresh_hi;        /* 0.5                                                */
    float bg_thresh_lo;        /* 0.0                                                */
    float bbox_means[4];       /* BBOX_NORMALIZE_MEANS (0, 0, 0, 0)                  */
    float bbox_stds[4];        /* BBOX_NORMALIZE_STDS (0.1, 0.1, 0.2, 0.2)           */
    float dim_means[5];        /* DIM_NORMALIZE_MEANS (1.6, 1.5, 4.0, 0, 0)          */
    float dim_stds[5];         /* DIM_NORMALIZE_STDS (0.5 x 5)                       */
    int kpts_grid;             /* cfg.KPTS_GRID = 28                                 */
} sb_proposal_target_cfg;

size_t sb_anchor_targets_workspace(int B, int A);
int sb_anchor_targets(const float* anchors, int A, const float* gt_left, const float* gt_right,
                      const float* gt_merge, int B, int K, int im_h, int im_w, const unsigned* keys,
                      float neg_overlap, float pos_overlap, int rpn_batchsize, int num_fg, void* workspace,
                      size_t workspace_bytes, float* labels, float* targets_left, float* targets_right,
                      float* inside_w, float* outside_w, sb_stream_t stream);
int sb_proposal_targets(const float* rois_left, const float* rois_right, int B, int R, const float* gt_left,
                        const float* gt_right, const float* gt_dim_orien, const float* gt_kpts, int K,
                        const unsigned* keys, const unsigned* words, const sb_proposal_target_cfg* cfg,
                        float* out_rois_left, float* out_rois_right, float* labels, float* bbox_targets_left,
                        float* bbox_targets_right, float* dim_orien_targets, int* kpts_targets,
                        float* kpts_weight, float* inside_w, float* outside_w, int* keep_inds, int* status,
                        sb_stream_t stream);
size_t sb_loss_workspace_bytes(void);
int sb_rpn_loss(const float* rpn_cls_score, const float* rpn_bbox_pred, const float* labels,
                const float* targets_left, const float* targets_right, const float* inside_w,
                const float* outside_w, int B, int A, const float* uncert, void* workspace,
                size_t workspace_bytes, float* losses, float* d_cls_score, float* d_bbox_pred,
                sb_stream_t stream);
int sb_rcnn_loss(const float* cls_score, const float* bbox_pred, const float* dim_orien_pred,
                 const float* kpts_pred, const float* left_border_pred, const float* right_border_pred,
                 const float* labels, const float* bbox_targets_left, const float* bbox_targets_right,
                 const float* dim_orien_targets, const int* kpts_targets, const float* kpts_weight,
                 const float* inside_w, const float* outside_w, int R, int n_classes, int kpts_grid,
                 const float* uncert, float* losses, float* d_cls_score, float* d_bbox_pred,
                 float* d_dim_orien_pred, float* d_kpts_pred, float* d_left_border_pred,
                 float* d_right_border_pred, sb_stream_t stream);
int sb_multitask_loss(const float* losses, const float* uncert, int n, float* total, float* d_uncert,
                      sb_stream_t stream);
size_t sb_clip_gradient_workspace(int n_tensors);
int sb_clip_gradient(float* const* grads, const size_t* counts, int n_tensors, float clip_norm,
                     void* workspace, size_t workspace_bytes, float* norm_out, sb_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * The optimizer step and the device-side refresh of the engine's packed weights (training step, SURVEY A16).
 *
 * sb_sgd_step -- torch.optim.SGD.step (dampening 0, no Nesterov) over n_tensors tensors.  HOST arrays of device
 *   pointers, element counts and per-tensor constants, passed to the kernels by value in chunks (graph-capturable):
 *   tensor i is params[i], grads[i], moms[i] (fp32, counts[i] >= 1 elements) with weight_decay[i] >= 0 and
 *   lr_mult[i] >= 0.  lr: fp32 [1] on the DEVICE (a captured step follows lr changes); momentum: a host float.
 *   Per element, in this order, each operation one IEEE fp32 operation rounded to nearest (no FMA contraction):
 *       d = g + wd * p;    m = momentum * m + d;    p = p - (lr * lr_mult) * m
 *   A zero-initialised m gives torch's first step exactly (momentum * 0 + d = d).  skip: int32 [1] on the device (the
 *   engine's found_inf): when *skip != 0 nothing is written and *skipped (int32 [1], device) is incremented by one --
 *   torch.cuda.amp.GradScaler's skip-on-overflow.  SB_EINVAL before any launch for a null pointer, n_tensors < 1, a
 *   zero count, a negative or non-finite weight_decay / lr_mult, or a non-finite momentum.
 *
 * sb_loss_scale_update -- torch.cuda.amp.GradScaler.update (torch._amp_update_scale_) in one thread on the device:
 *   when *found_inf != 0, *scale *= backoff_factor and *growth_tracker = 0; otherwise *growth_tracker + 1, and when that
 *   reaches growth_interval, *scale *= growth_factor and *growth_tracker = 0.  The scale is held within [2^-32, 2^32]:
 *   a growth past 2^32 leaves it unchanged (and resets the tracker, as torch does for a non-finite growth), a backoff
 *   below 2^-32 stops at 2^-32.  With power-of-two factors and a power-of-two start the scale and its reciprocal stay
 *   exact powers of two.  scale fp32 [1], growth_tracker and found_inf int32 [1], all device memory; graph-capturable.
 *   SB_EINVAL before any launch for a null pointer, a factor that is not a power of two, growth_factor <= 1,
 *   backoff_factor >= 1 or growth_interval < 1.
 *
 * sb_pack_plan / sb_pack_weights -- rewrite derived weight copies (packed, transposed, rounded, scaled) from fp32
 *   master tensors, one launch for a whole table of targets.  Target t maps a 4-d index (i0, i1, i2, i3) < shape:
 *       v = src[src_offset + sum_k i_k src_stride[k]]                    (strides may be negative: a tap flip)
 *       dst[dst_offset + sum_k i_k dst_stride[k]] = T(v);  dst16[same] = (half)v when dst16 != NULL
 *   with T one of SB_PACK_F32 (copy), SB_PACK_TF32 (round to TF32, nearest with ties away: (bits + 0x1000) & ~0x1fff,
 *   the integer rounding of ops.round_tf32_), SB_PACK_F16 (fp16, round to nearest even) and
 *   SB_PACK_SCALE_F16 (fp16 of the fp32 product v * scale[i_{scale_dim}]).  dst is fp32 for the first two, fp16 for
 *   the others; dst16 (an fp16 twin with dst's strides) is allowed with the fp32 transforms only.  dst_stride[3] must be
 *   1.  A target whose src_stride[3] != 1 is transposed through shared memory in tiles of up to 288 (i1, i2) rows x 32
 *   i3 columns: the reads walk i1 fastest (put the source's fastest dimension at i1), the writes walk i3, so both are
 *   coalesced.  sb_pack_plan validates a HOST table and fills its tile fields (tile0, tile, tiled) and *n_tiles;
 *   sb_pack_weights re-validates the host table and launches on `targets_dev`, a device copy of it made after the plan
 *   (upload it once, outside any capture; the launch is then graph-capturable).  SB_EINVAL before any launch for
 *   n_targets < 1, a null table / src / dst, a non-positive extent, dst_stride[3] != 1, an unknown transform, a scale
 *   missing or given without SB_PACK_SCALE_F16, a dst16 with an fp16 transform, an index that reaches below src or dst,
 *   or (sb_pack_weights) tile fields that differ from the plan's.  Targets must not overlap in dst.                */
#define SB_PACK_F32 0
#define SB_PACK_TF32 1
#define SB_PACK_F16 2
#define SB_PACK_SCALE_F16 3

typedef struct sb_pack_target {
    const float* src;
    void* dst;
    void* dst16;               /* optional fp16 twin of dst (SB_PACK_F32 / SB_PACK_TF32 only)              */
    const float* scale;        /* SB_PACK_SCALE_F16: per-channel scale, indexed by i_{scale_dim}           */
    long long src_offset;      /* elements                                                                 */
    long long dst_offset;      /* elements (dst and dst16)                                                 */
    long long shape[4];
    long long src_stride[4];   /* elements                                                                 */
    long long dst_stride[4];   /* elements; dst_stride[3] == 1                                             */
    int transform;             /* SB_PACK_*                                                                */
    int scale_dim;             /* 0..3                                                                     */
    long long tile0;           /* filled by sb_pack_plan: first tile (CTA) of this target                  */
    int tile[3];               /* filled by sb_pack_plan: tile extents along i1, i2, i3                    */
    int tiled;                 /* filled by sb_pack_plan: 1 = transposed through shared memory             */
} sb_pack_target;

int sb_sgd_step(float* const* params, float* const* grads, float* const* moms, const size_t* counts,
                const float* weight_decay, const float* lr_mult, int n_tensors, const float* lr, float momentum,
                const int* skip, int* skipped, sb_stream_t stream);
int sb_loss_scale_update(const int* found_inf, float* scale, int* growth_tracker, float growth_factor,
                         float backoff_factor, int growth_interval, sb_stream_t stream);
int sb_pack_plan(sb_pack_target* targets, int n_targets, long long* n_tiles);
int sb_pack_weights(const sb_pack_target* targets, const sb_pack_target* targets_dev, int n_targets,
                    sb_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * The training side of the input pipeline (SURVEY 8f-3): blobs, ground truth and random words of one step, made on
 * the device from flags and counters that live there, so one captured graph serves every entry of a dataset.
 *
 * sb_prep_stereo_pair -- _get_image_blob (minibatch.py:89-131) for one pair in one launch: both frames uint8 [H,W,3],
 *   both outputs fp32 [3,Ho,Wo] with (Ho, Wo) from sb_prep_image_size.  *flip (int32 [1], DEVICE) == 0: out_left /
 *   out_right are sb_prep_image of left / right.  *flip != 0 (minibatch.py:116-119): out_left is sb_prep_image of the
 *   column-mirrored RIGHT frame and out_right of the column-mirrored LEFT frame, bit for bit, without materialising
 *   the mirrored frames.
 * sb_prep_stereo_pairs -- sb_prep_stereo_pair for B pairs of one frame shape in one launch (the same kernel; the
 *   single-pair entry point is its B = 1 launch): left / right uint8 [B,H,W,3], flip int32 [B] on the DEVICE (one
 *   flag per pair, so one captured launch serves any mix of flipped and unflipped pairs), out_left / out_right fp32
 *   [B,3,Ho,Wo].  Pair b is sb_prep_stereo_pair of frames b with flag flip[b], bit for bit.  1 <= B <= 32767.
 * sb_train_gt -- the ground truth of a step (minibatch.py:43-85, roibatchLoader.py:72-107) for B images, one CTA per
 *   image.  Inputs are the roidb rows of each image at a fixed capacity N <= 1024: boxes_left / boxes_right /
 *   boxes_merge [B,N,4], gt_classes [B,N] int32, dim_orien [B,N,4] (w, h, l, alpha), kpts [B,N,6], n_rows [B] int32
 *   on the DEVICE (rows in use, clamped to [0, N] by the kernel) and words [B,N] uint32.  Rows with gt_classes == 0
 *   are dropped; boxes and keypoints are multiplied by im_scale in fp32 (a float32 array times a Python float);
 *   x1 = min(x1, im_width); (sin, cos) of theta are evaluated in fp64 and rounded (math.sin of a float32); a scaled
 *   keypoint outside [0, im_width - 1] becomes -1.  The kept rows are ordered by (word, row index) ascending -- the
 *   rule of sb_proposal_targets' samplers, in place of np.random.shuffle -- the first 30 (cfg.MAX_NUM_GT_BOXES) are
 *   written and the rest of every output is zero: gt_left / gt_right / gt_merge [B,30,5] (x1, y1, x2, y2, class),
 *   gt_dim_orien [B,30,5], gt_kpts [B,30,6], num_boxes [B] int32.  im_scale and im_width (the blob's width) are
 *   those of every image of the batch.
 * sb_random_words -- n uint32 words of Philox4x32-10: word i is element i % 4 of the block with key (seed lo, seed hi)
 *   and counter (i / 4, stream_id, *step lo, *step hi); *step is a uint64 on the DEVICE.  The words do not depend on
 *   the launch geometry.  Replaces the torch.randint refills of train.random_words between the replays of a step.
 * sb_step_advance -- *step += 1 in one thread: the last node of a captured step, so every replay draws new words.
 * SB_EINVAL before any launch for a null pointer, a non-positive size or scale, B outside its range, N > 1024 or
 * n == 0.                                                                                                         */
int sb_prep_stereo_pair(const uint8_t* left, const uint8_t* right, int H, int W, double scale, int rgb_input,
                        const int* flip, float* out_left, float* out_right, sb_stream_t stream);
int sb_prep_stereo_pairs(const uint8_t* left, const uint8_t* right, int B, int H, int W, double scale, int rgb_input,
                         const int* flip, float* out_left, float* out_right, sb_stream_t stream);
int sb_train_gt(const float* boxes_left, const float* boxes_right, const float* boxes_merge, const int* gt_classes,
                const float* dim_orien, const float* kpts, const int* n_rows, const unsigned* words, int B, int N,
                float im_scale, int im_width, float* gt_left, float* gt_right, float* gt_merge,
                float* gt_dim_orien, float* gt_kpts, int* num_boxes, sb_stream_t stream);
int sb_random_words(unsigned long long seed, const unsigned long long* step, unsigned stream_id, unsigned* out,
                    size_t n, sb_stream_t stream);
int sb_step_advance(unsigned long long* step, sb_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * KITTI average precision of a split (Car), the KITTI object devkit's evaluate_object restated (DESIGN.md §9).
 *
 * Rows: SB_KITTI_ROW doubles per label / result line -- trunc, occ, alpha, x1, y1, x2, y2, h, w, l, x, y, z, cos(ry),
 * sin(ry), score (0 for labels) -- and an int32 code per row: 0 Car, 1 Van, 2 DontCare, 3 anything else.  Images are
 * in CSR form: the gt rows of image i are gt_off[i] .. gt_off[i+1], its detection rows det_off[i] .. det_off[i+1], and
 * its pairs pair_off[i] .. pair_off[i+1], with pair_off[i+1] - pair_off[i] = n_det(i) * n_gt(i) (int64 offsets in
 * DEVICE memory, offsets[0] = 0).  Rows must be finite.
 * sb_kitti_overlaps -- the devkit's boxoverlap, groundBoxOverlap and box3DOverlap for every (detection, gt) pair of
 *   every image: the pair (j, i) of image k is element pair_off[k] + j * n_gt(k) + i of each output.  A DontCare gt
 *   column holds intersection / area(det) (the devkit's criterion 0), every other column intersection / union.
 * sb_kitti_eval -- eval_class for 3 metrics (2D, BEV, 3D) x n_bars IoU bars x 3 difficulties (easy, moderate, hard):
 *   configuration c = (metric * n_bars + bar) * 3 + difficulty, C = 9 * n_bars.  computeStatistics without and with
 *   false positives, getThresholds, and the precision / recall / orientation-similarity curves.  Outputs per
 *   configuration: thresholds [C,41] (0 past n_thresholds[c]), n_thresholds [C] int32, tp / fp / fn [C,41] int64,
 *   sim [C,41] (summed orientation similarity), precision / recall / aos [C,41] (precision and aos replaced by their
 *   maxima to the right), ap [C,4] = (precision R11, precision R40, aos R11, aos R40) in percent, n_gt [C] int64.
 *   bars: host array of n_bars (1..SB_KITTI_MAX_BARS) values in [0, 1].  The workspace is 256-byte aligned and at
 *   least sb_kitti_eval_workspace_bytes (0 for sizes it refuses).
 * SB_EINVAL before any launch for a null pointer, n_images < 1, a negative row or pair count, a bar outside [0, 1] or
 *   a workspace that is too small or misaligned.                                                                  */
#define SB_KITTI_ROW 16
#define SB_KITTI_MAX_THRESHOLDS 41
#define SB_KITTI_MAX_BARS 4

int sb_kitti_overlaps(const double* gt, const int* gt_code, const double* det, const long long* gt_off,
                      const long long* det_off, const long long* pair_off, int n_images, long long n_pairs,
                      double* ov_2d, double* ov_bev, double* ov_3d, sb_stream_t stream);
size_t sb_kitti_eval_workspace_bytes(int n_images, long long n_gt_rows, long long n_det_rows, long long n_pairs,
                                     int n_bars);
int sb_kitti_eval(const double* gt, const int* gt_code, const double* det, const int* det_code,
                  const long long* gt_off, const long long* det_off, const long long* pair_off, int n_images,
                  long long n_gt_rows, long long n_det_rows, long long n_pairs, const double* bars, int n_bars,
                  void* workspace, size_t workspace_bytes, double* thresholds, int* n_thresholds, long long* tp,
                  long long* fp, long long* fn, double* sim, double* precision, double* recall, double* aos,
                  double* ap, long long* n_gt, sb_stream_t stream);

/* ---------------------------------------------------------------------------------------------------------------
 * The training ground truth of a KITTI split (the reference's gt_roidb, DESIGN.md §10): kitti_utils.read_obj_data,
 * kitti.remove_occluded_keypoints for the left and then the right camera, and _load_kitti_annotation's filter.
 *
 * Rows: SB_KITTI_ANN_IN doubles per label line of type Car, Van, Truck or Misc (every other line is left out by the
 * caller) -- trunc, occ, alpha, w, h, l, x, y, z, cos(ry + pi/2), sin(ry + pi/2) -- and an int32 code per row: 0 Car,
 * 1 another of those types.  The rows of image i are obj_off[i] .. obj_off[i+1] in label order (int64 offsets in
 * DEVICE memory, obj_off[0] = 0; no cap per image).  calib: SB_KITTI_ANN_CALIB doubles per image in DEVICE memory --
 * p2_2 (P2 with [0,3] = 0), p2_3 (P3 with [0,3] = P3[0,3] - P2[0,3]), both 3x4 row-major, then t = (P2[0,3] -
 * P0[0,3]) / P2[0,0]; image_hw: int32 [n_images, 2] (H, W of the left image) in DEVICE memory.
 * sb_kitti_annotations -- one CTA per image, fp64 throughout.  Outputs: the kept rows of image i, in label order, at
 *   rows obj_off[i] .. obj_off[i] + n_kept[i] of out (float32 [n_rows, SB_KITTI_ANN_OUT]: boxes_left[4],
 *   boxes_right[4], boxes_merge[4], dim_orien[4] = (w, h, l, alpha), kpts[6] = (4 keypoints, visible left, visible
 *   right) of the left camera, kpts_right[6] of the right camera, truncation, occlusion), zeros in the image's other
 *   rows; n_kept [n_images] int32; status [n_images] int32: 0, 1 + the index (within the image's rows) of the object
 *   the reference indexes the SB_KITTI_DEPTH_COLS-column depth line out of range with (it raises IndexError there;
 *   nothing is kept) -- the first whose painted columns int(x1) .. int(x2) reach past the line, else the first with
 *   int(x1) or int(x2) past it -- or -1 for an image whose H or W is not positive (nothing is kept).  The workspace is 256-byte
 *   aligned and at least sb_kitti_annotations_workspace_bytes (0 for sizes it refuses).
 * SB_EINVAL before any launch for a null pointer, n_images < 1, a negative row count or a workspace that is too small
 *   or misaligned.                                                                                                 */
#define SB_KITTI_ANN_IN 11
#define SB_KITTI_ANN_OUT 30
#define SB_KITTI_ANN_CALIB 25
#define SB_KITTI_DEPTH_COLS 1260

size_t sb_kitti_annotations_workspace_bytes(int n_images, long long n_rows);
int sb_kitti_annotations(const double* rows, const int* codes, const long long* obj_off, const double* calib,
                         const int* image_hw, int n_images, long long n_rows, void* workspace,
                         size_t workspace_bytes, float* out, int* n_kept, int* status, sb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* STEREO_B200_H */
