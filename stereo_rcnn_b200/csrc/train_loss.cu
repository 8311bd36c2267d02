// train_loss.cu -- the training losses of the reference and their gradients w.r.t. the network outputs
// (SURVEY A16): what `loss.backward()` (trainval_net.py:226) feeds into the heads.
//
//   sb_rpn_loss        lib/model/rpn/stereo_rpn.py:114-140   CE over the sampled anchors + smooth-L1 (sigma 3) on the
//                                                            6-d left/right deltas
//   sb_rcnn_loss       lib/model/stereo_rcnn/stereo_rcnn.py:201-311  CE, smooth-L1 box (6-d, class-selected) and
//                                                            dimension/orientation (5-d), weighted CE on keypoint /
//                                                            left-border / right-border bins
//   sb_multitask_loss  trainval_net.py:214-219               sum_i L_i exp(-u_i) + u_i
//   sb_clip_gradient   lib/model/utils/net_utils.py:37-49    global-norm clipping (one pass, no per-parameter sync)
//
// _smooth_l1_loss is net_utils.py:79-99.  Reductions are two-level with a fixed order (per-CTA partial sums in
// double, then one CTA), so the losses are deterministic run to run; the reference's are not (atomics in cuDNN/THC).
// Gradients carry the multi-task factor exp(-u_i) when `uncert` is given (d total / d L_i), else 1.
#include "common.cuh"

namespace {

constexpr int kPartBlocks = 512;

__device__ __forceinline__ double block_sum(double v, double* s_buf) {      // all threads get the total; fixed order
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    __syncthreads();
    if (lane == 0) s_buf[warp] = v;
    __syncthreads();
    double t = 0.0;
    const int nw = (blockDim.x + 31) >> 5;
    for (int w = 0; w < nw; ++w) t += s_buf[w];
    return t;
}

// smooth-L1 of one element (net_utils.py:82-93): x = inside * (pred - target); returns outside * f(x), and the
// derivative w.r.t. pred in *g
__device__ __forceinline__ float smooth_l1(float pred, float target, float iw, float ow, float sigma2, float* g) {
    const float x = iw * (pred - target);
    const float a = fabsf(x);
    const bool quad = a < 1.f / sigma2;
    const float l = quad ? x * x * (sigma2 * 0.5f) : a - 0.5f / sigma2;
    *g = ow * iw * (quad ? sigma2 * x : (x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f)));
    return ow * l;
}

// ------------------------------------------------------------------------------------------------ RPN loss
struct RpnArgs {
    const float* cls_score;   // [n][2]
    const float* bbox_pred;   // [n][6]
    const float* labels;      // [n]
    const float4* tl;         // [n]
    const float4* tr;
    const float* inside_w;    // [n]
    const float* outside_w;
    long long n;              // B * A
    int B;
};

__global__ void __launch_bounds__(256)
rpn_loss_partial_kernel(const RpnArgs a, double* __restrict__ partial /*[kPartBlocks][3]*/) {
    __shared__ double s_buf[8];
    double ce = 0.0, sl = 0.0, cnt = 0.0;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n; i += (long long)gridDim.x * blockDim.x) {
        const float lab = a.labels[i];
        if (lab != -1.f) {
            const float s0 = a.cls_score[2 * i], s1 = a.cls_score[2 * i + 1];
            // lse - s = (m - s) + log1p(exp(-|s0 - s1|)): m + log(...) - s would cancel the small loss of a
            // well-classified anchor in fp32
            const float m = fmaxf(s0, s1);
            ce += (double)((m - (lab != 0.f ? s1 : s0)) + log1pf(expf(-fabsf(s0 - s1))));
            cnt += 1.0;
        }
        const float ow = a.outside_w[i];
        if (ow != 0.f) {
            const float iw = a.inside_w[i];
            const float4 l = a.tl[i], r = a.tr[i];
            const float t[6] = {l.x, l.y, l.z, l.w, r.x, r.z};         // stereo_rpn.py:128-131
            float g;
#pragma unroll
            for (int c = 0; c < 6; ++c) sl += (double)smooth_l1(a.bbox_pred[6 * i + c], t[c], iw, ow, 9.f, &g);
        }
    }
    ce = block_sum(ce, s_buf);
    sl = block_sum(sl, s_buf);
    cnt = block_sum(cnt, s_buf);
    if (threadIdx.x == 0) {
        partial[blockIdx.x * 3 + 0] = ce;
        partial[blockIdx.x * 3 + 1] = sl;
        partial[blockIdx.x * 3 + 2] = cnt;
    }
}

__global__ void __launch_bounds__(256)
rpn_loss_final_kernel(const double* __restrict__ partial, int nblocks, int B, float* __restrict__ losses,
                      double* __restrict__ scal /*[1]: n_keep*/) {
    __shared__ double s_buf[8];
    double ce = 0.0, sl = 0.0, cnt = 0.0;
    for (int i = threadIdx.x; i < nblocks; i += blockDim.x) {
        ce += partial[i * 3];
        sl += partial[i * 3 + 1];
        cnt += partial[i * 3 + 2];
    }
    ce = block_sum(ce, s_buf);
    sl = block_sum(sl, s_buf);
    cnt = block_sum(cnt, s_buf);
    if (threadIdx.x == 0) {
        losses[0] = (float)(ce / cnt);                                 // F.cross_entropy: mean over the kept anchors
        losses[1] = (float)(sl / (6.0 * B));                           // sum over dim 1, mean over [B, 6]
        scal[0] = cnt;
    }
}

__global__ void __launch_bounds__(256)
rpn_loss_grad_kernel(const RpnArgs a, const double* __restrict__ scal, const float* __restrict__ uncert,
                     float* __restrict__ d_cls, float* __restrict__ d_box) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= a.n) return;
    const float g_cls = (uncert ? expf(-uncert[0]) : 1.f) / (float)scal[0];
    const float g_box = (uncert ? expf(-uncert[1]) : 1.f) / (6.f * a.B);
    const float lab = a.labels[i];
    float d0 = 0.f, d1 = 0.f;
    if (lab != -1.f) {
        const float s0 = a.cls_score[2 * i], s1 = a.cls_score[2 * i + 1];
        // softmax of two logits: p_big = 1 / (1 + e), p_small = e / (1 + e), e = exp(-|s0 - s1|); the labelled
        // class's p - 1 is minus the other class's p, which does not cancel when p is close to 1
        const float e = expf(-fabsf(s0 - s1));
        const float inv = 1.f / (1.f + e);
        const float p0 = s0 >= s1 ? inv : e * inv, p1 = s0 >= s1 ? e * inv : inv;
        d0 = (lab != 0.f ? p0 : -p1) * g_cls;
        d1 = (lab != 0.f ? -p0 : p1) * g_cls;
    }
    d_cls[2 * i] = d0;
    d_cls[2 * i + 1] = d1;
    const float ow = a.outside_w[i], iw = a.inside_w[i];
    const float4 l = a.tl[i], r = a.tr[i];
    const float t[6] = {l.x, l.y, l.z, l.w, r.x, r.z};
#pragma unroll
    for (int c = 0; c < 6; ++c) {
        float g = 0.f;
        if (ow != 0.f) smooth_l1(a.bbox_pred[6 * i + c], t[c], iw, ow, 9.f, &g);
        d_box[6 * i + c] = g * g_box;
    }
}

// ----------------------------------------------------------------------------------------------- RCNN loss
struct RcnnArgs {
    const float* cls_score;      // [R][C]
    const float* bbox_pred;      // [R][6C]
    const float* dim_pred;       // [R][5C]
    const float* kpts_pred;      // [R][4G]
    const float* left_pred;      // [R][G]
    const float* right_pred;     // [R][G]
    const float* labels;         // [R]
    const float4* tl;            // [R]
    const float4* tr;
    const float* tdim;           // [R][5]
    const int* tkpts;            // [R][3]
    const float* wkpts;          // [R][3]
    const float4* inside_w;      // [R]
    const float4* outside_w;
    int R, C, G;
    const float* uncert;         // nullable; entries 2..5
    float* losses;               // [4]
    float* d_cls;                // nullable group
    float* d_bbox;
    float* d_dim;
    float* d_kpts;
    float* d_left;
    float* d_right;
};

// cross entropy of one row of n logits against class `cls`; optionally writes coef * (softmax - onehot)
__device__ __forceinline__ float row_ce(const float* __restrict__ x, int n, int cls, float* __restrict__ dx, float coef) {
    float m = -INFINITY;
    for (int j = 0; j < n; ++j) m = fmaxf(m, x[j]);
    float s = 0.f;
    for (int j = 0; j < n; ++j) s += expf(x[j] - m);
    if (dx) {
        const float inv = 1.f / s;
        for (int j = 0; j < n; ++j) dx[j] = coef * (expf(x[j] - m) * inv - (j == cls ? 1.f : 0.f));
    }
    return (m - x[cls]) + logf(s);                      // no cancellation of a small loss (see rpn_loss_partial_kernel)
}

__global__ void __launch_bounds__(1024)
rcnn_loss_kernel(const RcnnArgs a) {
    __shared__ double s_buf[32];
    __shared__ double s_w[3];
    const int R = a.R, C = a.C, G = a.G;
    double ce = 0.0, sb = 0.0, sd = 0.0, ck[3] = {0.0, 0.0, 0.0}, wk[3] = {0.0, 0.0, 0.0};
    for (int r = threadIdx.x; r < R; r += blockDim.x) {
        const int lab = (int)a.labels[r];
        ce += (double)row_ce(a.cls_score + (size_t)r * C, C, lab, nullptr, 0.f);
        const float4 l = a.tl[r], rr = a.tr[r], iw4 = a.inside_w[r], ow4 = a.outside_w[r];
        const float t[6] = {l.x, l.y, l.z, l.w, rr.x, rr.z};                    // stereo_rcnn.py:204-207
        const float iw[6] = {iw4.x, iw4.y, iw4.z, iw4.w, iw4.x, iw4.y};         // :209-215
        const float ow[6] = {ow4.x, ow4.y, ow4.z, ow4.w, ow4.x, ow4.y};
        const float* bp = a.bbox_pred + ((size_t)r * C + lab) * 6;              // gather by label (:268-270)
        const float* dp = a.dim_pred + ((size_t)r * C + lab) * 5;
        float g;
#pragma unroll
        for (int c = 0; c < 6; ++c) sb += (double)smooth_l1(bp[c], t[c], iw[c], ow[c], 1.f, &g);
#pragma unroll
        for (int c = 0; c < 5; ++c) sd += (double)smooth_l1(dp[c], a.tdim[(size_t)r * 5 + c], 1.f, 1.f, 1.f, &g);
        const float* preds[3] = {a.kpts_pred + (size_t)r * 4 * G, a.left_pred + (size_t)r * G, a.right_pred + (size_t)r * G};
        const int width[3] = {4 * G, G, G};
#pragma unroll
        for (int h = 0; h < 3; ++h) {
            const float w = a.wkpts[(size_t)r * 3 + h];
            wk[h] += (double)w;
            if (w != 0.f) ck[h] += (double)(row_ce(preds[h], width[h], a.tkpts[(size_t)r * 3 + h], nullptr, 0.f) * w);
        }
    }
    ce = block_sum(ce, s_buf);
    sb = block_sum(sb, s_buf);
    sd = block_sum(sd, s_buf);
    double lk = 0.0;
#pragma unroll
    for (int h = 0; h < 3; ++h) {
        ck[h] = block_sum(ck[h], s_buf);
        wk[h] = block_sum(wk[h], s_buf);
        lk += wk[h] < 1.0 ? ck[h] : ck[h] / wk[h];                              // :291-306
    }
    if (threadIdx.x == 0) {
        a.losses[0] = (float)(ce / R);
        a.losses[1] = (float)(sb / R);
        a.losses[2] = (float)(sd / R);
        a.losses[3] = (float)(lk / 3.0);
        for (int h = 0; h < 3; ++h) s_w[h] = wk[h] < 1.0 ? 1.0 : wk[h];
    }
    __syncthreads();
    if (!a.d_cls) return;
    const float e2 = a.uncert ? expf(-a.uncert[2]) : 1.f, e3 = a.uncert ? expf(-a.uncert[3]) : 1.f;
    const float e4 = a.uncert ? expf(-a.uncert[4]) : 1.f, e5 = a.uncert ? expf(-a.uncert[5]) : 1.f;
    for (int r = threadIdx.x; r < R; r += blockDim.x) {
        const int lab = (int)a.labels[r];
        row_ce(a.cls_score + (size_t)r * C, C, lab, a.d_cls + (size_t)r * C, e2 / R);
        const float4 l = a.tl[r], rr = a.tr[r], iw4 = a.inside_w[r], ow4 = a.outside_w[r];
        const float t[6] = {l.x, l.y, l.z, l.w, rr.x, rr.z};
        const float iw[6] = {iw4.x, iw4.y, iw4.z, iw4.w, iw4.x, iw4.y};
        const float ow[6] = {ow4.x, ow4.y, ow4.z, ow4.w, ow4.x, ow4.y};
        for (int c = 0; c < C; ++c) {
            float* db = a.d_bbox + ((size_t)r * C + c) * 6;
            float* dd = a.d_dim + ((size_t)r * C + c) * 5;
            const float* bp = a.bbox_pred + ((size_t)r * C + c) * 6;
            const float* dp = a.dim_pred + ((size_t)r * C + c) * 5;
#pragma unroll
            for (int k = 0; k < 6; ++k) {
                float g = 0.f;
                if (c == lab) smooth_l1(bp[k], t[k], iw[k], ow[k], 1.f, &g);
                db[k] = g * (e3 / R);
            }
#pragma unroll
            for (int k = 0; k < 5; ++k) {
                float g = 0.f;
                if (c == lab) smooth_l1(dp[k], a.tdim[(size_t)r * 5 + k], 1.f, 1.f, 1.f, &g);
                dd[k] = g * (e4 / R);
            }
        }
        const float* preds[3] = {a.kpts_pred + (size_t)r * 4 * G, a.left_pred + (size_t)r * G, a.right_pred + (size_t)r * G};
        float* outs[3] = {a.d_kpts + (size_t)r * 4 * G, a.d_left + (size_t)r * G, a.d_right + (size_t)r * G};
        const int width[3] = {4 * G, G, G};
#pragma unroll
        for (int h = 0; h < 3; ++h) {
            const float w = a.wkpts[(size_t)r * 3 + h];
            if (w != 0.f) {
                row_ce(preds[h], width[h], a.tkpts[(size_t)r * 3 + h], outs[h], w * e5 / (3.f * (float)s_w[h]));
            } else {
                for (int j = 0; j < width[h]; ++j) outs[h][j] = 0.f;
            }
        }
    }
}

__global__ void multitask_kernel(const float* __restrict__ losses, const float* __restrict__ uncert, int n,
                                 float* __restrict__ total, float* __restrict__ d_uncert) {
    if (threadIdx.x || blockIdx.x) return;
    float t = 0.f;
    for (int i = 0; i < n; ++i) {                                          // trainval_net.py:214-219, left to right
        const float e = expf(-uncert[i]);
        t = t + losses[i] * e + uncert[i];
        if (d_uncert) d_uncert[i] = 1.f - losses[i] * e;
    }
    total[0] = t;
}

// --------------------------------------------------------------------------------------------- clip_gradient
constexpr int kClipTensors = 48, kClipSlices = 32;
struct ClipChunk {
    float* g[kClipTensors];
    unsigned long long n[kClipTensors];
    int count;
};

__global__ void __launch_bounds__(256)
clip_sumsq_kernel(const ClipChunk c, double* __restrict__ partial /*[tensors][kClipSlices]*/, int base) {
    __shared__ double s_buf[8];
    const int t = blockIdx.x, s = blockIdx.y;
    const unsigned long long n = c.n[t];
    const unsigned long long per = (n + kClipSlices - 1) / kClipSlices;
    const unsigned long long lo = per * s, hi = lo + per < n ? lo + per : n;
    double acc = 0.0;
    for (unsigned long long i = lo + threadIdx.x; i < hi; i += blockDim.x) {
        const float v = c.g[t][i];
        acc += (double)v * (double)v;
    }
    acc = block_sum(acc, s_buf);
    if (threadIdx.x == 0) partial[(size_t)(base + t) * kClipSlices + s] = acc;
}

__global__ void __launch_bounds__(256)
clip_norm_kernel(const double* __restrict__ partial, int n_tensors, float clip, float* __restrict__ out /*[2]*/) {
    __shared__ double s_buf[8];
    double acc = 0.0;
    for (int i = threadIdx.x; i < n_tensors * kClipSlices; i += blockDim.x) acc += partial[i];
    acc = block_sum(acc, s_buf);
    if (threadIdx.x == 0) {
        const float total = (float)sqrt(acc);
        out[0] = total;
        out[1] = clip / fmaxf(total, clip);                                 // net_utils.py:46
    }
}

__global__ void __launch_bounds__(256)
clip_scale_kernel(const ClipChunk c, const float* __restrict__ norm) {
    const int t = blockIdx.x, s = blockIdx.y;
    const float f = norm[1];
    if (f == 1.f) return;
    const unsigned long long n = c.n[t];
    const unsigned long long per = (n + kClipSlices - 1) / kClipSlices;
    const unsigned long long lo = per * s, hi = lo + per < n ? lo + per : n;
    for (unsigned long long i = lo + threadIdx.x; i < hi; i += blockDim.x) c.g[t][i] *= f;
}

}  // namespace

extern "C" size_t sb_loss_workspace_bytes(void) { return (size_t)kPartBlocks * 3 * 8 + 64; }

extern "C" int sb_rpn_loss(const float* rpn_cls_score, const float* rpn_bbox_pred, const float* labels,
                           const float* targets_left, const float* targets_right, const float* inside_w,
                           const float* outside_w, int B, int A, const float* uncert, void* workspace,
                           size_t workspace_bytes, float* losses, float* d_cls_score, float* d_bbox_pred,
                           sb_stream_t stream) {
    if (!rpn_cls_score || !rpn_bbox_pred || !labels || !targets_left || !targets_right || !inside_w || !outside_w ||
        !workspace || !losses || B < 1 || A < 1 || workspace_bytes < sb_loss_workspace_bytes() ||
        (d_cls_score == nullptr) != (d_bbox_pred == nullptr))
        return SB_EINVAL;
    if ((reinterpret_cast<uintptr_t>(targets_left) | reinterpret_cast<uintptr_t>(targets_right) |
         reinterpret_cast<uintptr_t>(workspace)) & 15)
        return SB_EINVAL;
    RpnArgs a;
    a.cls_score = rpn_cls_score; a.bbox_pred = rpn_bbox_pred; a.labels = labels;
    a.tl = reinterpret_cast<const float4*>(targets_left); a.tr = reinterpret_cast<const float4*>(targets_right);
    a.inside_w = inside_w; a.outside_w = outside_w; a.n = (long long)B * A; a.B = B;
    double* partial = static_cast<double*>(workspace);
    double* scal = partial + (size_t)kPartBlocks * 3;
    cudaStream_t st = sb_cs(stream);
    const int blocks = (int)((a.n + 255) / 256 < kPartBlocks ? (a.n + 255) / 256 : kPartBlocks);
    rpn_loss_partial_kernel<<<blocks, 256, 0, st>>>(a, partial);
    SB_LAUNCHED();
    rpn_loss_final_kernel<<<1, 256, 0, st>>>(partial, blocks, B, losses, scal);
    SB_LAUNCHED();
    if (d_cls_score) {
        rpn_loss_grad_kernel<<<sb_div_up(a.n, 256), 256, 0, st>>>(a, scal, uncert, d_cls_score, d_bbox_pred);
        SB_LAUNCHED();
    }
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" int sb_rcnn_loss(const float* cls_score, const float* bbox_pred, const float* dim_orien_pred,
                            const float* kpts_pred, const float* left_border_pred, const float* right_border_pred,
                            const float* labels, const float* bbox_targets_left, const float* bbox_targets_right,
                            const float* dim_orien_targets, const int* kpts_targets, const float* kpts_weight,
                            const float* inside_w, const float* outside_w, int R, int n_classes, int kpts_grid,
                            const float* uncert, float* losses, float* d_cls_score, float* d_bbox_pred,
                            float* d_dim_orien_pred, float* d_kpts_pred, float* d_left_border_pred,
                            float* d_right_border_pred, sb_stream_t stream) {
    if (!cls_score || !bbox_pred || !dim_orien_pred || !kpts_pred || !left_border_pred || !right_border_pred || !labels ||
        !bbox_targets_left || !bbox_targets_right || !dim_orien_targets || !kpts_targets || !kpts_weight || !inside_w ||
        !outside_w || !losses || R < 1 || n_classes < 2 || kpts_grid < 1)
        return SB_EINVAL;
    const int ng = (d_cls_score != nullptr) + (d_bbox_pred != nullptr) + (d_dim_orien_pred != nullptr) +
                   (d_kpts_pred != nullptr) + (d_left_border_pred != nullptr) + (d_right_border_pred != nullptr);
    if (ng != 0 && ng != 6) return SB_EINVAL;
    if ((reinterpret_cast<uintptr_t>(bbox_targets_left) | reinterpret_cast<uintptr_t>(bbox_targets_right) |
         reinterpret_cast<uintptr_t>(inside_w) | reinterpret_cast<uintptr_t>(outside_w)) & 15)
        return SB_EINVAL;
    RcnnArgs a;
    a.cls_score = cls_score; a.bbox_pred = bbox_pred; a.dim_pred = dim_orien_pred; a.kpts_pred = kpts_pred;
    a.left_pred = left_border_pred; a.right_pred = right_border_pred; a.labels = labels;
    a.tl = reinterpret_cast<const float4*>(bbox_targets_left); a.tr = reinterpret_cast<const float4*>(bbox_targets_right);
    a.tdim = dim_orien_targets; a.tkpts = kpts_targets; a.wkpts = kpts_weight;
    a.inside_w = reinterpret_cast<const float4*>(inside_w); a.outside_w = reinterpret_cast<const float4*>(outside_w);
    a.R = R; a.C = n_classes; a.G = kpts_grid; a.uncert = uncert; a.losses = losses;
    a.d_cls = d_cls_score; a.d_bbox = d_bbox_pred; a.d_dim = d_dim_orien_pred; a.d_kpts = d_kpts_pred;
    a.d_left = d_left_border_pred; a.d_right = d_right_border_pred;
    rcnn_loss_kernel<<<1, 1024, 0, sb_cs(stream)>>>(a);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" int sb_multitask_loss(const float* losses, const float* uncert, int n, float* total, float* d_uncert,
                                 sb_stream_t stream) {
    if (!losses || !uncert || !total || n < 1 || n > 64) return SB_EINVAL;
    multitask_kernel<<<1, 32, 0, sb_cs(stream)>>>(losses, uncert, n, total, d_uncert);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" size_t sb_clip_gradient_workspace(int n_tensors) {
    return n_tensors < 1 ? 0 : (size_t)n_tensors * kClipSlices * 8 + 64;
}

extern "C" int sb_clip_gradient(float* const* grads, const size_t* counts, int n_tensors, float clip_norm,
                                void* workspace, size_t workspace_bytes, float* norm_out, sb_stream_t stream) {
    if (!grads || !counts || n_tensors < 1 || !(clip_norm > 0.f) || !workspace || !norm_out ||
        workspace_bytes < sb_clip_gradient_workspace(n_tensors) || (reinterpret_cast<uintptr_t>(workspace) & 7))
        return SB_EINVAL;
    for (int i = 0; i < n_tensors; ++i)
        if (!grads[i] || counts[i] == 0) return SB_EINVAL;
    cudaStream_t st = sb_cs(stream);
    double* partial = static_cast<double*>(workspace);
    for (int base = 0; base < n_tensors; base += kClipTensors) {
        ClipChunk c;
        c.count = n_tensors - base < kClipTensors ? n_tensors - base : kClipTensors;
        for (int i = 0; i < kClipTensors; ++i) {
            c.g[i] = i < c.count ? grads[base + i] : nullptr;
            c.n[i] = i < c.count ? (unsigned long long)counts[base + i] : 0ull;
        }
        clip_sumsq_kernel<<<dim3(c.count, kClipSlices), 256, 0, st>>>(c, partial, base);
        SB_LAUNCHED();
    }
    clip_norm_kernel<<<1, 256, 0, st>>>(partial, n_tensors, clip_norm, norm_out);
    SB_LAUNCHED();
    for (int base = 0; base < n_tensors; base += kClipTensors) {
        ClipChunk c;
        c.count = n_tensors - base < kClipTensors ? n_tensors - base : kClipTensors;
        for (int i = 0; i < kClipTensors; ++i) {
            c.g[i] = i < c.count ? grads[base + i] : nullptr;
            c.n[i] = i < c.count ? (unsigned long long)counts[base + i] : 0ull;
        }
        clip_scale_kernel<<<dim3(c.count, kClipSlices), 256, 0, st>>>(c, norm_out);
        SB_LAUNCHED();
    }
    SB_CHECK_LAUNCH();
    return SB_OK;
}
