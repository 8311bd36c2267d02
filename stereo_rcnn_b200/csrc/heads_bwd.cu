// heads_bwd.cu -- the pieces of the R-CNN heads' training pass that the tensor-core convolutions cannot express
// (sm_90a): dropout from explicit random words, the raw keypoint logits the loss reads, the fp32 backward of the box
// tail's three linears, the backward of the keypoint tail (kpts_class over the height-summed deconv output) into the
// deconv's phase-major gradient, and the permutation of weight gradients into the reference's layout.
// Every reduction runs in a fixed order (no atomics): results are bit-identical run to run.
#include <cuda_fp16.h>

#include "common.cuh"

namespace {

// x[i] = word[i] < thr ? 0 : x[i] * scale (in place; fp16 or fp32)
__global__ void __launch_bounds__(256)
dropout_kernel(void* __restrict__ x, int is_half, long long n, const unsigned* __restrict__ words,
               unsigned long long thr, float scale) {
    const long long stride = (long long)gridDim.x * 256;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += stride) {
        const bool drop = (unsigned long long)__ldg(words + i) < thr;
        if (is_half) {
            __half* p = reinterpret_cast<__half*>(x) + i;
            *p = drop ? __float2half_rn(0.f) : __float2half_rn(__half2float(*p) * scale);
        } else {
            float* p = reinterpret_cast<float*>(x) + i;
            *p = drop ? 0.f : *p * scale;
        }
    }
}

// [R,6,G] logits -> kpts_pred [R,4G] (channels 0..3), left [R,G] (4), right [R,G] (5)
__global__ void __launch_bounds__(256)
kpts_logits_kernel(const float* __restrict__ pred_all, long long n, int G, float* __restrict__ kp,
                   float* __restrict__ lb, float* __restrict__ rb) {
    const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
    if (i >= n) return;
    const long long r = i / (6 * G);
    const int k = (int)(i / G % 6), x = (int)(i % G);
    const float v = pred_all[i];
    if (k < 4) kp[r * 4 * G + k * G + x] = v;
    else (k == 4 ? lb : rb)[r * G + x] = v;
}

struct BoxTailGrad {
    const float *d_cls, *d_box, *d_dim;     // [R,nc], [R,6nc], [R,5nc]
    const float *w_cls, *w_box, *w_dim;     // [nc,K], [6nc,K], [5nc,K]
    float *dw_cls, *db_cls, *dw_box, *db_box, *dw_dim, *db_dim;
};

// output o of the concatenation (cls | box | dim): its gradient column and weight / gradient rows
__device__ __forceinline__ void box_out(const BoxTailGrad& a, int nc, int o, const float** d, int* ld, int* col,
                                        const float** w, float** dw, float** db) {
    if (o < nc) { *d = a.d_cls; *ld = nc; *col = o; *w = a.w_cls; *dw = a.dw_cls; *db = a.db_cls; }
    else if (o < 7 * nc) { *d = a.d_box; *ld = 6 * nc; *col = o - nc; *w = a.w_box; *dw = a.dw_box; *db = a.db_box; }
    else { *d = a.d_dim; *ld = 5 * nc; *col = o - 7 * nc; *w = a.w_dim; *dw = a.dw_dim; *db = a.db_dim; }
}

// d pre-activation of RCNN_top.3: dz[r][k] = grad_scale * mask_scale * [fc7[r][k] > 0] * sum_o d[r][o] W[o][k]
// (o ascending: cls, box, dim); grid (R, K / 256).  DEV_SCALE: grad_scale is read from gs_dev (device, fp32 [1])
template <bool DEV_SCALE>
__global__ void __launch_bounds__(256)
box_tail_dx_kernel(BoxTailGrad a, int nc, const float* __restrict__ fc7, int K, float mask_scale, float gs,
                   const float* __restrict__ gs_dev, __half* __restrict__ dz16, float* __restrict__ dz32,
                   int* nonfinite) {
    __shared__ float dv[48];
    if (DEV_SCALE) gs = __ldg(gs_dev);
    const int r = blockIdx.x, tid = threadIdx.x, n_out = 12 * nc;
    if (tid < n_out) {
        const float* d; const float* w; float *dw, *db; int ld, col;
        box_out(a, nc, tid, &d, &ld, &col, &w, &dw, &db);
        dv[tid] = d[(size_t)r * ld + col];
    }
    __syncthreads();
    const int k = blockIdx.y * 256 + tid;
    if (k >= K) return;
    float s = 0.f;
    for (int o = 0; o < n_out; ++o) {
        const float* w = o < nc ? a.w_cls + (size_t)o * K
                       : (o < 7 * nc ? a.w_box + (size_t)(o - nc) * K : a.w_dim + (size_t)(o - 7 * nc) * K);
        s = fmaf(dv[o], __ldg(w + k), s);
    }
    const size_t e = (size_t)r * K + k;
    const float v = fc7[e] > 0.f ? s * mask_scale * gs : 0.f;
    const __half h = __float2half_rn(v);
    dz32[e] = v;
    dz16[e] = h;
    if (nonfinite && (!isfinite(v) || __hisinf(h))) *nonfinite = 1;
}

// sum over r of f(r) with eight interleaved partial sums combined as a tree: a fixed order, error ~ (R/8 + 3) ulp
template <typename F>
__device__ __forceinline__ float ordered_sum(int R, F f) {
    float p[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    int r = 0;
    for (; r + 7 < R; r += 8) {
#pragma unroll
        for (int j = 0; j < 8; ++j) p[j] += f(r + j);
    }
    for (int j = 0; r < R; ++r, ++j) p[j] += f(r);
    return ((p[0] + p[1]) + (p[2] + p[3])) + ((p[4] + p[5]) + (p[6] + p[7]));
}

// dW[o][k] = sum_r d[r][o] fc7[r][k], db[o] = sum_r d[r][o]; grid (K / 256, 12nc), one thread per (o, k)
__global__ void __launch_bounds__(256)
box_tail_dw_kernel(BoxTailGrad a, int nc, int R, const float* __restrict__ fc7, int K, int* nonfinite) {
    const int o = blockIdx.y, k = blockIdx.x * 256 + threadIdx.x;
    const float* d; const float* w; float *dw, *db; int ld, col;
    box_out(a, nc, o, &d, &ld, &col, &w, &dw, &db);
    if (k < K) {
        const float v = ordered_sum(R, [&](int r) { return d[(size_t)r * ld + col] * fc7[(size_t)r * K + k]; });
        dw[(size_t)col * K + k] = v;
        if (nonfinite && !isfinite(v)) *nonfinite = 1;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const float v = ordered_sum(R, [&](int r) { return d[(size_t)r * ld + col]; });
        db[col] = v;
        if (nonfinite && !isfinite(v)) *nonfinite = 1;
    }
}

// Keypoint tail, one CTA per RoI, one thread per channel c (blockDim = C).  logits[k][x] = sum_c w[k][c] colsum[x][c]
// + G b[k] with colsum[x][c] = sum_y up[y][x][c], so with dp = d logits:
//   d up[y][x][c] = [up > 0] sum_k w[k][c] dp[k][x]   (the same for every y; stored x grad_scale, fp16, phase-major:
//                   pixel (y, x) -> (y / 2, x / 2), channel block (y % 2) * 2 + x % 2, the deconv's (a, b) phase)
//   per-RoI partials: dW[k][c] <- sum_x dp[k][x] colsum[x][c], d deconv bias[c] <- sum_{y,x} d up, sum_x dp[k][x]
// DEV_SCALE: grad_scale is read from gs_dev (device, fp32 [1])
template <bool DEV_SCALE>
__global__ void __launch_bounds__(1024)
kpts_tail_bwd_kernel(const __half* __restrict__ up, int G, int C, const float* __restrict__ w,
                     const float* __restrict__ d_kp, const float* __restrict__ d_lb, const float* __restrict__ d_rb,
                     float gs, const float* __restrict__ gs_dev, __half* __restrict__ dup, float* __restrict__ part,
                     int part_ld, int* nonfinite) {
    extern __shared__ float dp[];       // [6][G]
    if (DEV_SCALE) gs = __ldg(gs_dev);
    const int r = blockIdx.x, c = threadIdx.x, Gh = G / 2;
    for (int i = c; i < 6 * G; i += blockDim.x) {
        const int k = i / G, x = i % G;
        dp[i] = k < 4 ? d_kp[(size_t)r * 4 * G + i] : (k == 4 ? d_lb : d_rb)[(size_t)r * G + x];
    }
    __syncthreads();
    float wk[6], aw[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) { wk[k] = __ldg(w + k * C + c); aw[k] = 0.f; }
    float ab = 0.f;
    bool bad = false;
    const __half* ur = up + (size_t)r * G * G * C + c;
    __half* dr = dup + (size_t)r * G * G * C + c;
    const __half zero = __float2half_rn(0.f);
    for (int x = 0; x < G; ++x) {
        float g = 0.f;
#pragma unroll
        for (int k = 0; k < 6; ++k) g = fmaf(wk[k], dp[k * G + x], g);
        const __half h = __float2half_rn(g * gs);
        bad |= __hisinf(h) || !isfinite(g);
        float cs[4] = {0.f, 0.f, 0.f, 0.f};
        int on = 0;
        for (int y = 0; y < G; ++y) {
            const float u = __half2float(ur[((size_t)y * G + x) * C]);
            cs[y & 3] += u;
            on += u > 0.f;
            dr[(((size_t)(y >> 1) * Gh + (x >> 1)) * 4 + (y & 1) * 2 + (x & 1)) * C] = u > 0.f ? h : zero;
        }
        const float colsum = (cs[0] + cs[1]) + (cs[2] + cs[3]);
#pragma unroll
        for (int k = 0; k < 6; ++k) aw[k] = fmaf(dp[k * G + x], colsum, aw[k]);
        ab = fmaf(g, (float)on, ab);
    }
    float* pr = part + (size_t)r * part_ld;
#pragma unroll
    for (int k = 0; k < 6; ++k) pr[k * C + c] = aw[k];
    pr[6 * C + c] = ab;
    if (c < 6) {
        float s = 0.f;
        for (int x = 0; x < G; ++x) s += dp[c * G + x];
        pr[7 * C + c] = s;
    }
    if (bad && nonfinite) *nonfinite = 1;
}

// sums the per-RoI partials over r in a fixed order: dw [6][C], db_up [C], db [6] (= G * sum of d logits)
__global__ void __launch_bounds__(256)
kpts_tail_bwd_reduce_kernel(const float* __restrict__ part, int part_ld, int R, int C, int G, float* __restrict__ dw,
                            float* __restrict__ db, float* __restrict__ db_up, int* nonfinite) {
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= 7 * C + 6) return;
    float v = ordered_sum(R, [&](int r) { return part[(size_t)r * part_ld + i]; });
    if (i < 6 * C) dw[i] = v;
    else if (i < 7 * C) db_up[i - 6 * C] = v;
    else db[i - 7 * C] = v = v * (float)G;
    if (nonfinite && !isfinite(v)) *nonfinite = 1;
}

__global__ void __launch_bounds__(256)
permute3_kernel(const float* __restrict__ src, int d1, int d2, long long n, long long s0, long long s1, long long s2,
                float* __restrict__ dst) {
    const long long stride = (long long)gridDim.x * 256;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += stride) {
        const long long t = i / d2;
        dst[t / d1 * s0 + t % d1 * s1 + i % d2 * s2] = src[i];
    }
}

bool misaligned(const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) != 0; }

int grid_for(long long n) { return (int)(n < 256LL * 4 * 132 * 8 ? (n + 255) / 256 : 4 * 132 * 8); }

size_t kpts_part_ld(int C) { return (size_t)7 * C + 8; }

// grad_scale_dev (device, may be NULL): the gradient scale read on the device in place of grad_scale
int box_tail_backward(const float* d_cls_score, const float* d_bbox_pred, const float* d_dim_orien_pred,
                      const float* fc7, int R, int K, int n_classes, const float* w_cls, const float* w_box,
                      const float* w_dim, float mask_scale, float grad_scale, const float* grad_scale_dev, float* dw_cls,
                      float* db_cls, float* dw_box, float* db_box, float* dw_dim, float* db_dim, void* dz16, float* dz32,
                      int* nonfinite, cudaStream_t st) {
    if (R < 1 || K < 1 || n_classes < 1 || n_classes > 4) return SB_EINVAL;
    if (!(mask_scale > 0.f) || !isfinite(mask_scale)) return SB_EINVAL;
    if (!grad_scale_dev && (!(grad_scale > 0.f) || !isfinite(grad_scale))) return SB_EINVAL;
    const void* need[] = {d_cls_score, d_bbox_pred, d_dim_orien_pred, fc7, w_cls, w_box, w_dim, dw_cls, db_cls,
                          dw_box, db_box, dw_dim, db_dim, dz16, dz32};
    for (const void* q : need)
        if (!q) return SB_EINVAL;
    if (misaligned(dz16, 2)) return SB_EINVAL;
    if ((long long)R * K >= 0x7fffffffLL) return SB_EINVAL;
    BoxTailGrad a = {d_cls_score, d_bbox_pred, d_dim_orien_pred, w_cls, w_box, w_dim,
                     dw_cls, db_cls, dw_box, db_box, dw_dim, db_dim};
    const dim3 grid(R, sb_div_up(K, 256));
    if (grad_scale_dev)
        box_tail_dx_kernel<true><<<grid, 256, 0, st>>>(a, n_classes, fc7, K, mask_scale, 0.f, grad_scale_dev,
                                                       reinterpret_cast<__half*>(dz16), dz32, nonfinite);
    else
        box_tail_dx_kernel<false><<<grid, 256, 0, st>>>(a, n_classes, fc7, K, mask_scale, grad_scale, nullptr,
                                                        reinterpret_cast<__half*>(dz16), dz32, nonfinite);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    box_tail_dw_kernel<<<dim3(sb_div_up(K, 256), 12 * n_classes), 256, 0, st>>>(a, n_classes, R, fc7, K, nonfinite);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

int kpts_tail_backward(const void* up16, int R, int G, int C, const float* w, const float* d_kpts_pred,
                       const float* d_left_border_pred, const float* d_right_border_pred, float grad_scale,
                       const float* grad_scale_dev, void* dup16, float* dw, float* db, float* db_up, int* nonfinite,
                       void* workspace, size_t workspace_bytes, cudaStream_t st) {
    if (R < 1 || G < 2 || G > 64 || (G & 1) || C < 32 || C > 1024 || (C & 31)) return SB_EINVAL;
    if (!grad_scale_dev && (!(grad_scale > 0.f) || !isfinite(grad_scale))) return SB_EINVAL;
    const void* need[] = {up16, w, d_kpts_pred, d_left_border_pred, d_right_border_pred, dup16, dw, db, db_up,
                          workspace};
    for (const void* q : need)
        if (!q) return SB_EINVAL;
    if (misaligned(up16, 2) || misaligned(dup16, 2) || misaligned(workspace, 4)) return SB_EINVAL;
    if (workspace_bytes < (size_t)R * kpts_part_ld(C) * sizeof(float)) return SB_EINVAL;
    const int part_ld = (int)kpts_part_ld(C);
    float* part = reinterpret_cast<float*>(workspace);
    const size_t smem = 6 * G * sizeof(float);
    if (grad_scale_dev)
        kpts_tail_bwd_kernel<true><<<R, C, smem, st>>>(
            reinterpret_cast<const __half*>(up16), G, C, w, d_kpts_pred, d_left_border_pred, d_right_border_pred,
            0.f, grad_scale_dev, reinterpret_cast<__half*>(dup16), part, part_ld, nonfinite);
    else
        kpts_tail_bwd_kernel<false><<<R, C, smem, st>>>(
            reinterpret_cast<const __half*>(up16), G, C, w, d_kpts_pred, d_left_border_pred, d_right_border_pred,
            grad_scale, nullptr, reinterpret_cast<__half*>(dup16), part, part_ld, nonfinite);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    kpts_tail_bwd_reduce_kernel<<<sb_div_up(7 * C + 6, 256), 256, 0, st>>>(part, part_ld, R, C, G, dw, db, db_up,
                                                                            nonfinite);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

}  // namespace

extern "C" int sb_dropout_words(void* x, int x_is_half, long long n, const unsigned* words, double p,
                                sb_stream_t stream) {
    if (n < 0 || (x_is_half != 0 && x_is_half != 1) || !(p >= 0.0 && p < 1.0)) return SB_EINVAL;
    if (n > 0 && (!x || !words)) return SB_EINVAL;
    if (misaligned(x, x_is_half ? 2 : 4) || misaligned(words, 4)) return SB_EINVAL;
    if (n == 0) return SB_OK;
    const unsigned long long thr = (unsigned long long)ceil(p * 4294967296.0);   // word < p 2^32
    dropout_kernel<<<grid_for(n), 256, 0, sb_cs(stream)>>>(x, x_is_half, n, words, thr, (float)(1.0 / (1.0 - p)));
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" int sb_kpts_logits(const float* kpts_pred_all, int R, int G, float* kpts_pred, float* left_border_pred,
                              float* right_border_pred, sb_stream_t stream) {
    if (R < 0 || G < 1) return SB_EINVAL;
    if (R == 0) return SB_OK;
    if (!kpts_pred_all || !kpts_pred || !left_border_pred || !right_border_pred) return SB_EINVAL;
    const long long n = (long long)R * 6 * G;
    kpts_logits_kernel<<<sb_div_up(n, 256), 256, 0, sb_cs(stream)>>>(kpts_pred_all, n, G, kpts_pred, left_border_pred,
                                                                     right_border_pred);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" int sb_box_tail_backward(const float* d_cls_score, const float* d_bbox_pred, const float* d_dim_orien_pred,
                                    const float* fc7, int R, int K, int n_classes, const float* w_cls,
                                    const float* w_box, const float* w_dim, float mask_scale, float grad_scale,
                                    float* dw_cls, float* db_cls, float* dw_box, float* db_box, float* dw_dim,
                                    float* db_dim, void* dz16, float* dz32, int* nonfinite, sb_stream_t stream) {
    return box_tail_backward(d_cls_score, d_bbox_pred, d_dim_orien_pred, fc7, R, K, n_classes, w_cls, w_box, w_dim,
                             mask_scale, grad_scale, nullptr, dw_cls, db_cls, dw_box, db_box, dw_dim, db_dim, dz16,
                             dz32, nonfinite, sb_cs(stream));
}

extern "C" int sb_box_tail_backward_devscale(const float* d_cls_score, const float* d_bbox_pred,
                                             const float* d_dim_orien_pred, const float* fc7, int R, int K,
                                             int n_classes, const float* w_cls, const float* w_box, const float* w_dim,
                                             float mask_scale, const float* grad_scale, float* dw_cls, float* db_cls,
                                             float* dw_box, float* db_box, float* dw_dim, float* db_dim, void* dz16,
                                             float* dz32, int* nonfinite, sb_stream_t stream) {
    if (!grad_scale) return SB_EINVAL;
    return box_tail_backward(d_cls_score, d_bbox_pred, d_dim_orien_pred, fc7, R, K, n_classes, w_cls, w_box, w_dim,
                             mask_scale, 0.f, grad_scale, dw_cls, db_cls, dw_box, db_box, dw_dim, db_dim, dz16, dz32,
                             nonfinite, sb_cs(stream));
}

extern "C" size_t sb_kpts_tail_backward_workspace(int R, int C) {
    if (R < 1 || C < 1) return 0;
    return (size_t)R * kpts_part_ld(C) * sizeof(float);
}

extern "C" int sb_kpts_tail_backward(const void* up16, int R, int G, int C, const float* w, const float* d_kpts_pred,
                                     const float* d_left_border_pred, const float* d_right_border_pred,
                                     float grad_scale, void* dup16, float* dw, float* db, float* db_up, int* nonfinite,
                                     void* workspace, size_t workspace_bytes, sb_stream_t stream) {
    return kpts_tail_backward(up16, R, G, C, w, d_kpts_pred, d_left_border_pred, d_right_border_pred, grad_scale,
                              nullptr, dup16, dw, db, db_up, nonfinite, workspace, workspace_bytes, sb_cs(stream));
}

extern "C" int sb_kpts_tail_backward_devscale(const void* up16, int R, int G, int C, const float* w,
                                              const float* d_kpts_pred, const float* d_left_border_pred,
                                              const float* d_right_border_pred, const float* grad_scale, void* dup16,
                                              float* dw, float* db, float* db_up, int* nonfinite, void* workspace,
                                              size_t workspace_bytes, sb_stream_t stream) {
    if (!grad_scale) return SB_EINVAL;
    return kpts_tail_backward(up16, R, G, C, w, d_kpts_pred, d_left_border_pred, d_right_border_pred, 0.f, grad_scale,
                              dup16, dw, db, db_up, nonfinite, workspace, workspace_bytes, sb_cs(stream));
}

extern "C" int sb_permute3(const float* src, int d0, int d1, int d2, long long s0, long long s1, long long s2,
                           float* dst, sb_stream_t stream) {
    if (d0 < 1 || d1 < 1 || d2 < 1 || !src || !dst) return SB_EINVAL;
    const long long n = (long long)d0 * d1 * d2;
    // the strides must lay the three dimensions out densely in some order: sorted by stride, each equals the product
    // of the smaller ones' extents (then every destination element is written exactly once, inside [dst, dst + n))
    long long s[3] = {s0, s1, s2}, d[3] = {d0, d1, d2};
    for (int i = 0; i < 3; ++i)
        for (int j = i + 1; j < 3; ++j)
            if (s[j] < s[i] || (s[j] == s[i] && d[j] < d[i])) {
                long long t = s[i]; s[i] = s[j]; s[j] = t;
                t = d[i]; d[i] = d[j]; d[j] = t;
            }
    long long expect = 1;
    for (int i = 0; i < 3; ++i) {
        if (d[i] > 1 && s[i] != expect) return SB_EINVAL;
        if (s[i] < 0) return SB_EINVAL;
        expect *= d[i];
    }
    const uintptr_t a = reinterpret_cast<uintptr_t>(src), b = reinterpret_cast<uintptr_t>(dst);
    const uintptr_t bytes = (uintptr_t)n * sizeof(float);
    if (a < b + bytes && b < a + bytes) return SB_EINVAL;     // out of place only
    permute3_kernel<<<grid_for(n), 256, 0, sb_cs(stream)>>>(src, d1, d2, n, s0, s1, s2, dst);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}
