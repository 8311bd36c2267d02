// conv_simt.cu -- fp32 SIMT implicit-GEMM convolution on NHWC activations (sm_90a).
//
// Exact-fp32 companion of the tensor-core TF32 kernel (conv_tc.cu): same descriptor, same fused
// epilogue (frozen-BN scale/shift or bias, residual add, FPN bilinear upsample-add, ReLU,
// strided / channel-offset output addressing).  Used for layers the tensor-core kernel does
// not take (Cin % 32 != 0, stride 2) and as the fp32 yardstick the TF32 path is measured
// against.  Covers the nn.Conv2d / BatchNorm2d / ReLU / `out += residual` call sites of
// lib/model/stereo_rcnn/resnet.py:66-102,243-286 and lib/model/rpn/stereo_rpn.py:32-40.
//
// Tile: 128 output pixels x 64 output channels per CTA, K chunks of 16 input channels of
// one filter tap; 256 threads, 8x4 accumulators each; A/B staged through shared memory
// with 128-bit global loads, register-prefetched one chunk ahead.
#include "common.cuh"

namespace {

constexpr int BM = 128, BN = 64, BK = 16;

struct EpiCtx {
    float rh, rw;  // align_corners=True source scale for the FPN upsample
};

__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }

__global__ void __launch_bounds__(256)
conv_simt_kernel(sb_conv_desc d) {
    __shared__ __align__(16) float As[2][BK][BM + 4];
    __shared__ __align__(16) float Bs[2][BK][BN + 4];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;
    const long long M = (long long)d.N * d.Ho * d.Wo;
    const long long m0 = (long long)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;

    // A loader: 2 float4 per thread: pixel row (tid>>2) and (tid>>2)+64, k-quad (tid&3)
    const int a_kq = tid & 3;
    int a_hi[2], a_wi[2];
    long long a_base[2];
    bool a_ok[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        long long m = m0 + (tid >> 2) + 64 * i;
        a_ok[i] = m < M;
        long long mm = a_ok[i] ? m : 0;
        int wo = (int)(mm % d.Wo);
        long long t = mm / d.Wo;
        int ho = (int)(t % d.Ho);
        int n = (int)(t / d.Ho);
        a_hi[i] = ho * d.stride - d.pad;
        a_wi[i] = wo * d.stride - d.pad;
        a_base[i] = (long long)n * d.H * d.W;
    }
    // B loader: 1 float4 per thread: cout row (tid>>2), k-quad (tid&3)
    const int b_co = n0 + (tid >> 2);
    const bool b_ok = b_co < d.Cout;
    const long long wrow = (long long)d.kh * d.kw * d.Cin;

    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    const int cchunks = d.Cin / BK;
    const int nk = d.kh * d.kw * cchunks;
    float4 ra[2], rb;
    auto gload = [&](int kc) {
        const int tap = kc / cchunks, cc = kc - tap * cchunks;
        const int r = tap / d.kw, s = tap - r * d.kw;
        const int ci = cc * BK + a_kq * 4;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int hi = a_hi[i] + r, wi = a_wi[i] + s;
            const bool ok = a_ok[i] && hi >= 0 && hi < d.H && wi >= 0 && wi < d.W;
            ra[i] = ok ? ld4(d.in + (a_base[i] + (long long)hi * d.W + wi) * d.in_ld + ci)
                       : make_float4(0.f, 0.f, 0.f, 0.f);
            if (ok && d.in_biased) {
                ra[i].x = sb_unbias_tf32(ra[i].x); ra[i].y = sb_unbias_tf32(ra[i].y);
                ra[i].z = sb_unbias_tf32(ra[i].z); ra[i].w = sb_unbias_tf32(ra[i].w);
            }
        }
        rb = b_ok ? ld4(d.wgt + (long long)b_co * wrow + (long long)tap * d.Cin + ci)
                  : make_float4(0.f, 0.f, 0.f, 0.f);
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int m = (tid >> 2) + 64 * i;
            As[buf][a_kq * 4 + 0][m] = ra[i].x;
            As[buf][a_kq * 4 + 1][m] = ra[i].y;
            As[buf][a_kq * 4 + 2][m] = ra[i].z;
            As[buf][a_kq * 4 + 3][m] = ra[i].w;
        }
        const int n = tid >> 2;
        Bs[buf][a_kq * 4 + 0][n] = rb.x;
        Bs[buf][a_kq * 4 + 1][n] = rb.y;
        Bs[buf][a_kq * 4 + 2][n] = rb.z;
        Bs[buf][a_kq * 4 + 3][n] = rb.w;
    };

    gload(0);
    sstore(0);
    __syncthreads();
    for (int kc = 0; kc < nk; ++kc) {
        const int buf = kc & 1;
        if (kc + 1 < nk) gload(kc + 1);
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 8 + 4]);
            const float4 b = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        if (kc + 1 < nk) sstore(buf ^ 1);
        __syncthreads();
    }

    // ---- fused epilogue -------------------------------------------------------------
    const int c = n0 + tx * 4;
    if (c >= d.Cout) return;
    const bool vec = (c + 3 < d.Cout);
    float sc[4], sh[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const bool in = c + j < d.Cout;
        sc[j] = (d.scale && in) ? d.scale[c + j] : 1.f;
        sh[j] = (d.shift && in) ? d.shift[c + j] : 0.f;
    }
    float rh = 0.f, rw = 0.f;
    if (d.up_src) {
        rh = d.Ho > 1 ? __fdiv_rn((float)(d.UH - 1), (float)(d.Ho - 1)) : 0.f;
        rw = d.Wo > 1 ? __fdiv_rn((float)(d.UW - 1), (float)(d.Wo - 1)) : 0.f;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const long long m = m0 + ty * 8 + i;
        if (m >= M) break;
        const int wo = (int)(m % d.Wo);
        const long long t = m / d.Wo;
        const int ho = (int)(t % d.Ho);
        const int n = (int)(t / d.Ho);
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = __fadd_rn(__fmul_rn(acc[i][j], sc[j]), sh[j]);
        if (d.residual) {
            const float* r = d.residual + ((long long)(n * d.Ho + ho) * d.Wo + wo) * d.res_ld + c;
#pragma unroll
            for (int j = 0; j < 4; ++j) if (c + j < d.Cout) v[j] += d.res_biased ? sb_unbias_tf32(r[j]) : r[j];
        }
        if (d.up_src) {
            const float sy = __fmul_rn(rh, (float)ho), sx = __fmul_rn(rw, (float)wo);
            const int y1 = (int)sy, x1 = (int)sx;
            const int yp = y1 < d.UH - 1 ? 1 : 0, xp = x1 < d.UW - 1 ? 1 : 0;
            const float ly1 = sy - (float)y1, ly0 = 1.f - ly1, lx1 = sx - (float)x1, lx0 = 1.f - lx1;
            const float* u00 = d.up_src + (((long long)n * d.UH + y1) * d.UW + x1) * d.Cout + c;
            const float* u01 = u00 + (long long)xp * d.Cout;
            const float* u10 = u00 + (long long)yp * d.UW * d.Cout;
            const float* u11 = u10 + (long long)xp * d.Cout;
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (c + j < d.Cout)
                    v[j] += ly0 * (lx0 * u00[j] + lx1 * u01[j]) + ly1 * (lx0 * u10[j] + lx1 * u11[j]);
        }
        if (d.relu) {
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = fmaxf(v[j], 0.f);
        }
        if (d.out_mode) {
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = sb_store_mode(v[j], d.out_mode);
        }
        float* o = d.out + (long long)n * d.out_n_stride + (long long)ho * d.out_h_stride +
                   (long long)wo * d.out_w_stride + d.out_coff + c;
        if (vec && ((reinterpret_cast<uintptr_t>(o) & 15) == 0)) {
            *reinterpret_cast<float4*>(o) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
#pragma unroll
            for (int j = 0; j < 4; ++j) if (c + j < d.Cout) o[j] = v[j];
        }
    }
}

// stem: 7x7/2 pad 3, Cin = 3 (NCHW image) -> 64 ch NHWC, + BN + ReLU.  One thread = one output
// pixel x 16 channels; weights [64][7][7][3] staged in shared memory.
__global__ void __launch_bounds__(256)
stem_kernel(const float* __restrict__ im, int N, int H, int W, int Ho, int Wo,
            const float* __restrict__ wgt, const float* __restrict__ scale,
            const float* __restrict__ shift, float* __restrict__ out, int out_mode) {
    __shared__ float ws[147][64];   // [tap*3+ci][co]
    for (int e = threadIdx.x; e < 147 * 64; e += 256) {
        int co = e / 147, k = e % 147;
        ws[k][co] = wgt[e];
    }
    __syncthreads();
    const int cq = threadIdx.x & 3;          // 16-channel quarter
    const long long pix = (long long)blockIdx.x * 64 + (threadIdx.x >> 2);
    const long long M = (long long)N * Ho * Wo;
    if (pix >= M) return;
    const int wo = (int)(pix % Wo);
    const long long t = pix / Wo;
    const int ho = (int)(t % Ho), n = (int)(t / Ho);
    float acc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = 0.f;
    const float* base = im + (long long)n * 3 * H * W;
    for (int r = 0; r < 7; ++r) {
        const int hi = ho * 2 - 3 + r;
        if (hi < 0 || hi >= H) continue;
        for (int s = 0; s < 7; ++s) {
            const int wi = wo * 2 - 3 + s;
            if (wi < 0 || wi >= W) continue;
#pragma unroll
            for (int ci = 0; ci < 3; ++ci) {
                const float x = __ldg(base + ((long long)ci * H + hi) * W + wi);
                const float* wr = &ws[(r * 7 + s) * 3 + ci][cq * 16];
#pragma unroll
                for (int j = 0; j < 16; ++j) acc[j] = fmaf(x, wr[j], acc[j]);
            }
        }
    }
    float* o = out + pix * 64 + cq * 16;
#pragma unroll
    for (int j = 0; j < 16; j += 4) {
        float4 v;
        v.x = fmaxf(__fadd_rn(__fmul_rn(acc[j + 0], scale[cq * 16 + j + 0]), shift[cq * 16 + j + 0]), 0.f);
        v.y = fmaxf(__fadd_rn(__fmul_rn(acc[j + 1], scale[cq * 16 + j + 1]), shift[cq * 16 + j + 1]), 0.f);
        v.z = fmaxf(__fadd_rn(__fmul_rn(acc[j + 2], scale[cq * 16 + j + 2]), shift[cq * 16 + j + 2]), 0.f);
        v.w = fmaxf(__fadd_rn(__fmul_rn(acc[j + 3], scale[cq * 16 + j + 3]), shift[cq * 16 + j + 3]), 0.f);
        if (out_mode) {
            v.x = sb_store_mode(v.x, out_mode); v.y = sb_store_mode(v.y, out_mode);
            v.z = sb_store_mode(v.z, out_mode); v.w = sb_store_mode(v.w, out_mode);
        }
        *reinterpret_cast<float4*>(o + j) = v;
    }
}

// stem im2col: NCHW image -> rows of the 7x7/2 pad-3 patch matrix [M = N*Ho*Wo][160] with
// k = ci*49 + r*7 + s (the reference's own [Cout][Cin][kh][kw] weight order: 4 consecutive k are
// 4 consecutive input pixels of one row, i.e. one or two 32-byte sectors) for k < 147, zero up to 160 (a multiple of the 32-wide K tile of
// the tensor-core kernel).  One thread = one float4 (4 consecutive k) of one output pixel.
__global__ void __launch_bounds__(256)
stem_im2col_kernel(const float* __restrict__ im, int N, int H, int W, int Ho, int Wo, float4* __restrict__ out) {
    const long long total = (long long)N * Ho * Wo * 40;
    const long long e = (long long)blockIdx.x * 256 + threadIdx.x;
    if (e >= total) return;
    const int g = (int)(e % 40);
    long long t = e / 40;
    const int wo = (int)(t % Wo); t /= Wo;
    const int ho = (int)(t % Ho);
    const int n = (int)(t / Ho);
    const float* base = im + (long long)n * 3 * H * W;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int k = g * 4 + j;
        float x = 0.f;
        if (k < 147) {
            const int ci = k / 49, tap = k - ci * 49;
            const int r = tap / 7, s2 = tap - r * 7;
            const int hi = ho * 2 - 3 + r, wi = wo * 2 - 3 + s2;
            if (hi >= 0 && hi < H && wi >= 0 && wi < W)
                x = sb_round_tf32(__ldg(base + ((long long)ci * H + hi) * W + wi));   // RN, not the MMA's truncation
        }
        v[j] = x;
    }
    out[e] = make_float4(v[0], v[1], v[2], v[3]);
}

}  // namespace

extern "C" int sb_stem_im2col(const float* im_nchw, int N, int H, int W, float* out, sb_stream_t stream) {
    const int Ho = (H + 6 - 7) / 2 + 1, Wo = (W + 6 - 7) / 2 + 1;
    const long long total = (long long)N * Ho * Wo * 40;
    if (total <= 0) return SB_EINVAL;
    stem_im2col_kernel<<<sb_div_up(total, 256), 256, 0, sb_cs(stream)>>>(im_nchw, N, H, W, Ho, Wo, (float4*)out);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" int sb_conv2d_simt(const sb_conv_desc* d, sb_stream_t stream) {
    if (!d || !d->in || !d->wgt || !d->out) return SB_EINVAL;
    // fp32 operands and the fp32 output only: an fp16 descriptor would be read as fp32 (past the end of its
    // buffers) and its twin never written
    if (d->in_dtype != 0 || d->out16) return SB_EINVAL;
    if (d->Cin % BK != 0 || d->in_ld % 4 != 0 || d->in_ld < d->Cin) return SB_EINVAL;
    const long long M = (long long)d->N * d->Ho * d->Wo;
    if (M == 0) return SB_OK;
    dim3 grid(sb_div_up(M, BM), sb_div_up(d->Cout, BN));
    conv_simt_kernel<<<grid, 256, 0, sb_cs(stream)>>>(*d);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" int sb_stem_conv(const float* im_nchw, int N, int H, int W, const float* wgt, const float* scale,
                            const float* shift, float* out_nhwc, int out_mode, sb_stream_t stream) {
    const int Ho = (H + 6 - 7) / 2 + 1, Wo = (W + 6 - 7) / 2 + 1;
    const long long M = (long long)N * Ho * Wo;
    if (M <= 0) return SB_EINVAL;
    stem_kernel<<<sb_div_up(M, 64), 256, 0, sb_cs(stream)>>>(im_nchw, N, H, W, Ho, Wo, wgt, scale, shift, out_nhwc, out_mode);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}
