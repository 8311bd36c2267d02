// conv_tc.cu -- implicit-GEMM convolution on Hopper tensor cores (wgmma, sm_90a only).
//
// The dense contractions of the Stereo R-CNN forward -- every 1x1 / 3x3 convolution of the
// ResNet-101 trunk, FPN, RPN, the 25088->2048 box-head FC, the keypoint-head convs, the
// 2x2 deconv (as four 1x1s) and the 7x7 stem -- run through this one kernel:
//
//   D[M = output pixels, N = Cout] = sum over taps (r,s) and Cin chunks of
//        A[(pixel shifted by tap), Cin chunk] * W[Cout, tap, Cin chunk]^T
//
//   * operands are fp16 in HBM by default (in_dtype 1: NHWC activations, [Cout][kh][kw][Cin] weights, both rounded
//     to nearest once by their producer) and feed `wgmma ... .f16.f16`; the fp32 / tf32 mode (in_dtype 0, the
//     tensor core reads the top 19 bits) is kept for comparison.  Accumulation is fp32 in registers either way; the
//     exact-fp32 SIMT kernel (conv_simt.cu) is the yardstick.
//   * TMA moves every operand tile: weights through a 2-D map, activations through a 2-D map (1x1: pixels are rows
//     of a flat [M, Cin] matrix) or a 4-D [C, W, H, N] map (3x3: an 8x16 pixel patch per tile; the tap shift is a
//     coordinate offset and the hardware zero-fills the padding halo, so im2col never exists in memory).  128-byte
//     swizzle, 1024-byte aligned stages, one 128-byte row (64 fp16 / 32 fp32 = one K-step) per pixel per stage.
//     The stem variant builds its A tile in the kernel instead (patch gather warps, see below).
//   * warp-specialised persistent CTAs (one per SM): warps 0..7 are two consumer warpgroups -- each issues the
//     m64nNk16 (k8 for tf32) wgmma of 64 of the tile's 128 rows and owns their fp32 accumulators -- and warp 8 is
//     the TMA producer.  One mbarrier ring (full / empty) of stages sized so that nearly all shared memory holds
//     operands (4 stages of 48 KB for 256-wide tiles, 6 of 32 KB for 128-wide ones); the producer runs ahead into
//     the next tile while the consumers finish the epilogue of the current one.
//   * fused epilogue straight out of the accumulator registers: folded frozen-BN scale/shift or bias, residual add,
//     FPN bilinear (align_corners) upsample-add, ReLU, the TF32 store modes, fp32 and/or fp16 ("twin") stores with
//     arbitrary n/h/w strides and channel offset (RPN L|R concat, deconv scatter).
//   * programmatic dependent launch: the prologue (barrier init, descriptor prefetch) overlaps the previous
//     kernel's tail; dependents are released after the CTA's last operand loads are issued.
//   * optional per-CTA phase trace (sb_conv_trace) for tools/conv_trace.py.
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>

#include "common.cuh"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace {

constexpr int TW = 16, TH = 8;        // spatial patch of a 3x3 tile (TW*TH == BLOCK_M)
constexpr int kMaxCout = 2048;
constexpr int kConsumerWarps = 8;     // two warpgroups x 64 accumulator rows
constexpr int kProducerWarp = kConsumerWarps;
constexpr int kThreads = 32 * (kConsumerWarps + 1);
constexpr int kStemGatherWarps = 8;   // 2 threads per A-tile row: each builds 4 of the 8 16-byte groups of a K-step
constexpr int kStemThreads = kThreads + 32 * kStemGatherWarps;

struct TcParams {
    sb_conv_desc d;
    int patch;            // 0: flat [M,Cin] rows (1x1), 1: 8x16 spatial patches (3x3 / pad 1)
    int tiles_w, tiles_h; // patch mode
    int num_m_tiles, num_n_tiles;
    int kblocks_per_tap;  // Cin / BLOCK_K
    int num_k_blocks;     // taps * kblocks_per_tap
    long long M;
    int pdl_late;         // fire griddepcontrol.launch_dependents after the last operand loads instead of at entry
    unsigned long long* trace;   // optional per-CTA phase timestamps (sb_conv_trace), 16 words per CTA
    // STEM variant: the A operand is gathered from the NCHW fp32 image [N,3,sH,sW] (7x7 / stride 2 / pad 3 patches)
    const float* stem_im;
    int sH, sW;
    // MASK variant (dgrad of the backward pass): output element e is kept only where mask16[e] > 0 (the ReLU mask of
    // a saved forward tensor with the output's layout), after the residual add
    const __half* mask16;
};

__device__ __forceinline__ unsigned long long gtimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t) :: "memory");
    return t;
}
constexpr int kTraceWords = 16, kTraceCtas = 304;

constexpr size_t conv_smem(int block_n, int stages) {
    return (size_t)stages * (BLOCK_M * kRowBytes + block_n * kRowBytes) + 1024 + 2 * stages * 8;
}

template <int BLOCK_N, int kStages, bool HAS_RES, bool HAS_UP, bool IN16, bool STEM = false, bool MASK = false>
__global__ void __launch_bounds__(STEM ? kStemThreads : kThreads, 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
               const TcParams p) {
    static_assert(!STEM || (IN16 && !HAS_RES && !HAS_UP), "stem variant");
    static_assert(!MASK || (IN16 && !HAS_UP && !STEM), "mask variant");
    constexpr uint32_t kABytes = BLOCK_M * kRowBytes, kBBytes = BLOCK_N * kRowBytes;
    constexpr int BLOCK_K = IN16 ? 64 : 32;     // elements per K-step
    constexpr uint32_t kStageBytes = kABytes + kBBytes;
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + kStages * kStageBytes);
    uint64_t* empty = full + kStages;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const sb_conv_desc& d = p.d;
    unsigned long long* tr = p.trace ? p.trace + (size_t)blockIdx.x * kTraceWords : nullptr;
    if (tr && threadIdx.x == 0) {
        unsigned smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        tr[0] = gtimer(); tr[8] = clock64(); tr[6] = smid;
    }
    if (warp == kProducerWarp && lane == 0) {
        if (!STEM) prefetch_tmap(&map_a);
        prefetch_tmap(&map_b);
        // STEM: a stage is full when the weight tile has landed (1 expect_tx arrival) and the gather threads have
        // written their patch rows.  A stage is empty when every consumer warp's MMAs on it have completed.
        for (int i = 0; i < kStages; ++i) {
            mbar_init(&full[i], STEM ? 1 + 32 * kStemGatherWarps : 1);
            mbar_init(&empty[i], kConsumerWarps);
        }
        fence_barrier_init();
    }
    __syncthreads();
    // Programmatic dependent launch: everything above (barrier init, descriptor prefetch) overlapped the previous
    // kernel's tail.  Let the next kernel start its own prologue, then wait for the producers of our activations.
    if (!p.pdl_late) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (tr && threadIdx.x == 0) { tr[1] = gtimer(); tr[9] = clock64(); }

    const int num_tiles = p.num_m_tiles * p.num_n_tiles;

    if (warp == kProducerWarp) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int mt = tile / p.num_n_tiles, nt = tile - mt * p.num_n_tiles;
                int n_img = 0, h0 = 0, w0 = 0;
                if (p.patch) {
                    const int tw = mt % p.tiles_w;
                    const int t2 = mt / p.tiles_w;
                    h0 = (t2 % p.tiles_h) * TH;
                    n_img = t2 / p.tiles_h;
                    w0 = tw * TW;
                }
                for (int kb = 0; kb < p.num_k_blocks; ++kb) {
                    const int tap = kb / p.kblocks_per_tap;
                    const int c0 = (kb - tap * p.kblocks_per_tap) * BLOCK_K;
                    mbar_wait(&empty[stage], phase ^ 1);
                    uint8_t* sa = smem + stage * kStageBytes;
                    mbar_expect_tx(&full[stage], STEM ? kBBytes : kStageBytes);
                    if (!STEM) {
                        if (p.patch) {
                            const int r = tap / d.kw, s = tap - r * d.kw;
                            tma_load_4d(&map_a, &full[stage], sa, c0, w0 + s - d.pad, h0 + r - d.pad, n_img);
                        } else {
                            tma_load_2d(&map_a, &full[stage], sa, c0, mt * BLOCK_M);
                        }
                    }
                    tma_load_2d(&map_b, &full[stage], sa + kABytes, tap * d.Cin + c0, nt * BLOCK_N);
                    if (++stage == kStages) { stage = 0; phase ^= 1; }
                }
            }
            if (p.pdl_late) asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
            if (tr) { tr[3] = gtimer(); tr[11] = clock64(); }
        }
    } else if (STEM && warp > kProducerWarp) {
        // ===================== stem patch gather =====================
        // The 7x7 / stride-2 / pad-3 stem convolution (resnet.py:111) as an implicit GEMM: row gr of the A tile holds
        // the 147 taps (ci, r, s) of one output pixel, zero padded to 3 K-steps of 64 fp16, built straight from the
        // NCHW fp32 image into the 128-byte-swizzled stage (16-byte group j of row r at j ^ (r & 7)), so the patch
        // matrix is never written or read.  Image reads hit L1 / L2: every input pixel is used by ~12 taps of
        // neighbouring outputs.  Two threads build a row (4 groups each per K-step); all loads of a K-step are issued
        // before the first use and before the wait for the stage, so a thread exposes the load latency once per
        // K-step, not once per tap.
        constexpr int kPer = 8 / (kStemGatherWarps / 4);       // 16-byte groups per thread and K-step
        const int gt = threadIdx.x - kThreads;
        const int gr = gt & 127, gh = gt >> 7;
        int stage = 0;
        uint32_t phase = 0;
        const int H = p.sH, W = p.sW;
        const long long HW = (long long)H * W;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            const int mt = tile / p.num_n_tiles;
            const long long m = (long long)mt * BLOCK_M + gr;
            const bool valid = m < p.M;
            int n = 0, ho = 0, wo = 0;
            if (valid) {
                const int hw = d.Ho * d.Wo;
                n = (int)(m / hw);
                const int rem = (int)(m - (long long)n * hw);
                ho = rem / d.Wo;
                wo = rem - ho * d.Wo;
            }
            const int y0 = 2 * ho - 3, x0 = 2 * wo - 3;
            const float* img = p.stem_im + (long long)n * 3 * HW;
            const float* base = img + (long long)y0 * W + x0;
            const bool interior = valid && y0 >= 0 && y0 + 6 < H && x0 >= 0 && x0 + 6 < W;
#pragma unroll
            for (int kb = 0; kb < 3; ++kb) {
                float v[kPer * 8];
#pragma unroll
                for (int g = 0; g < kStemGatherWarps / 4; ++g) {          // g == gh: keeps every tap index a constant
                    if (g != gh) continue;
                    if (interior) {
#pragma unroll
                        for (int i = 0; i < kPer * 8; ++i) {
                            const int k = kb * 64 + g * kPer * 8 + i;
                            const int ci = k / 49, r = (k % 49) / 7, sx = k % 7;
                            v[i] = k < 147 ? __ldg(base + ci * HW + r * W + sx) : 0.f;
                        }
                    } else {
#pragma unroll
                        for (int i = 0; i < kPer * 8; ++i) {
                            const int k = kb * 64 + g * kPer * 8 + i;
                            const int ci = k / 49, r = (k % 49) / 7, sx = k % 7;
                            const int yy = y0 + r, xx = x0 + sx;
                            const bool ok = valid && k < 147 && yy >= 0 && yy < H && xx >= 0 && xx < W;
                            const int yc = min(max(yy, 0), H - 1), xc = min(max(xx, 0), W - 1);
                            const float t = __ldg(img + (k < 147 ? ci : 0) * HW + (long long)yc * W + xc);   // always in bounds
                            v[i] = ok ? t : 0.f;
                        }
                    }
                }
                mbar_wait(&empty[stage], phase ^ 1);
                const uint32_t row = smem_u32(smem + stage * kStageBytes) + gr * 128;
#pragma unroll
                for (int jj = 0; jj < kPer; ++jj) {
                    const int j = gh * kPer + jj;
                    uint32_t h[4];
#pragma unroll
                    for (int e2 = 0; e2 < 4; ++e2) {
                        __half2 pk = __floats2half2_rn(v[jj * 8 + 2 * e2], v[jj * 8 + 2 * e2 + 1]);
                        h[e2] = *reinterpret_cast<uint32_t*>(&pk);
                    }
                    sts128u(row + ((uint32_t)(j ^ (gr & 7)) << 4), make_uint4(h[0], h[1], h[2], h[3]));
                }
                fence_proxy_async();          // generic-proxy writes -> visible to the tensor core's async-proxy reads
                mbar_arrive(&full[stage]);
                if (++stage == kStages) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        // ===================== consumers: wgmma main loop + epilogue (warps 0..7) =====================
        // Warpgroup wg computes rows 64*wg .. 64*wg+63 of the tile against all BLOCK_N columns.  This thread holds
        // rows r_lo and r_lo + 8, columns 8*j + cq + {0,1} for j < BLOCK_N/8 (wgmma.cuh: fragment layout).
        const int wg = warp >> 2;
        const int r_lo = 64 * wg + 16 * (warp & 3) + (lane >> 2);
        const int cq = 2 * (lane & 3);
        constexpr int kAcc = BLOCK_N / 2;
        float acc[kAcc];
#pragma unroll
        for (int i = 0; i < kAcc; ++i) acc[i] = 0.f;
        float rh = 0.f, rw = 0.f;
        if (HAS_UP) {
            rh = d.Ho > 1 ? __fdiv_rn((float)(d.UH - 1), (float)(d.Ho - 1)) : 0.f;
            rw = d.Wo > 1 ? __fdiv_rn((float)(d.UW - 1), (float)(d.Wo - 1)) : 0.f;
        }
        const bool relu = d.relu != 0;
        const int out_mode = d.out_mode;
        const bool res_biased = d.res_biased != 0;
        int stage = 0;
        uint32_t phase = 0;
        for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
            const int mt = tile / p.num_n_tiles, nt = tile - mt * p.num_n_tiles;
            int prev = 0;
            for (int kb = 0; kb < p.num_k_blocks; ++kb) {
                mbar_wait(&full[stage], phase);
                if (tr && threadIdx.x == 0 && kb == 0 && tile == (int)blockIdx.x) { tr[2] = gtimer(); tr[10] = clock64(); }
                const uint32_t sa = smem_u32(smem + stage * kStageBytes);
                const uint64_t da = make_smem_desc(sa + wg * (kABytes / 2)), db = make_smem_desc(sa + kABytes);
#pragma unroll
                for (int i = 0; i < kAcc; ++i) reg_fence(acc[i]);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k)    // advance 32 bytes (16 fp16 / 8 tf32) inside the 128-byte swizzle row
                    Wgmma<BLOCK_N, IN16>::mma(acc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2), (kb | k) != 0);
                wgmma_commit();
#pragma unroll
                for (int i = 0; i < kAcc; ++i) reg_fence(acc[i]);
                // keep one K-step of MMAs in flight: the previous step's are complete, its stage may be refilled
                wgmma_wait<1>();
                if (kb > 0 && lane == 0) mbar_arrive(&empty[prev]);
                prev = stage;
                if (++stage == kStages) { stage = 0; phase ^= 1; }
            }
            wgmma_wait<0>();
#pragma unroll
            for (int i = 0; i < kAcc; ++i) reg_fence(acc[i]);
            if (lane == 0) mbar_arrive(&empty[prev]);

            // ---- epilogue: per row {output offset, residual row, upsample source + weights}, then per column pair
            long long ooff[2];
            bool valid[2];
            long long rrow[2];
            int uoff[2];
            float uly[2], ulx[2];
            bool by[2], bx[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = r_lo + 8 * h;
                int n_img, ho, wo;
                long long m = 0;
                if (p.patch) {
                    const int tw = mt % p.tiles_w;
                    const int t2 = mt / p.tiles_w;
                    ho = (t2 % p.tiles_h) * TH + row / TW;
                    wo = tw * TW + row % TW;
                    n_img = t2 / p.tiles_h;
                    valid[h] = ho < d.Ho && wo < d.Wo;
                } else {
                    m = (long long)mt * BLOCK_M + row;
                    valid[h] = m < p.M;
                    const unsigned mm = valid[h] ? (unsigned)m : 0u;      // M < 2^31 (checked on the host)
                    const unsigned hw = (unsigned)(d.Ho * d.Wo);
                    n_img = (int)(mm / hw);
                    const unsigned rem = mm - (unsigned)n_img * hw;
                    ho = (int)(rem / (unsigned)d.Wo);
                    wo = (int)(rem - (unsigned)ho * (unsigned)d.Wo);
                }
                ooff[h] = (long long)n_img * d.out_n_stride + (long long)ho * d.out_h_stride +
                          (long long)wo * d.out_w_stride + d.out_coff;
                rrow[h] = HAS_RES && valid[h] ? m * d.res_ld : 0;        // (residual: 1x1 convs, flat rows only)
                uoff[h] = 0; uly[h] = ulx[h] = 0.f; by[h] = bx[h] = false;
                if (HAS_UP && valid[h]) {
                    const float sy = __fmul_rn(rh, (float)ho), sx = __fmul_rn(rw, (float)wo);
                    const int y1 = (int)sy, x1 = (int)sx;
                    by[h] = y1 < d.UH - 1;
                    bx[h] = x1 < d.UW - 1;
                    uoff[h] = (int)((((long long)n_img * d.UH + y1) * d.UW + x1) * d.Cout);
                    uly[h] = sy - (float)y1;
                    ulx[h] = sx - (float)x1;
                }
            }
#pragma unroll
            for (int j = 0; j < BLOCK_N / 8; ++j) {
                const int c = nt * BLOCK_N + 8 * j + cq;      // Cout % 4 == 0: c < Cout implies c + 1 < Cout
                if (c >= d.Cout) break;
                const float2 sc = d.scale ? __ldg(reinterpret_cast<const float2*>(d.scale + c)) : make_float2(1.f, 1.f);
                const float2 sh = d.shift ? __ldg(reinterpret_cast<const float2*>(d.shift + c)) : make_float2(0.f, 0.f);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    if (!valid[h]) continue;
                    float x0 = fmaf(acc[4 * j + 2 * h], sc.x, sh.x);
                    float x1 = fmaf(acc[4 * j + 2 * h + 1], sc.y, sh.y);
                    if (HAS_RES) {
                        float2 r = __ldg(reinterpret_cast<const float2*>(d.residual + rrow[h] + c));
                        if (res_biased) { r.x = sb_unbias_tf32(r.x); r.y = sb_unbias_tf32(r.y); }
                        x0 += r.x; x1 += r.y;
                    }
                    if (HAS_UP) {
                        const float* u00 = d.up_src + uoff[h] + c;
                        const long long dx = bx[h] ? d.Cout : 0;
                        const long long dy = by[h] ? (long long)d.UW * d.Cout : 0;
                        const float2 a = __ldg(reinterpret_cast<const float2*>(u00));
                        const float2 bq = __ldg(reinterpret_cast<const float2*>(u00 + dx));
                        const float2 g = __ldg(reinterpret_cast<const float2*>(u00 + dy));
                        const float2 hh = __ldg(reinterpret_cast<const float2*>(u00 + dy + dx));
                        const float ly1 = uly[h], ly0 = 1.f - ly1, lx1 = ulx[h], lx0 = 1.f - lx1;
                        x0 += ly0 * (lx0 * a.x + lx1 * bq.x) + ly1 * (lx0 * g.x + lx1 * hh.x);
                        x1 += ly0 * (lx0 * a.y + lx1 * bq.y) + ly1 * (lx0 * g.y + lx1 * hh.y);
                    }
                    if (MASK) {
                        const __half2 mk = *reinterpret_cast<const __half2*>(p.mask16 + ooff[h] + c);
                        if (!(__low2float(mk) > 0.f)) x0 = 0.f;
                        if (!(__high2float(mk) > 0.f)) x1 = 0.f;
                    }
                    if (relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
                    if (out_mode == 1) { x0 = sb_round_tf32(x0); x1 = sb_round_tf32(x1); }
                    else if (out_mode == 2) { x0 = sb_bias_tf32(x0); x1 = sb_bias_tf32(x1); }
                    if (d.out) *reinterpret_cast<float2*>(d.out + ooff[h] + c) = make_float2(x0, x1);
                    if (d.out16) {   // fp16 twin (round to nearest) for the next tensor-core consumer
                        if (out_mode == 2) { x0 = sb_unbias_tf32(x0); x1 = sb_unbias_tf32(x1); }
                        *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(d.out16) + ooff[h] + c) =
                            __floats2half2_rn(x0, x1);
                    }
                }
            }
            if (tr && threadIdx.x == 0 && tile == (int)blockIdx.x) { tr[4] = gtimer(); tr[12] = clock64(); }
        }
    }

    __syncthreads();
    if (tr && threadIdx.x == 0) { tr[5] = gtimer(); tr[13] = clock64(); }
}

// ------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) != cudaSuccess ||
            qres != cudaDriverEntryPointSuccess)
            return nullptr;
        fn = (EncodeTiledFn)p;
    }
    return fn;
}

bool make_map(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
              const cuuint32_t* box, bool f16) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = enc(m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void*>(base), dims,
                     strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

// Tile-width choice.  Per SM and clock an H100 retires ~1024 dense fp16 MACs and ingests ~64 B from L2, so a
// 64-element K-step of a 128-row tile costs max(MMA cycles, bytes / 64):
//   BN=128: max(1024 * 128 * 64 / 1024 / 8, (16+16) KB / 64) = 512 cycles    BN=256: max(1024, (16+32) KB / 64) = 1024
// and the persistent grid runs ceil(tiles/SMs) waves.  Pick the cheaper of the two for Cout >= 256 (ties: 256, half
// the A-tile reloads).
int pick_block_n(int cout, long long m_tiles, int num_sms) {
    if (cout <= 32) return 32;
    if (cout <= 64) return 64;
    if (cout < 256) return 128;
    const long long t128 = m_tiles * ((cout + 127) / 128), t256 = m_tiles * ((cout + 255) / 256);
    const long long c128 = ((t128 + num_sms - 1) / num_sms) * 512, c256 = ((t256 + num_sms - 1) / num_sms) * 1024;
    return c256 <= c128 ? 256 : 128;
}

template <int BN, int ST, bool RES, bool UP, bool IN16, bool STEM = false, bool MASK = false>
int launch_t(const CUtensorMap& ma, const CUtensorMap& mb, const TcParams& p, cudaStream_t st) {
    constexpr size_t smem = conv_smem(BN, ST);
    static_assert(smem <= 227 * 1024, "smem budget");
    auto kern = conv_tc_kernel<BN, ST, RES, UP, IN16, STEM, MASK>;
    static bool attr_done[kSbMaxDevices] = {false};
    bool& attr = attr_done[sb_cur_device()];
    if (!attr) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
        attr = true;
    }
    const int tiles = p.num_m_tiles * p.num_n_tiles;
    int slots = sb_num_sms();
    if (p.d.max_ctas > 0 && p.d.max_ctas < slots) slots = p.d.max_ctas;
    const int grid = tiles < slots ? tiles : slots;
    static const bool use_pdl = getenv("SB_NO_PDL") == nullptr;
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(STEM ? kStemThreads : kThreads);
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attrs[1];
    attrs[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attrs[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attrs;
    cfg.numAttrs = use_pdl ? 1 : 0;
    cudaError_t le = cudaLaunchKernelEx(&cfg, kern, ma, mb, p);
    SB_LAUNCHED();
    if (le != cudaSuccess) return (int)le;
    SB_CHECK_LAUNCH();
    return SB_OK;
}

template <int BN, int ST>
int launch(const CUtensorMap& ma, const CUtensorMap& mb, const TcParams& p, cudaStream_t st) {
    const bool res = p.d.residual != nullptr, up = p.d.up_src != nullptr;   // never both (supported())
    if (p.mask16)       // dgrad: fp16 operands, never an upsample source (sb_conv2d_tc_dgrad)
        return res ? launch_t<BN, ST, true, false, true, false, true>(ma, mb, p, st)
                   : launch_t<BN, ST, false, false, true, false, true>(ma, mb, p, st);
    if (p.d.in_dtype == 1) {
        if (up) return launch_t<BN, ST, false, true, true>(ma, mb, p, st);
        return res ? launch_t<BN, ST, true, false, true>(ma, mb, p, st) : launch_t<BN, ST, false, false, true>(ma, mb, p, st);
    }
    if (up) return launch_t<BN, ST, false, true, false>(ma, mb, p, st);
    return res ? launch_t<BN, ST, true, false, false>(ma, mb, p, st) : launch_t<BN, ST, false, false, false>(ma, mb, p, st);
}

}  // namespace

extern "C" int sb_conv2d_tc_supported(const sb_conv_desc* d) {
    if (!d || !d->in || !d->wgt) return 0;
    const int bk = d->in_dtype == 1 ? 64 : 32;
    if (d->in_dtype != 0 && d->in_dtype != 1) return 0;
    if (d->stride != 1 || d->Cin % bk != 0 || d->in_ld % (d->in_dtype == 1 ? 8 : 4) != 0) return 0;
    if (!d->out && !d->out16) return 0;
    const bool k1 = d->kh == 1 && d->kw == 1 && d->pad == 0;
    const bool k3 = d->kh == 3 && d->kw == 3 && d->pad == 1;
    if (!k1 && !k3) return 0;
    if (d->Cout > kMaxCout || (d->Cout & 3)) return 0;
    if (d->residual && (d->up_src || !k1)) return 0;      // the residual epilogue assumes flat (1x1) rows
    if (d->up_src && (long long)d->N * d->UH * d->UW * d->Cout >= 0x7fffffffLL) return 0;
    if ((long long)d->N * d->out_n_stride + d->out_coff >= 0x7fffffffLL) return 0;
    if ((reinterpret_cast<uintptr_t>(d->in) & 15) || (reinterpret_cast<uintptr_t>(d->wgt) & 15) ||
        (reinterpret_cast<uintptr_t>(d->out) & 15) || (reinterpret_cast<uintptr_t>(d->out16) & 7))
        return 0;
    if ((d->out_coff & 3) || (d->out_n_stride & 3) || (d->out_h_stride & 3) || (d->out_w_stride & 3)) return 0;
    if (d->residual && ((d->res_ld & 3) || (reinterpret_cast<uintptr_t>(d->residual) & 15))) return 0;
    if ((reinterpret_cast<uintptr_t>(d->scale) & 15) || (reinterpret_cast<uintptr_t>(d->shift) & 15)) return 0;
    if (d->up_src && ((d->Cout & 3) || (reinterpret_cast<uintptr_t>(d->up_src) & 15))) return 0;
    if (d->Ho != d->H || d->Wo != d->W) return 0;
    if ((long long)d->N * d->Ho * d->Wo >= 0x7fffffffLL) return 0;
    return 1;
}

// ---- optional phase trace (tools/conv_trace.py): 16 words per CTA, kTraceCtas CTAs per launch
namespace {
unsigned long long* g_trace = nullptr;
int g_trace_cap = 0, g_trace_n = 0;
struct TraceInfo { int v[12]; };
TraceInfo g_trace_info[4096];
}  // namespace

extern "C" size_t sb_conv_trace_bytes(int max_launches) {
    return (size_t)max_launches * kTraceCtas * kTraceWords * sizeof(unsigned long long);
}
extern "C" int sb_conv_trace(void* buf, int max_launches) {
    if (max_launches > 4096) return SB_EINVAL;
    g_trace = (unsigned long long*)buf;
    g_trace_cap = buf ? max_launches : 0;
    g_trace_n = 0;
    return SB_OK;
}
extern "C" int sb_conv_trace_info(int id, int* out12) {
    if (id < 0 || id >= g_trace_n) return SB_EINVAL;
    for (int i = 0; i < 12; ++i) out12[i] = g_trace_info[id].v[i];
    return SB_OK;
}
extern "C" int sb_conv_trace_count(void) { return g_trace_n; }

namespace {
int conv2d_tc(const sb_conv_desc* d, const __half* mask16, sb_stream_t stream) {
    if (!sb_conv2d_tc_supported(d)) return SB_EINVAL;
    TcParams p;
    p.d = *d;
    p.mask16 = mask16;
    // default: release the dependent launch once this CTA's last operand loads are issued -- an early release lets
    // the next kernel's CTAs sit in griddepcontrol.wait on SMs the other stream's chain could be using
    static const bool pdl_late = getenv("SB_PDL_LATE") == nullptr || atoi(getenv("SB_PDL_LATE")) != 0;
    p.pdl_late = pdl_late ? 1 : 0;
    p.trace = nullptr;
    p.stem_im = nullptr;
    p.sH = p.sW = 0;
    // spatial 8x16 tiles for 3x3 convs, and for the FPN laterals so that the bilinear upsample taps of a tile
    // (5x9 source pixels) stay in L1 instead of being re-fetched from L2 for every output row
    p.patch = (d->kh == 3 || d->up_src) ? 1 : 0;
    p.M = (long long)d->N * d->Ho * d->Wo;
    if (p.M == 0) return SB_OK;
    const bool f16 = d->in_dtype == 1;
    const int BLOCK_K = f16 ? 64 : 32;
    const int esz = f16 ? 2 : 4;
    p.kblocks_per_tap = d->Cin / BLOCK_K;
    p.num_k_blocks = d->kh * d->kw * p.kblocks_per_tap;
    p.tiles_w = (d->W + TW - 1) / TW;
    p.tiles_h = (d->H + TH - 1) / TH;
    p.num_m_tiles = p.patch ? d->N * p.tiles_h * p.tiles_w : (int)((p.M + BLOCK_M - 1) / BLOCK_M);
    int BN = pick_block_n(d->Cout, p.num_m_tiles, sb_num_sms());
    if (d->residual && BN == 256) BN = 128;   // residual layers are HBM-bound: the narrower tile keeps more CTAs busy
    if (const char* e = getenv("SB_TC_BLOCK_N")) { int v = atoi(e); if ((v == 128 || v == 256) && d->Cout >= 256) BN = v; }
    p.num_n_tiles = (d->Cout + BN - 1) / BN;
    if (g_trace && g_trace_n < g_trace_cap) {
        const int id = g_trace_n++;
        p.trace = g_trace + (size_t)id * kTraceCtas * kTraceWords;
        int* v = g_trace_info[id].v;
        v[0] = d->Cin; v[1] = d->Cout; v[2] = d->kh; v[3] = (int)p.M; v[4] = BN; v[5] = p.num_m_tiles * p.num_n_tiles;
        v[6] = p.num_k_blocks; v[7] = d->residual ? 1 : 0; v[8] = d->up_src ? 1 : 0; v[9] = 0;
        v[10] = d->max_ctas; v[11] = d->N;
    }
    CUtensorMap ma, mb;
    if (p.patch) {
        cuuint64_t dims[4] = {(cuuint64_t)d->Cin, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)d->N};
        cuuint64_t strides[3] = {(cuuint64_t)d->in_ld * esz, (cuuint64_t)d->W * d->in_ld * esz,
                                 (cuuint64_t)d->H * d->W * d->in_ld * esz};
        cuuint32_t box[4] = {(cuuint32_t)BLOCK_K, TW, TH, 1};
        if (!make_map(&ma, d->in, 4, dims, strides, box, f16)) return SB_EINVAL;
    } else {
        // a row may be SHORTER than Cin (in_ld < Cin: the stem's 152-wide patch rows under a 192-wide zero-padded weight):
        // the map's inner extent is then the row length and TMA zero-fills the rest of the last K-step
        cuuint64_t dims[2] = {(cuuint64_t)(d->in_ld < d->Cin ? d->in_ld : d->Cin), (cuuint64_t)p.M};
        cuuint64_t strides[1] = {(cuuint64_t)d->in_ld * esz};
        cuuint32_t box[2] = {(cuuint32_t)BLOCK_K, BLOCK_M};
        if (!make_map(&ma, d->in, 2, dims, strides, box, f16)) return SB_EINVAL;
    }
    {
        const cuuint64_t ktot = (cuuint64_t)d->kh * d->kw * d->Cin;
        cuuint64_t dims[2] = {ktot, (cuuint64_t)d->Cout};
        cuuint64_t strides[1] = {ktot * esz};
        cuuint32_t box[2] = {(cuuint32_t)BLOCK_K, (cuuint32_t)BN};
        if (!make_map(&mb, d->wgt, 2, dims, strides, box, f16)) return SB_EINVAL;
    }
    cudaStream_t st = sb_cs(stream);
    switch (BN) {
        case 32: return launch<32, 9>(ma, mb, p, st);
        case 64: return launch<64, 8>(ma, mb, p, st);
        case 256: return launch<256, 4>(ma, mb, p, st);
        default: return launch<128, 6>(ma, mb, p, st);
    }
}
}  // namespace

extern "C" int sb_conv2d_tc(const sb_conv_desc* d, sb_stream_t stream) { return conv2d_tc(d, nullptr, stream); }

// Data gradient of a convolution as the forward implicit GEMM on transposed weights (the caller packs them
// [Cin][kh][kw][Cout], taps flipped, frozen-BN scale folded in), with the ReLU mask of a saved tensor applied after
// the optional residual add.  mask16 has the output's element layout (out strides and channel offset).
extern "C" int sb_conv2d_tc_dgrad(const sb_conv_desc* d, const void* mask16, sb_stream_t stream) {
    if (!d || d->in_dtype != 1 || d->up_src || d->relu || d->out_mode != 0) return SB_EINVAL;
    if (reinterpret_cast<uintptr_t>(mask16) & 3) return SB_EINVAL;
    if (!mask16) return conv2d_tc(d, nullptr, stream);
    return conv2d_tc(d, reinterpret_cast<const __half*>(mask16), stream);
}

// The stem (resnet.py:111-112: Conv2d(3, 64, 7, stride 2, pad 3) + frozen BN + ReLU) as an implicit GEMM on the tensor
// cores, patches gathered inside the kernel (conv_tc_kernel<.., STEM>): image NCHW fp32 [N,3,H,W], weights fp16
// [64][192] in (ci, r, s) order zero padded from 147, out NHWC fp16 [N,Ho,Wo,64].
extern "C" int sb_stem_conv_tc(const float* im_nchw, int N, int H, int W, const void* wgt16, const float* scale,
                               const float* shift, void* out16, sb_stream_t stream) {
    if (!im_nchw || !wgt16 || !out16 || N < 1 || H < 7 || W < 7) return SB_EINVAL;
    if ((reinterpret_cast<uintptr_t>(wgt16) & 15) || (reinterpret_cast<uintptr_t>(out16) & 15) ||
        (reinterpret_cast<uintptr_t>(scale) & 15) || (reinterpret_cast<uintptr_t>(shift) & 15))
        return SB_EINVAL;
    const int Ho = (H + 6 - 7) / 2 + 1, Wo = (W + 6 - 7) / 2 + 1;
    TcParams p = {};
    sb_conv_desc& d = p.d;
    d.wgt = reinterpret_cast<const float*>(wgt16);
    d.scale = scale; d.shift = shift;
    d.out16 = out16;
    d.N = N; d.H = H; d.W = W; d.Cin = 192; d.Cout = 64; d.kh = d.kw = 1; d.stride = 2; d.pad = 3;
    d.Ho = Ho; d.Wo = Wo; d.relu = 1; d.in_dtype = 1;
    d.out_w_stride = 64; d.out_h_stride = (long long)Wo * 64; d.out_n_stride = (long long)Ho * Wo * 64;
    p.M = (long long)N * Ho * Wo;
    if (p.M >= 0x7fffffffLL || p.M * 64 >= 0x7fffffffLL) return SB_EINVAL;
    p.num_m_tiles = (int)((p.M + BLOCK_M - 1) / BLOCK_M); p.num_n_tiles = 1;
    p.kblocks_per_tap = 3; p.num_k_blocks = 3;
    static const bool pdl_late = getenv("SB_PDL_LATE") == nullptr || atoi(getenv("SB_PDL_LATE")) != 0;
    p.pdl_late = pdl_late ? 1 : 0;
    p.stem_im = im_nchw; p.sH = H; p.sW = W;
    p.mask16 = nullptr;
    CUtensorMap mb;
    {
        cuuint64_t dims[2] = {192, 64};
        cuuint64_t strides[1] = {192 * 2};
        cuuint32_t box[2] = {64, 64};
        if (!make_map(&mb, wgt16, 2, dims, strides, box, true)) return SB_EINVAL;
    }
    return launch_t<64, 8, false, false, true, true>(mb, mb, p, sb_cs(stream));
}
