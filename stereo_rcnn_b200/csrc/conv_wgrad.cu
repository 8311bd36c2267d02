// conv_wgrad.cu -- backward-pass pieces of the trunk + FPN that are not a forward-shaped convolution (sm_90a only).
//
//   * sb_conv_wgrad: weight gradient of a 1x1 / 3x3 (pad 1, stride 1) convolution on the tensor cores,
//       dW[Cout, tap, Cin] = sum over pixels p of dY[p, Cout] * X[p + tap, Cin]
//     K is the pixel dimension, so both fp16 NHWC operands are MN-major with respect to K.  TMA moves 64-pixel x
//     64-channel boxes (128-byte swizzle) and wgmma reads them through transposed-operand descriptors.  1x1 convs
//     use flat [C, M] maps.  3x3 convs use [C, W, H, N] maps: a K-block is 64 pixels of one image row, the tap
//     shift is a coordinate offset and TMA zero-fills the halo (and the dY pixels past the row end).
//     The output has few tiles (a 256->256 3x3 conv has 2 x 9 x 2 of 128 x 128), so K is split over pixel ranges.
//     Every split writes its fp32 partial tile.  A second pass sums the partials in a fixed order, applies the
//     folded frozen-BN scale s[cout], divides out the gradient scale and writes the reference layout
//     [Cout][Cin][kh][kw].  Bias gradients are column sums of the fp32 dY, also two-level in a fixed order.
//     No float atomics: results are bit-identical run to run.  A non-finite gradient sets *nonfinite = 1.
//   * sb_conv_wgrad_acc: the same GEMM on strided operands (dY may be a channel slice of a wider tensor), with the
//     results optionally added to the destination in stream order -- a sum over several convs that share one weight
//     (the RPN conv over five levels and two images) stays bit-identical run to run -- and the rows of dW / db split
//     over two destinations (the fused RPN head holds the reference's two 1x1 convs).
//   * sb_fpn_grad_combine: the gradient of one FPN level,
//       dP = scale * dP_in + up^T(dT) + scatter2(scale * dP6)
//     where up^T is the transpose of the align_corners bilinear upsample of stereo_rcnn.py:91-108 (a gather over the
//     fine pixels that read each coarse pixel, not atomics) and scatter2 the backward of P6 = P5[::2, ::2].
#include <cuda.h>
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"
#include "tc_ptx.cuh"

namespace {

constexpr int kWgBM = 128, kWgBN = 128, kWgBK = 64;   // Cout x Cin tile, pixels per K-block
constexpr int kWgStages = 5;
constexpr int kWgThreads = 32 * 9;                     // two consumer warpgroups + one TMA producer warp
constexpr uint32_t kBox = 64 * 128;                    // one 64-pixel x 64-channel fp16 box
constexpr uint32_t kWgStageBytes = 4 * kBox;           // dY: 2 boxes (128 Cout), X: 2 boxes (128 Cin)
constexpr size_t kWgSmem = (size_t)kWgStages * kWgStageBytes + 1024 + 2 * kWgStages * 8;
constexpr int kBiasChunks = 256;

// MN-major, 128-byte swizzle descriptor of one 64-element-wide atom column: rows are K (one 128-byte row per pixel),
// 8-row groups 1024 bytes apart.  An instruction reads at most one atom along M / N (m64, n64), so the leading-byte
// offset (atom stride along M / N) is never used; both offset fields hold the 8-row group stride.
__device__ __forceinline__ uint64_t make_smem_desc_mn(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFF) >> 4);
    d |= (uint64_t)(1024 >> 4) << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;
    return d;
}

// D[64 x 64] += A[64 x 16] * B[64 x 16]^T with both operands MN-major (imm-trans-a = imm-trans-b = 1, fp16 only)
__device__ __forceinline__ void wgmma_n64_tt(float* d, uint64_t da, uint64_t db, uint32_t accumulate) {
    asm volatile(
        "{\n.reg .pred p;\nsetp.ne.b32 p, %34, 0;\n"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 1, 1;\n}\n"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(da), "l"(db), "r"(accumulate));
}

struct WgParams {
    int patch;                 // 0: flat [C, M] maps (1x1), 1: [C, W, H, N] maps (3x3, pad 1)
    int N, H, W, k;            // k = kernel size (1 or 3)
    int wchunks;               // patch: 64-pixel chunks per image row
    int num_kb;                // K-blocks in total
    int kb_per_split, splits;
    int m_tiles, n_tiles, tiles;
    float* part;               // [splits][tiles][128][128] fp32 partial tiles
};

__global__ void __launch_bounds__(kWgThreads, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap map_dy, const __grid_constant__ CUtensorMap map_x,
                  const WgParams p) {
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint64_t* full = reinterpret_cast<uint64_t*>(smem + kWgStages * kWgStageBytes);
    uint64_t* empty = full + kWgStages;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    const int tile = blockIdx.x % p.tiles, split = blockIdx.x / p.tiles;
    // tile = (mt * taps + tap) * n_tiles + nt
    const int nt = tile % p.n_tiles, t2 = tile / p.n_tiles;
    const int taps = p.k * p.k;
    const int tap = t2 % taps, mt = t2 / taps;
    const int kb0 = split * p.kb_per_split;
    const int kb1 = min(p.num_kb, kb0 + p.kb_per_split);

    if (warp == 8 && lane == 0) {
        prefetch_tmap(&map_dy);
        prefetch_tmap(&map_x);
        for (int i = 0; i < kWgStages; ++i) {
            mbar_init(&full[i], 1);
            mbar_init(&empty[i], 8);
        }
        fence_barrier_init();
    }
    __syncthreads();
    asm volatile("griddepcontrol.wait;" ::: "memory");

    if (warp == 8) {
        if (lane == 0) {
            const int r = tap / p.k, s = tap - r * p.k;
            int stage = 0;
            uint32_t phase = 0;
            for (int kb = kb0; kb < kb1; ++kb) {
                mbar_wait(&empty[stage], phase ^ 1);
                uint8_t* sa = smem + stage * kWgStageBytes;
                mbar_expect_tx(&full[stage], kWgStageBytes);
                if (p.patch) {
                    const int wc = kb % p.wchunks, rowi = kb / p.wchunks;
                    const int h = rowi % p.H, n = rowi / p.H, w0 = wc * kWgBK;
                    for (int j = 0; j < 2; ++j) {
                        tma_load_4d(&map_dy, &full[stage], sa + j * kBox, mt * kWgBM + 64 * j, w0, h, n);
                        tma_load_4d(&map_x, &full[stage], sa + (2 + j) * kBox, nt * kWgBN + 64 * j, w0 + s - 1,
                                    h + r - 1, n);
                    }
                } else {
                    for (int j = 0; j < 2; ++j) {
                        tma_load_2d(&map_dy, &full[stage], sa + j * kBox, mt * kWgBM + 64 * j, kb * kWgBK);
                        tma_load_2d(&map_x, &full[stage], sa + (2 + j) * kBox, nt * kWgBN + 64 * j, kb * kWgBK);
                    }
                }
                if (++stage == kWgStages) { stage = 0; phase ^= 1; }
            }
        }
    } else {
        // warpgroup wg owns Cout rows 64*wg .. 64*wg+63 against both 64-wide Cin halves (acc[0..31], acc[32..63])
        const int wg = warp >> 2;
        float acc[64];
#pragma unroll
        for (int i = 0; i < 64; ++i) acc[i] = 0.f;
        int stage = 0, prev = 0;
        uint32_t phase = 0;
        for (int kb = kb0; kb < kb1; ++kb) {
            mbar_wait(&full[stage], phase);
            const uint32_t sa = smem_u32(smem + stage * kWgStageBytes);
            const uint64_t da = make_smem_desc_mn(sa + wg * kBox);
            const uint64_t db0 = make_smem_desc_mn(sa + 2 * kBox), db1 = make_smem_desc_mn(sa + 3 * kBox);
#pragma unroll
            for (int i = 0; i < 64; ++i) reg_fence(acc[i]);
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < 4; ++k) {    // 16 pixels = 16 rows of 128 bytes per MMA
                const uint64_t o = (uint64_t)(k * 2048 >> 4);
                wgmma_n64_tt(acc, da + o, db0 + o, (kb > kb0 || k > 0) ? 1u : 0u);
                wgmma_n64_tt(acc + 32, da + o, db1 + o, (kb > kb0 || k > 0) ? 1u : 0u);
            }
            wgmma_commit();
#pragma unroll
            for (int i = 0; i < 64; ++i) reg_fence(acc[i]);
            wgmma_wait<1>();
            if (kb > kb0 && lane == 0) mbar_arrive(&empty[prev]);
            prev = stage;
            if (++stage == kWgStages) { stage = 0; phase ^= 1; }
        }
        wgmma_wait<0>();
#pragma unroll
        for (int i = 0; i < 64; ++i) reg_fence(acc[i]);
        // fragment: acc[32*c + 4*j + 2*h + e] is row 64*wg + 16*(warp&3) + lane/4 + 8*h, column 64*c + 8*j + 2*(lane%4) + e
        float* dst = p.part + ((size_t)split * p.tiles + tile) * (kWgBM * kWgBN);
        const int r_lo = 64 * wg + 16 * (warp & 3) + (lane >> 2), cq = 2 * (lane & 3);
#pragma unroll
        for (int c = 0; c < 2; ++c)
#pragma unroll
            for (int j = 0; j < 8; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    *reinterpret_cast<float2*>(dst + (r_lo + 8 * h) * kWgBN + 64 * c + 8 * j + cq) =
                        make_float2(acc[32 * c + 4 * j + 2 * h], acc[32 * c + 4 * j + 2 * h + 1]);
    }
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}

// second pass: dW[co][ci][r][s] = s[co] / grad_scale * sum over splits (ascending) of the partial tiles.  Rows
// co < o.split go to o.dw, rows o.split <= co < o.rows to o.dw_hi (row co - split), rows past o.rows are dropped;
// o.accumulate adds the result to what the destination holds.
struct WgOut {
    float *dw, *dw_hi, *db, *db_hi;
    int rows, split, accumulate;
};

__device__ __forceinline__ void store_row_value(float* lo, float* hi, int split, int co, size_t row_elems, size_t i,
                                                float v, int accumulate, int* nonfinite) {
    float* dst = co < split ? lo + (size_t)co * row_elems + i : hi + (size_t)(co - split) * row_elems + i;
    if (accumulate) v = *dst + v;
    *dst = v;
    if (nonfinite && !isfinite(v)) *nonfinite = 1;
}

// DEV_SCALE: the gradient scale is read from grad_scale (device, fp32 [1]) and inv_scale = 1 / *grad_scale, exact for
// a power of two; otherwise inv_scale is the host's
template <bool DEV_SCALE>
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, WgParams p, int Cin, WgOut o,
                                    const float* __restrict__ scale, float inv_scale,
                                    const float* __restrict__ grad_scale, int* nonfinite) {
    const int taps = p.k * p.k;
    const long long total = (long long)o.rows * Cin * taps;
    const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= total) return;
    if (DEV_SCALE) inv_scale = 1.0f / __ldg(grad_scale);
    const int co = (int)(e / ((long long)Cin * taps));
    const int rem = (int)(e - (long long)co * Cin * taps);
    const int ci = rem / taps, tap = rem - ci * taps;
    const int tile = ((co / kWgBM) * taps + tap) * p.n_tiles + ci / kWgBN;
    const float* src = part + (size_t)tile * (kWgBM * kWgBN) + (co % kWgBM) * kWgBN + ci % kWgBN;
    const size_t sstride = (size_t)p.tiles * (kWgBM * kWgBN);
    float acc = 0.f;
    for (int s = 0; s < p.splits; ++s) acc += __ldg(src + s * sstride);
    const float v = acc * (scale ? __ldg(scale + co) : 1.f) * inv_scale;
    store_row_value(o.dw, o.dw_hi, o.split, co, (size_t)Cin * taps, rem, v, o.accumulate, nonfinite);
}

// bias gradient, first level: partial[chunk][c] = sum of rows [chunk*rows, ...) of dy[M][C] (row pitch ld, ascending)
__global__ void colsum_partial_kernel(const float* __restrict__ dy, long long M, int C, long long ld, long long rows,
                                      float* __restrict__ partial) {
    const long long r0 = (long long)blockIdx.x * rows;
    const long long r1 = min(M, r0 + rows);
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float acc = 0.f;
        for (long long r = r0; r < r1; ++r) acc += __ldg(dy + r * ld + c);
        partial[(size_t)blockIdx.x * C + c] = acc;
    }
}

template <bool DEV_SCALE>
__global__ void colsum_final_kernel(const float* __restrict__ partial, int chunks, int C, float inv_scale,
                                    const float* __restrict__ grad_scale, WgOut o, int* nonfinite) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= o.rows) return;
    if (DEV_SCALE) inv_scale = 1.0f / __ldg(grad_scale);
    float acc = 0.f;
    for (int i = 0; i < chunks; ++i) acc += partial[(size_t)i * C + c];
    store_row_value(o.db, o.db_hi, o.split, c, 1, 0, acc * inv_scale, o.accumulate, nonfinite);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

bool make_map16(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                const cuuint32_t* box) {
    static EncodeTiledFn enc = nullptr;
    if (!enc) {
        void* fp = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            return false;
        enc = (EncodeTiledFn)fp;
    }
    cuuint32_t estr[4] = {1, 1, 1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box,
               estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// launch geometry shared by the workspace query and the launch
WgParams plan(int N, int H, int W, int Cin, int Cout, int k) {
    WgParams p = {};
    p.patch = k == 3 ? 1 : 0;
    p.N = N; p.H = H; p.W = W; p.k = k;
    p.wchunks = (W + kWgBK - 1) / kWgBK;
    const long long M = (long long)N * H * W;
    p.num_kb = p.patch ? N * H * p.wchunks : (int)((M + kWgBK - 1) / kWgBK);
    p.m_tiles = (Cout + kWgBM - 1) / kWgBM;
    p.n_tiles = (Cin + kWgBN - 1) / kWgBN;
    p.tiles = p.m_tiles * k * k * p.n_tiles;
    // about two CTAs per SM in total, every split at least 8 K-blocks long
    int splits = (2 * sb_num_sms() + p.tiles - 1) / p.tiles;
    splits = max(1, min(splits, p.num_kb / 8));
    p.kb_per_split = (p.num_kb + splits - 1) / splits;
    p.splits = (p.num_kb + p.kb_per_split - 1) / p.kb_per_split;
    return p;
}

size_t part_bytes(const WgParams& p) { return (size_t)p.splits * p.tiles * kWgBM * kWgBN * sizeof(float); }

int bias_chunks(long long M) { return (int)min((long long)kBiasChunks, M); }

size_t wgrad_workspace(int N, int H, int W, int Cin, int Cout, int k) {
    if (N < 1 || H < 1 || W < 1 || Cin < 1 || Cout < 1 || (k != 1 && k != 3)) return 0;
    const WgParams p = plan(N, H, W, Cin, Cout, k);
    return part_bytes(p) + (size_t)kBiasChunks * Cout * sizeof(float) + 256;
}

bool misaligned(const void* q, uintptr_t a) { return (reinterpret_cast<uintptr_t>(q) & (a - 1)) != 0; }

// dy16 / x16 / dy32 rows (pixels) are dy_ld / x_ld / dy32_ld elements apart; every argument is checked before the
// first launch.  grad_scale (device, may be NULL): the gradient scale read on the device in place of inv_grad_scale
int conv_wgrad(const void* dy16, int dy_ld, const void* x16, int x_ld, int N, int H, int W, int Cin, int Cout, int k,
               const float* scale, float inv_grad_scale, const float* grad_scale, const float* dy32, int dy32_ld,
               WgOut o, int* nonfinite, void* workspace, size_t workspace_bytes, cudaStream_t st) {
    if (!dy16 || !x16 || !o.dw || N < 1 || H < 1 || W < 1 || (k != 1 && k != 3)) return SB_EINVAL;
    if (Cin < 64 || Cout < 64 || Cin % 64 || Cout % 64 || (o.db && !dy32)) return SB_EINVAL;
    if (dy_ld < Cout || x_ld < Cin || dy_ld % 8 || x_ld % 8 || (dy32 && dy32_ld < Cout)) return SB_EINVAL;
    if (o.rows < 1 || o.rows > Cout || o.split < 1 || o.split > o.rows || (o.split < o.rows && !o.dw_hi) ||
        (o.db && o.split < o.rows && !o.db_hi))
        return SB_EINVAL;
    if (misaligned(dy16, 16) || misaligned(x16, 16) || misaligned(workspace, 16) || misaligned(dy32, 4))
        return SB_EINVAL;
    if (workspace_bytes < wgrad_workspace(N, H, W, Cin, Cout, k)) return SB_EINVAL;
    const long long M = (long long)N * H * W;
    if (M >= 0x7fffffffLL) return SB_EINVAL;
    WgParams p = plan(N, H, W, Cin, Cout, k);
    p.part = reinterpret_cast<float*>(workspace);

    CUtensorMap mdy, mx;
    const cuuint64_t yl = (cuuint64_t)dy_ld * 2, xl = (cuuint64_t)x_ld * 2;
    if (p.patch) {
        cuuint64_t dd[4] = {(cuuint64_t)Cout, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
        cuuint64_t ds[3] = {yl, W * yl, (cuuint64_t)H * W * yl};
        cuuint64_t xd[4] = {(cuuint64_t)Cin, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
        cuuint64_t xs[3] = {xl, W * xl, (cuuint64_t)H * W * xl};
        cuuint32_t box[4] = {64, (cuuint32_t)kWgBK, 1, 1};
        if (!make_map16(&mdy, dy16, 4, dd, ds, box) || !make_map16(&mx, x16, 4, xd, xs, box)) return SB_EINVAL;
    } else {
        cuuint64_t dd[2] = {(cuuint64_t)Cout, (cuuint64_t)M}, ds[1] = {yl};
        cuuint64_t xd[2] = {(cuuint64_t)Cin, (cuuint64_t)M}, xs[1] = {xl};
        cuuint32_t box[2] = {64, (cuuint32_t)kWgBK};
        if (!make_map16(&mdy, dy16, 2, dd, ds, box) || !make_map16(&mx, x16, 2, xd, xs, box)) return SB_EINVAL;
    }
    static bool attr_done[kSbMaxDevices] = {false};
    bool& attr = attr_done[sb_cur_device()];
    if (!attr) {
        cudaError_t e = cudaFuncSetAttribute(conv_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kWgSmem);
        if (e != cudaSuccess) return (int)e;
        attr = true;
    }
    conv_wgrad_kernel<<<p.tiles * p.splits, kWgThreads, kWgSmem, st>>>(mdy, mx, p);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    const long long total = (long long)o.rows * Cin * k * k;
    if (grad_scale)
        wgrad_reduce_kernel<true><<<sb_div_up(total, 256), 256, 0, st>>>(p.part, p, Cin, o, scale, 0.f, grad_scale,
                                                                        nonfinite);
    else
        wgrad_reduce_kernel<false><<<sb_div_up(total, 256), 256, 0, st>>>(p.part, p, Cin, o, scale, inv_grad_scale,
                                                                         nullptr, nonfinite);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    if (o.db) {
        float* bp = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(workspace) + part_bytes(p));
        const int chunks = bias_chunks(M);
        const long long rows = (M + chunks - 1) / chunks;
        colsum_partial_kernel<<<chunks, 256, 0, st>>>(dy32, M, Cout, dy32_ld, rows, bp);
        SB_LAUNCHED();
        SB_CHECK_LAUNCH();
        if (grad_scale)
            colsum_final_kernel<true><<<sb_div_up(o.rows, 256), 256, 0, st>>>(bp, chunks, Cout, 0.f, grad_scale, o,
                                                                             nonfinite);
        else
            colsum_final_kernel<false><<<sb_div_up(o.rows, 256), 256, 0, st>>>(bp, chunks, Cout, inv_grad_scale,
                                                                              nullptr, o, nonfinite);
        SB_LAUNCHED();
        SB_CHECK_LAUNCH();
    }
    return SB_OK;
}

}  // namespace

extern "C" size_t sb_conv_wgrad_workspace(int N, int H, int W, int Cin, int Cout, int k) {
    return wgrad_workspace(N, H, W, Cin, Cout, k);
}

extern "C" int sb_conv_wgrad(const void* dy16, const void* x16, int N, int H, int W, int Cin, int Cout, int k,
                             const float* scale, float inv_grad_scale, float* dw, const float* dy32, float* db,
                             int* nonfinite, void* workspace, size_t workspace_bytes, sb_stream_t stream) {
    const WgOut o = {dw, nullptr, db, nullptr, Cout, Cout, 0};
    return conv_wgrad(dy16, Cout, x16, Cin, N, H, W, Cin, Cout, k, scale, inv_grad_scale, nullptr, dy32, Cout, o,
                      nonfinite, workspace, workspace_bytes, sb_cs(stream));
}

extern "C" int sb_conv_wgrad_devscale(const void* dy16, const void* x16, int N, int H, int W, int Cin, int Cout, int k,
                                      const float* scale, const float* grad_scale, float* dw, const float* dy32,
                                      float* db, int* nonfinite, void* workspace, size_t workspace_bytes,
                                      sb_stream_t stream) {
    if (!grad_scale) return SB_EINVAL;
    const WgOut o = {dw, nullptr, db, nullptr, Cout, Cout, 0};
    return conv_wgrad(dy16, Cout, x16, Cin, N, H, W, Cin, Cout, k, scale, 0.f, grad_scale, dy32, Cout, o, nonfinite,
                      workspace, workspace_bytes, sb_cs(stream));
}

extern "C" size_t sb_conv_wgrad_acc_workspace(int N, int H, int W, int Cin, int Cout, int k) {
    return wgrad_workspace(N, H, W, Cin, Cout, k);
}

extern "C" int sb_conv_wgrad_acc(const void* dy16, int dy_ld, const void* x16, int x_ld, int N, int H, int W, int Cin,
                                 int Cout, int k, const float* scale, float inv_grad_scale, const float* dy32,
                                 int dy32_ld, int accumulate, int rows, int split, float* dw, float* db, float* dw_hi,
                                 float* db_hi, int* nonfinite, void* workspace, size_t workspace_bytes,
                                 sb_stream_t stream) {
    const WgOut o = {dw, dw_hi, db, db_hi, rows, split, accumulate ? 1 : 0};
    return conv_wgrad(dy16, dy_ld, x16, x_ld, N, H, W, Cin, Cout, k, scale, inv_grad_scale, nullptr, dy32, dy32_ld, o,
                      nonfinite, workspace, workspace_bytes, sb_cs(stream));
}

extern "C" int sb_conv_wgrad_acc_devscale(const void* dy16, int dy_ld, const void* x16, int x_ld, int N, int H, int W,
                                          int Cin, int Cout, int k, const float* scale, const float* grad_scale,
                                          const float* dy32, int dy32_ld, int accumulate, int rows, int split,
                                          float* dw, float* db, float* dw_hi, float* db_hi, int* nonfinite,
                                          void* workspace, size_t workspace_bytes, sb_stream_t stream) {
    if (!grad_scale) return SB_EINVAL;
    const WgOut o = {dw, dw_hi, db, db_hi, rows, split, accumulate ? 1 : 0};
    return conv_wgrad(dy16, dy_ld, x16, x_ld, N, H, W, Cin, Cout, k, scale, 0.f, grad_scale, dy32, dy32_ld, o,
                      nonfinite, workspace, workspace_bytes, sb_cs(stream));
}

// ------------------------------------------------------------------ FPN level gradient
namespace {

// align_corners source row of fine row `o` (the forward's arithmetic, conv_tc.cu epilogue): y1 and weight of y1 + 1
struct UpTap { int i1; float l1; bool b; };
__device__ __forceinline__ UpTap up_tap(float r, int o, int n_coarse) {
    const float s = __fmul_rn(r, (float)o);
    UpTap t;
    t.i1 = (int)s;
    t.l1 = s - (float)t.i1;
    t.b = t.i1 < n_coarse - 1;
    return t;
}

// weight with which fine row o reads coarse row y (0 if it does not): the forward's taps are (i1, 1 - l1) and
// (b ? i1 + 1 : i1, l1)
__device__ __forceinline__ float up_weight(const UpTap& t, int y) {
    float w = 0.f;
    if (t.i1 == y) w += 1.f - t.l1;
    if ((t.b ? t.i1 + 1 : t.i1) == y) w += t.l1;
    return w;
}

// fine rows [lo, hi] whose taps can touch coarse row y (i1 is non-decreasing in o)
__device__ __forceinline__ void fine_range(float r, int y, int n_coarse, int n_fine, int& lo, int& hi) {
    if (r <= 0.f) { lo = 0; hi = n_fine - 1; return; }
    lo = max(0, (int)floorf((float)(y - 1) / r) - 2);
    while (lo > 0 && up_tap(r, lo - 1, n_coarse).i1 >= y - 1) --lo;
    while (lo < n_fine && up_tap(r, lo, n_coarse).i1 < y - 1) ++lo;
    hi = lo;
    while (hi + 1 < n_fine && up_tap(r, hi + 1, n_coarse).i1 <= y) ++hi;
}

// one block per coarse pixel, threads over channels (fixed summation order: fine rows, then fine columns, ascending);
// DEV_SCALE: scale is read from scale_dev (device, fp32 [1])
template <bool DEV_SCALE>
__global__ void fpn_grad_combine_kernel(const float* __restrict__ dp, const float* __restrict__ dt, int N, int H,
                                        int W, int TH, int TW, int C, const float* __restrict__ dp6, int H6, int W6,
                                        float scale, const float* __restrict__ scale_dev, float* __restrict__ out,
                                        __half* __restrict__ out16) {
    if (DEV_SCALE) scale = __ldg(scale_dev);
    const int pix = blockIdx.x;
    const int x = pix % W, y = (pix / W) % H, n = pix / (W * H);
    int ylo = 0, yhi = -1, xlo = 0, xhi = -1;
    float rh = 0.f, rw = 0.f;
    if (dt) {
        rh = TH > 1 ? __fdiv_rn((float)(H - 1), (float)(TH - 1)) : 0.f;
        rw = TW > 1 ? __fdiv_rn((float)(W - 1), (float)(TW - 1)) : 0.f;
        fine_range(rh, y, H, TH, ylo, yhi);
        fine_range(rw, x, W, TW, xlo, xhi);
    }
    const bool p6 = dp6 && !(y & 1) && !(x & 1);
    const size_t o = (size_t)pix * C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float acc = dp ? scale * dp[o + c] : 0.f;
        for (int yy = ylo; yy <= yhi; ++yy) {
            const float wy = up_weight(up_tap(rh, yy, H), y);
            if (wy == 0.f) continue;
            const float* row = dt + ((size_t)n * TH + yy) * TW * C + c;
            float racc = 0.f;
            for (int xx = xlo; xx <= xhi; ++xx) {
                const float wx = up_weight(up_tap(rw, xx, W), x);
                if (wx != 0.f) racc += wx * row[(size_t)xx * C];
            }
            acc += wy * racc;
        }
        if (p6) acc += scale * dp6[(((size_t)n * H6 + (y >> 1)) * W6 + (x >> 1)) * C + c];
        if (out) out[o + c] = acc;
        if (out16) out16[o + c] = __float2half_rn(acc);
    }
}

int fpn_grad_combine(const float* dp, const float* dt, int N, int H, int W, int TH, int TW, int C, const float* dp6,
                     int H6, int W6, float scale, const float* scale_dev, float* out, void* out16, cudaStream_t st) {
    if (N < 1 || H < 1 || W < 1 || C < 1 || (!out && !out16)) return SB_EINVAL;
    if (dt && (TH < 1 || TW < 1)) return SB_EINVAL;
    if (dp6 && (H6 != (H - 1) / 2 + 1 || W6 != (W - 1) / 2 + 1)) return SB_EINVAL;
    const long long pixels = (long long)N * H * W;
    if (pixels >= 0x7fffffffLL) return SB_EINVAL;
    const int threads = C < 256 ? C : 256;
    if (scale_dev)
        fpn_grad_combine_kernel<true><<<(int)pixels, threads, 0, st>>>(dp, dt, N, H, W, TH, TW, C, dp6, H6, W6, 0.f,
                                                                        scale_dev, out, reinterpret_cast<__half*>(out16));
    else
        fpn_grad_combine_kernel<false><<<(int)pixels, threads, 0, st>>>(dp, dt, N, H, W, TH, TW, C, dp6, H6, W6, scale,
                                                                         nullptr, out, reinterpret_cast<__half*>(out16));
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

}  // namespace

extern "C" int sb_fpn_grad_combine(const float* dp, const float* dt, int N, int H, int W, int TH, int TW, int C,
                                   const float* dp6, int H6, int W6, float scale, float* out, void* out16,
                                   sb_stream_t stream) {
    return fpn_grad_combine(dp, dt, N, H, W, TH, TW, C, dp6, H6, W6, scale, nullptr, out, out16, sb_cs(stream));
}

extern "C" int sb_fpn_grad_combine_devscale(const float* dp, const float* dt, int N, int H, int W, int TH, int TW,
                                            int C, const float* dp6, int H6, int W6, const float* scale, float* out,
                                            void* out16, sb_stream_t stream) {
    if (!scale) return SB_EINVAL;
    return fpn_grad_combine(dp, dt, N, H, W, TH, TW, C, dp6, H6, W6, 0.f, scale, out, out16, sb_cs(stream));
}
