// optim.cu -- the optimizer step of a training step and the device-side refresh of the engine's packed weights
// (SURVEY A16).
//
//   sb_sgd_step      torch.optim.SGD.step (trainval_net.py:168,227), dampening 0, no Nesterov: multi-tensor, the
//                    learning rate read on the device, skipped when the backward raised found_inf
//   sb_pack_plan     validate a table of pack targets and assign its tiles
//   sb_pack_weights  rewrite every derived copy of a table (K-major, TF32-rounded, fp16, transposed and flipped, frozen-BN
//                    scale folded) from the fp32 masters in one launch
//
// Both are pure bandwidth: every element is read once and written once per output.
#include <cuda_fp16.h>
#include <math.h>

#include "common.cuh"

namespace {

// --------------------------------------------------------------------------------------------- SGD
constexpr int kSgdTensors = 48, kSgdThreads = 256, kSgdBlockElems = 4096;    // 4 float4 per thread per CTA
struct SgdChunk {
    float* p[kSgdTensors];
    const float* g[kSgdTensors];
    float* m[kSgdTensors];
    unsigned long long n[kSgdTensors];
    float wd[kSgdTensors];
    float lrm[kSgdTensors];
    unsigned block0[kSgdTensors + 1];       // first CTA of tensor i; block0[count] = grid size
    int count;
};

__device__ __forceinline__ void sgd_one(float& p, float g, float& m, float wd, float mom, float lr) {
    const float d = __fadd_rn(g, __fmul_rn(wd, p));
    m = __fadd_rn(__fmul_rn(mom, m), d);
    p = __fsub_rn(p, __fmul_rn(lr, m));
}

__global__ void __launch_bounds__(kSgdThreads)
sgd_step_kernel(const SgdChunk c, const float* __restrict__ lr, float momentum, const int* __restrict__ skip,
                int* __restrict__ skipped, int count_skip) {
    if (*skip != 0) {
        if (count_skip && blockIdx.x == 0 && threadIdx.x == 0) *skipped += 1;
        return;
    }
    int lo = 0, hi = c.count - 1;                 // the tensor of this CTA: last t with block0[t] <= blockIdx.x
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (c.block0[mid] <= blockIdx.x) lo = mid; else hi = mid - 1;
    }
    const int t = lo;
    const unsigned long long n = c.n[t];
    const unsigned long long begin = (unsigned long long)(blockIdx.x - c.block0[t]) * kSgdBlockElems;
    const unsigned long long end = begin + kSgdBlockElems < n ? begin + kSgdBlockElems : n;
    float* __restrict__ P = c.p[t];
    const float* __restrict__ G = c.g[t];
    float* __restrict__ M = c.m[t];
    const float wd = c.wd[t];
    const float step = __fmul_rn(*lr, c.lrm[t]);
    unsigned long long i = begin;
    if (((reinterpret_cast<uintptr_t>(P) | reinterpret_cast<uintptr_t>(G) | reinterpret_cast<uintptr_t>(M)) & 15) == 0) {
        const unsigned long long v_end = begin + ((end - begin) & ~3ull);
        for (unsigned long long j = begin + 4ull * threadIdx.x; j < v_end; j += 4ull * kSgdThreads) {
            float4 p = *reinterpret_cast<const float4*>(P + j);
            const float4 g = __ldcs(reinterpret_cast<const float4*>(G + j));
            float4 m = *reinterpret_cast<const float4*>(M + j);
            sgd_one(p.x, g.x, m.x, wd, momentum, step);
            sgd_one(p.y, g.y, m.y, wd, momentum, step);
            sgd_one(p.z, g.z, m.z, wd, momentum, step);
            sgd_one(p.w, g.w, m.w, wd, momentum, step);
            *reinterpret_cast<float4*>(P + j) = p;
            *reinterpret_cast<float4*>(M + j) = m;
        }
        i = v_end;
    }
    for (unsigned long long j = i + threadIdx.x; j < end; j += kSgdThreads) {      // tail, or misaligned tensors
        float p = P[j], m = M[j];
        sgd_one(p, G[j], m, wd, momentum, step);
        P[j] = p;
        M[j] = m;
    }
}

// --------------------------------------------------------------------------------------------- weight packing
constexpr int kPackThreads = 256, kPackRows = 288, kPackCols = 32, kPackFlat = 4096;

__device__ __forceinline__ float tf32_nearest(float v) {           // engine.ops.round_tf32_, bit for bit
    return __uint_as_float((__float_as_uint(v) + 0x1000u) & ~0x1fffu);
}

// q / d and q % d for small q (q * d < 2^32) by one multiply: m = ceil(2^32 / d)
struct FastDiv {
    unsigned long long m;
    unsigned d;
    __device__ explicit FastDiv(unsigned d_) : m(((1ull << 32) + d_ - 1) / d_), d(d_) {}
    __device__ __forceinline__ unsigned div(unsigned q) const { return (unsigned)((q * m) >> 32); }
};

__device__ __forceinline__ void pack_store(const sb_pack_target& T, long long off, float v, long long ci) {
    switch (T.transform) {
        case SB_PACK_F32: static_cast<float*>(T.dst)[off] = v; break;
        case SB_PACK_TF32: static_cast<float*>(T.dst)[off] = tf32_nearest(v); break;
        case SB_PACK_F16: static_cast<__half*>(T.dst)[off] = __float2half_rn(v); break;
        default: static_cast<__half*>(T.dst)[off] = __float2half_rn(__fmul_rn(v, T.scale[ci])); break;
    }
    if (T.dst16) static_cast<__half*>(T.dst16)[off] = __float2half_rn(v);
}

__global__ void __launch_bounds__(kPackThreads)
pack_weights_kernel(const sb_pack_target* __restrict__ tab, int n_targets) {
    __shared__ float tile[kPackRows * (kPackCols + 1)];
    const long long blk = blockIdx.x;
    int lo = 0, hi = n_targets - 1;              // the target of this CTA: last t with tile0 <= blockIdx.x
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (tab[mid].tile0 <= blk) lo = mid; else hi = mid - 1;
    }
    const sb_pack_target T = tab[lo];             // a private copy: stores through dst cannot alias it
    const int t1 = T.tile[0], t2 = T.tile[1], t3 = T.tile[2];
    const long long n1 = (T.shape[1] + t1 - 1) / t1, n2 = (T.shape[2] + t2 - 1) / t2, n3 = (T.shape[3] + t3 - 1) / t3;
    long long r = blk - T.tile0;
    const long long c3 = r % n3;
    r /= n3;
    const long long c2 = r % n2;
    r /= n2;
    const long long c1 = r % n1;
    const long long i0 = r / n1;
    const long long b1 = c1 * t1, b2 = c2 * t2, b3 = c3 * t3;
    const int e1 = (int)min((long long)t1, T.shape[1] - b1), e2 = (int)min((long long)t2, T.shape[2] - b2),
              e3 = (int)min((long long)t3, T.shape[3] - b3);
    const long long s1 = T.src_stride[1], s2 = T.src_stride[2], s3 = T.src_stride[3];
    const long long d1 = T.dst_stride[1], d2 = T.dst_stride[2];
    const float* __restrict__ src = T.src + (T.src_offset + i0 * T.src_stride[0] + b1 * s1 + b2 * s2 + b3 * s3);
    const long long dbase = T.dst_offset + i0 * T.dst_stride[0] + b1 * d1 + b2 * d2 + b3;
    const long long sc_base = T.scale_dim == 0 ? i0 : T.scale_dim == 1 ? b1 : T.scale_dim == 2 ? b2 : b3;
    auto sc_index = [&](int k, int a, int b) -> long long {
        return sc_base + (T.scale_dim == 1 ? k : T.scale_dim == 2 ? a : T.scale_dim == 3 ? b : 0);
    };
    if (!T.tiled) {                               // i3 is contiguous in both: straight through
        for (int b = threadIdx.x; b < e3; b += kPackThreads)
            pack_store(T, dbase + b, src[(long long)b * s3], sc_index(0, 0, b));
        return;
    }
    // tile element (k, a, b) = (i1 - b1, i2 - b2, i3 - b3) lives at row a * e1 + k, column b
    const FastDiv div1((unsigned)e1);
    const int n_el = e1 * e2 * e3;
    if (T.tiled == 1) {                           // reads: i1 fastest, then i2, then i3
        const FastDiv div2((unsigned)e2);
        for (int idx = threadIdx.x; idx < n_el; idx += kPackThreads) {
            const unsigned q = div1.div(idx), k = idx - q * e1;
            const unsigned b = div2.div(q), a = q - b * e2;
            tile[(a * e1 + k) * (kPackCols + 1) + b] = src[k * s1 + a * s2 + b * s3];
        }
    } else {                                      // reads: i1 fastest, then i3, then i2
        const FastDiv div3((unsigned)e3);
        for (int idx = threadIdx.x; idx < n_el; idx += kPackThreads) {
            const unsigned q = div1.div(idx), k = idx - q * e1;
            const unsigned a = div3.div(q), b = q - a * e3;
            tile[(a * e1 + k) * (kPackCols + 1) + b] = src[k * s1 + a * s2 + b * s3];
        }
    }
    __syncthreads();
    const int rows = e1 * e2;                     // writes: i3 fastest (one 32-wide run per row)
    for (int row = threadIdx.x / kPackCols; row < rows; row += kPackThreads / kPackCols) {
        const int b = threadIdx.x % kPackCols;
        if (b >= e3) continue;
        const unsigned a = div1.div(row), k = row - a * e1;
        pack_store(T, dbase + k * d1 + a * d2 + b, tile[row * (kPackCols + 1) + b], sc_index(k, a, b));
    }
}

// the tiling of one target (what sb_pack_plan assigns and sb_pack_weights re-checks)
void pack_tiling(const sb_pack_target& t, int tile[3], int* tiled) {
    if (t.src_stride[3] == 1 || t.shape[3] == 1) {
        tile[0] = 1;
        tile[1] = 1;
        tile[2] = kPackFlat;
        *tiled = 0;
        return;
    }
    const long long t1 = t.shape[1] < kPackRows ? t.shape[1] : kPackRows;
    const long long t2 = t.shape[2] < kPackRows / t1 ? t.shape[2] : kPackRows / t1;
    tile[0] = (int)t1;
    tile[1] = (int)t2;
    tile[2] = kPackCols;
    // reads walk i1 first; then whichever of i2 / i3 the source stores closer (shorter |stride|)
    const long long s2 = t.src_stride[2] < 0 ? -t.src_stride[2] : t.src_stride[2];
    const long long s3 = t.src_stride[3] < 0 ? -t.src_stride[3] : t.src_stride[3];
    *tiled = (t.shape[2] > 1 && s2 <= s3) ? 1 : 2;
}

long long pack_tiles(const sb_pack_target& t, const int tile[3]) {
    return t.shape[0] * ((t.shape[1] + tile[0] - 1) / tile[0]) * ((t.shape[2] + tile[1] - 1) / tile[1]) *
           ((t.shape[3] + tile[2] - 1) / tile[2]);
}

bool pack_target_ok(const sb_pack_target& t) {
    if (!t.src || !t.dst || t.transform < SB_PACK_F32 || t.transform > SB_PACK_SCALE_F16) return false;
    if ((t.scale != nullptr) != (t.transform == SB_PACK_SCALE_F16)) return false;
    if (t.scale_dim < 0 || t.scale_dim > 3) return false;
    if (t.dst16 && t.transform >= SB_PACK_F16) return false;
    if (t.dst_stride[3] != 1) return false;
    long long slo = t.src_offset, dlo = t.dst_offset;
    for (int k = 0; k < 4; ++k) {
        if (t.shape[k] < 1 || t.shape[k] > (1ll << 40)) return false;
        if (t.src_stride[k] < 0) slo += (t.shape[k] - 1) * t.src_stride[k];
        if (t.dst_stride[k] < 0) dlo += (t.shape[k] - 1) * t.dst_stride[k];
    }
    return slo >= 0 && dlo >= 0;
}

}  // namespace

extern "C" int sb_sgd_step(float* const* params, float* const* grads, float* const* moms, const size_t* counts,
                           const float* weight_decay, const float* lr_mult, int n_tensors, const float* lr,
                           float momentum, const int* skip, int* skipped, sb_stream_t stream) {
    if (!params || !grads || !moms || !counts || !weight_decay || !lr_mult || n_tensors < 1 || !lr || !skip ||
        !skipped || !isfinite(momentum))
        return SB_EINVAL;
    for (int i = 0; i < n_tensors; ++i)
        if (!params[i] || !grads[i] || !moms[i] || counts[i] == 0 || !(weight_decay[i] >= 0.f) ||
            !isfinite(weight_decay[i]) || !(lr_mult[i] >= 0.f) || !isfinite(lr_mult[i]))
            return SB_EINVAL;
    for (int base = 0; base < n_tensors; base += kSgdTensors) {      // every chunk's grid must fit before any launch
        unsigned long long blocks = 0;
        for (int i = base; i < n_tensors && i < base + kSgdTensors; ++i)
            blocks += (counts[i] + kSgdBlockElems - 1) / kSgdBlockElems;
        if (blocks >= (1ull << 31)) return SB_EINVAL;
    }
    cudaStream_t st = sb_cs(stream);
    for (int base = 0; base < n_tensors; base += kSgdTensors) {
        SgdChunk c;
        c.count = n_tensors - base < kSgdTensors ? n_tensors - base : kSgdTensors;
        unsigned blocks = 0;
        for (int i = 0; i < kSgdTensors; ++i) {
            const bool on = i < c.count;
            c.p[i] = on ? params[base + i] : nullptr;
            c.g[i] = on ? grads[base + i] : nullptr;
            c.m[i] = on ? moms[base + i] : nullptr;
            c.n[i] = on ? (unsigned long long)counts[base + i] : 0ull;
            c.wd[i] = on ? weight_decay[base + i] : 0.f;
            c.lrm[i] = on ? lr_mult[base + i] : 0.f;
            c.block0[i] = blocks;
            if (on) blocks += (unsigned)((c.n[i] + kSgdBlockElems - 1) / kSgdBlockElems);
        }
        c.block0[kSgdTensors] = blocks;
        sgd_step_kernel<<<blocks, kSgdThreads, 0, st>>>(c, lr, momentum, skip, skipped, base == 0);
        SB_LAUNCHED();
    }
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" int sb_pack_plan(sb_pack_target* targets, int n_targets, long long* n_tiles) {
    if (!targets || n_targets < 1 || !n_tiles) return SB_EINVAL;
    long long total = 0;
    for (int i = 0; i < n_targets; ++i) {
        sb_pack_target& t = targets[i];
        if (!pack_target_ok(t)) return SB_EINVAL;
        pack_tiling(t, t.tile, &t.tiled);
        t.tile0 = total;
        total += pack_tiles(t, t.tile);
        if (total >= (1ll << 31)) return SB_EINVAL;
    }
    *n_tiles = total;
    return SB_OK;
}

extern "C" int sb_pack_weights(const sb_pack_target* targets, const sb_pack_target* targets_dev, int n_targets,
                               sb_stream_t stream) {
    if (!targets || !targets_dev || n_targets < 1) return SB_EINVAL;
    long long total = 0;
    for (int i = 0; i < n_targets; ++i) {
        const sb_pack_target& t = targets[i];
        if (!pack_target_ok(t)) return SB_EINVAL;
        int tile[3], tiled;
        pack_tiling(t, tile, &tiled);
        if (tile[0] != t.tile[0] || tile[1] != t.tile[1] || tile[2] != t.tile[2] || tiled != t.tiled ||
            t.tile0 != total)
            return SB_EINVAL;
        total += pack_tiles(t, tile);
        if (total >= (1ll << 31)) return SB_EINVAL;
    }
    pack_weights_kernel<<<(unsigned)total, kPackThreads, 0, sb_cs(stream)>>>(targets_dev, n_targets);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}
