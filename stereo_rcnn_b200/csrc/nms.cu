// nms.cu -- bitmask NMS with a device-side greedy reduction (sm_90a).
//
// Replaces lib/model/nms/src/nms_cuda_kernel.cu:41-161 of the reference
// (nms_kernel + the host-side scan of nms_cuda_compute).  Same arithmetic
// (devIoU with "+1" areas, strict '>' against the threshold, boxes pre-sorted),
// different machine mapping:
//   * only the upper triangle of 64x64 tiles is computed (the reference computes
//     the full square and never reads the lower half);
//   * the greedy scan runs on the device, one 64-box chunk at a time: the chunk's
//     diagonal tile is resolved with warp shuffles, and both the tile and the
//     chunk's suppression word (OR of that word over all boxes kept so far) are
//     requested from L2 one chunk ahead of their use;
//   * no cudaMalloc / cudaMemcpy / default-stream sync: workspace is caller-owned,
//     everything is ordered on the caller's stream;
//   * two box sets that share scores (left / right proposals) are reduced in
//     lock step and intersected on the fly (np.intersect1d of
//     proposal_layer.py:128), stopping as soon as `max_out` survivors exist.
#include "common.cuh"

namespace {

constexpr int kTile = 64;
constexpr int kMaxWords = 256;  // n <= 16384

__global__ void __launch_bounds__(kTile)
nms_mask_kernel(const float* __restrict__ boxes0, const float* __restrict__ boxes1, int stride,
                int n, float thresh, unsigned long long* __restrict__ mask0,
                unsigned long long* __restrict__ mask1) {
    const int row = blockIdx.y, col = blockIdx.x;
    if (col < row) return;  // upper triangle only
    const float* boxes = blockIdx.z ? boxes1 : boxes0;
    unsigned long long* mask = blockIdx.z ? mask1 : mask0;
    const int cb = (n + kTile - 1) / kTile;
    const int row_size = min(n - row * kTile, kTile);
    const int col_size = min(n - col * kTile, kTile);
    __shared__ float4 cbox[kTile];
    const int t = threadIdx.x;
    if (t < col_size) {
        const float* p = boxes + (size_t)(col * kTile + t) * stride;
        cbox[t] = make_float4(p[0], p[1], p[2], p[3]);
    }
    __syncthreads();
    if (t < row_size) {
        const int i = row * kTile + t;
        const float* p = boxes + (size_t)i * stride;
        const float4 cur = make_float4(p[0], p[1], p[2], p[3]);
        unsigned long long bits = 0;
        const int start = (row == col) ? t + 1 : 0;
        for (int j = start; j < col_size; ++j)
            if (sb_iou_gt(cur, cbox[j], thresh)) bits |= 1ULL << j;
        mask[(size_t)i * cb + col] = bits;
    }
}

// One CTA, 256 threads per side.  keep_out receives ascending indices of boxes kept by *every* side; at most
// max_out of them.
//
// The scan is a chain of 64-box chunks, and each link needs two things from the mask in L2: the chunk's diagonal
// tile, and the suppression word of the chunk = OR of word c over every box kept so far.  Both are requested one
// chunk ahead, so a link costs max(resolve, one L2 round trip) instead of two round trips back to back:
//   * thread j of a side owns chunk j: while chunk c is being resolved it gathers word c+1 of the rows chunk j
//     kept (j < c), and the partial words are OR-reduced into shared memory;
//   * warp 0 of the side holds, for the rows of chunk c, word c (the diagonal tile, resolved with shuffles as
//     before) and word c+1: the boxes chunk c itself keeps are known only after the resolve, and their word c+1 is
//     then already in registers ("carry").
template <int NS>
__global__ void __launch_bounds__(256 * NS)
nms_reduce_kernel(const unsigned long long* __restrict__ mask0,
                  const unsigned long long* __restrict__ mask1, int n, int max_out,
                  int* __restrict__ keep_out, int* __restrict__ num_out) {
    __shared__ unsigned long long keepbits[NS][kMaxWords];   // per side: survivors of every resolved chunk
    __shared__ unsigned long long colacc[NS][2];             // [c & 1]: OR of word c over the survivors of chunks < c-1... see below
    __shared__ int count;
    const int side = threadIdx.x >> 8, t = threadIdx.x & 255, lane = t & 31;
    const unsigned long long* mask = side ? mask1 : mask0;
    const int cb = (n + kTile - 1) / kTile;
    if (t < 2) colacc[side][t] = 0;
    if (threadIdx.x == 0) count = 0;
    // warp 0: rows lane and lane+32 of the current chunk: word c (d*) and word c+1 (e*)
    unsigned long long d0 = 0, d1 = 0, e0 = 0, e1 = 0, carry = 0;
    auto load_rows = [&](int c, unsigned long long& a0, unsigned long long& a1, unsigned long long& b0,
                         unsigned long long& b1) {
        const int csize = min(n - c * kTile, kTile);
        const size_t r0 = (size_t)(c * kTile + lane) * cb, r1 = r0 + (size_t)32 * cb;
        a0 = (lane < csize) ? mask[r0 + c] : 0ULL;
        a1 = (lane + 32 < csize) ? mask[r1 + c] : 0ULL;
        b0 = (lane < csize && c + 1 < cb) ? mask[r0 + c + 1] : 0ULL;
        b1 = (lane + 32 < csize && c + 1 < cb) ? mask[r1 + c + 1] : 0ULL;
    };
    if (t < 32) load_rows(0, d0, d1, e0, e1);
    __syncthreads();
    for (int c = 0; c < cb; ++c) {
        // ---- requests for chunk c+1, in flight while chunk c is resolved
        unsigned long long nd0 = 0, nd1 = 0, ne0 = 0, ne1 = 0, part = 0;
        if (c + 1 < cb) {
            if (t < 32) load_rows(c + 1, nd0, nd1, ne0, ne1);
            if (t < c) {      // word c+1 of the rows chunk t kept
                unsigned long long kb = keepbits[side][t];
                const unsigned long long* col = mask + (size_t)t * kTile * cb + (c + 1);
                while (kb) {
                    unsigned long long v[4];
#pragma unroll
                    for (int u = 0; u < 4; ++u) {          // four independent loads per trip
                        const int b = kb ? __ffsll((long long)kb) - 1 : -1;
                        kb &= kb - 1;                       // (0 & anything) stays 0
                        v[u] = b >= 0 ? col[(size_t)b * cb] : 0ULL;
                    }
                    part |= (v[0] | v[1]) | (v[2] | v[3]);
                }
            }
        }
        // ---- resolve chunk c inside warp 0 of each side
        if (t < 32) {
            const int csize = min(n - c * kTile, kTile);
            const unsigned long long valid = csize >= 64 ? ~0ULL : ((1ULL << csize) - 1ULL);
            unsigned long long cur = colacc[side][c & 1] | carry | ~valid, kb = 0;
#pragma unroll 8
            for (int b = 0; b < 32; ++b) {
                const unsigned long long row = __shfl_sync(0xffffffffu, d0, b);
                if (!((cur >> b) & 1ULL)) { kb |= 1ULL << b; cur |= row; }
            }
#pragma unroll 8
            for (int b = 0; b < 32; ++b) {
                const unsigned long long row = __shfl_sync(0xffffffffu, d1, b);
                if (!((cur >> (b + 32)) & 1ULL)) { kb |= 1ULL << (b + 32); cur |= row; }
            }
            // word c+1 of the rows this chunk keeps -> next chunk's carry (every lane gets the full OR)
            unsigned long long mine = (((kb >> lane) & 1ULL) ? e0 : 0ULL) | (((kb >> (lane + 32)) & 1ULL) ? e1 : 0ULL);
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) mine |= __shfl_xor_sync(0xffffffffu, mine, o);
            carry = mine;
            if (lane == 0) { keepbits[side][c] = kb; colacc[side][c & 1] = 0; }    // slot c&1 is reused for word c+2
            d0 = nd0; d1 = nd1; e0 = ne0; e1 = ne1;
        }
        // ---- OR-reduce the gathered partial words of chunk c+1 into colacc[(c+1)&1]
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) part |= __shfl_xor_sync(0xffffffffu, part, o);
        if (lane == 0 && part) atomicOr(&colacc[side][(c + 1) & 1], part);
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long both = keepbits[0][c];
            if (NS == 2) both &= keepbits[NS - 1][c];
            int cnt = count;
            while (both && cnt < max_out) {
                int b = __ffsll((long long)both) - 1;
                both &= both - 1;
                keep_out[cnt++] = c * kTile + b;
            }
            count = cnt;
        }
        __syncthreads();
        if (count >= max_out) break;
    }
    if (threadIdx.x == 0) *num_out = count;
}

}  // namespace

// shared with proposal.cu
int sb_nms_launch(const float* boxes0, const float* boxes1, int stride, int n, float thresh,
                  unsigned long long* mask0, unsigned long long* mask1, int max_out, int* keep,
                  int* num_out, cudaStream_t st) {
    if (n > kTile * kMaxWords) return SB_EINVAL;
    const int ns = boxes1 ? 2 : 1;
    if (n == 0) {
        cudaMemsetAsync(num_out, 0, sizeof(int), st);
        return SB_OK;
    }
    const int cb = (n + kTile - 1) / kTile;
    dim3 grid(cb, cb, ns);
    nms_mask_kernel<<<grid, kTile, 0, st>>>(boxes0, boxes1, stride, n, thresh, mask0, mask1);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    if (ns == 1)
        nms_reduce_kernel<1><<<1, 256, 0, st>>>(mask0, mask0, n, max_out, keep, num_out);
    else
        nms_reduce_kernel<2><<<1, 512, 0, st>>>(mask0, mask1, n, max_out, keep, num_out);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" size_t sb_nms_workspace_bytes(int n) {
    size_t cb = (size_t)(n + kTile - 1) / kTile;
    return (size_t)n * cb * sizeof(unsigned long long) + 256;
}

extern "C" int sb_nms(const float* dets, int n, float thresh, int* keep, int* num_out,
                      void* workspace, size_t workspace_bytes, sb_stream_t stream) {
    if (n < 0 || !keep || !num_out) return SB_EINVAL;
    if (n > 0 && (!dets || !workspace || workspace_bytes < sb_nms_workspace_bytes(n))) return SB_EINVAL;
    return sb_nms_launch(dets, nullptr, 5, n, thresh, (unsigned long long*)workspace, nullptr, n, keep,
                         num_out, sb_cs(stream));
}

extern "C" int sb_nms_mask(const float* dets, int n, float thresh, uint64_t* mask, sb_stream_t stream) {
    if (n <= 0) return n == 0 ? SB_OK : SB_EINVAL;
    if (n > kTile * kMaxWords || !dets || !mask) return SB_EINVAL;
    const int cb = (n + kTile - 1) / kTile;
    cudaMemsetAsync(mask, 0, (size_t)n * cb * sizeof(uint64_t), sb_cs(stream));
    dim3 grid(cb, cb, 1);
    nms_mask_kernel<<<grid, kTile, 0, sb_cs(stream)>>>(dets, nullptr, 5, n, thresh,
                                                      (unsigned long long*)mask, nullptr);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}
