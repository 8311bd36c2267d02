// train_input.cu -- the training side of the input pipeline (SURVEY 8f-3): the blobs of a stereo pair with the flip
// augmentation (minibatch.py:116-119), the per-step ground truth (minibatch.py:43-85, roibatchLoader.py:72-107) and
// the random words of a step (Philox4x32-10), all from device-side flags and counters so that one captured graph
// serves every entry of a dataset.  No host synchronisation anywhere.
#include <math.h>

#include "common.cuh"
#include "prep_image.cuh"

namespace {

constexpr int kMaxGtRows = 1024;       // annotation-row capacity N of sb_train_gt (one CTA ranks them in shared memory)
constexpr int kMaxNumGt = 30;          // cfg.MAX_NUM_GT_BOXES (config.py:283)
constexpr int kMaxPrepPairs = 32767;   // 2 B CTAs along grid z, whose limit is 65535

// blockIdx.z = 2 b + side: pair b of the batch, side 0 (left blob) or 1 (right blob)
__global__ void __launch_bounds__(256)
prep_stereo_pair_kernel(const uint8_t* __restrict__ left, const uint8_t* __restrict__ right, int H, int W, double inv,
                        int rgb, const int* __restrict__ flip, float* __restrict__ out_left,
                        float* __restrict__ out_right, int Ho, int Wo) {
    const int x = blockIdx.x * 256 + threadIdx.x, y = blockIdx.y, b = blockIdx.z >> 1, side = blockIdx.z & 1;
    if (x >= Wo) return;
    const int f = flip[b] != 0;
    const size_t in_off = (size_t)b * H * W * 3, out_off = (size_t)b * 3 * Ho * Wo;
    // flipped: the left blob is the mirrored right frame and the right blob the mirrored left frame
    const uint8_t* src = ((side == 0) != (f != 0) ? left : right) + in_off;
    prep_pixel(src, H, W, inv, rgb, f, (side == 0 ? out_left : out_right) + out_off, Ho, Wo, x, y);
}

__global__ void __launch_bounds__(256)
train_gt_kernel(const float* __restrict__ boxes_left, const float* __restrict__ boxes_right,
                const float* __restrict__ boxes_merge, const int* __restrict__ gt_classes,
                const float* __restrict__ dim_orien, const float* __restrict__ kpts, const int* __restrict__ n_rows,
                const unsigned* __restrict__ words, int N, float im_scale, int im_width, float* __restrict__ gt_left,
                float* __restrict__ gt_right, float* __restrict__ gt_merge, float* __restrict__ gt_dim_orien,
                float* __restrict__ gt_kpts, int* __restrict__ num_boxes) {
    __shared__ unsigned s_word[kMaxGtRows];
    __shared__ unsigned char s_valid[kMaxGtRows];
    __shared__ int s_count;
    const int b = blockIdx.x, t = threadIdx.x;
    const int n = min(max(n_rows[b], 0), N);
    boxes_left += (size_t)b * N * 4; boxes_right += (size_t)b * N * 4; boxes_merge += (size_t)b * N * 4;
    gt_classes += (size_t)b * N; dim_orien += (size_t)b * N * 4; kpts += (size_t)b * N * 6; words += (size_t)b * N;
    gt_left += b * kMaxNumGt * 5; gt_right += b * kMaxNumGt * 5; gt_merge += b * kMaxNumGt * 5;
    gt_dim_orien += b * kMaxNumGt * 5; gt_kpts += b * kMaxNumGt * 6;
    if (t == 0) s_count = 0;
    for (int i = t; i < kMaxNumGt * 5; i += 256) gt_left[i] = gt_right[i] = gt_merge[i] = gt_dim_orien[i] = 0.f;
    for (int i = t; i < kMaxNumGt * 6; i += 256) gt_kpts[i] = 0.f;
    for (int i = t; i < N; i += 256) {
        s_word[i] = words[i];
        s_valid[i] = i < n && gt_classes[i] != 0;                    // minibatch.py:43
    }
    __syncthreads();
    const float wmax = (float)im_width, kmax = (float)(im_width - 1);
    for (int i = t; i < N; i += 256) {
        if (!s_valid[i]) continue;
        atomicAdd(&s_count, 1);
        // position of row i in the order (word, row index) ascending over the kept rows: np.random.shuffle
        // (roibatchLoader.py:75) with the permutation given by explicit words, the rule of sb_proposal_targets
        const unsigned w = s_word[i];
        int r = 0;
        for (int j = 0; j < N; ++j) r += s_valid[j] && (s_word[j] < w || (s_word[j] == w && j < i));
        if (r >= kMaxNumGt) continue;                                // roibatchLoader.py:83
        const float cls = (float)gt_classes[i];
        const float* src[3] = {boxes_left, boxes_right, boxes_merge};
        float* dst[3] = {gt_left, gt_right, gt_merge};
#pragma unroll
        for (int k = 0; k < 3; ++k) {                                // minibatch.py:47-63: float32 array * scale
            float* o = dst[k] + r * 5;
            o[0] = fminf(__fmul_rn(src[k][i * 4 + 0], im_scale), wmax);
            o[1] = __fmul_rn(src[k][i * 4 + 1], im_scale);
            o[2] = __fmul_rn(src[k][i * 4 + 2], im_scale);
            o[3] = __fmul_rn(src[k][i * 4 + 3], im_scale);
            o[4] = cls;
        }
        float* d = gt_dim_orien + r * 5;                             // minibatch.py:65-69: math.sin of the float32
        d[0] = dim_orien[i * 4 + 0]; d[1] = dim_orien[i * 4 + 1]; d[2] = dim_orien[i * 4 + 2];
        const double th = (double)dim_orien[i * 4 + 3];
        d[3] = (float)sin(th);
        d[4] = (float)cos(th);
#pragma unroll
        for (int k = 0; k < 6; ++k) {                                // minibatch.py:71-76
            const float v = __fmul_rn(kpts[i * 6 + k], im_scale);
            gt_kpts[r * 6 + k] = (v < 0.f || v > kmax) ? -1.f : v;
        }
    }
    __syncthreads();
    if (t == 0) num_boxes[b] = min(s_count, kMaxNumGt);
}

// Philox4x32-10 (Salmon, Moraes, Dror, Shaw: "Parallel random numbers: as easy as 1, 2, 3", SC'11)
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int r = 0; r < 10; ++r) {
        const unsigned hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
        const unsigned hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
        c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
        k.x += 0x9E3779B9u;
        k.y += 0xBB67AE85u;
    }
    return c;
}

__global__ void __launch_bounds__(256)
random_words_kernel(unsigned long long seed, const unsigned long long* __restrict__ step, unsigned stream_id,
                    unsigned* __restrict__ out, size_t n, int aligned) {
    const unsigned long long s = *step;
    const uint2 key = make_uint2((unsigned)seed, (unsigned)(seed >> 32));
    const size_t groups = (n + 3) / 4;
    for (size_t g = (size_t)blockIdx.x * 256 + threadIdx.x; g < groups; g += (size_t)gridDim.x * 256) {
        const uint4 r = philox4x32_10(make_uint4((unsigned)g, stream_id, (unsigned)s, (unsigned)(s >> 32)), key);
        if (aligned && g * 4 + 4 <= n) {
            reinterpret_cast<uint4*>(out)[g] = r;
        } else {
            const unsigned v[4] = {r.x, r.y, r.z, r.w};
            for (int k = 0; k < 4 && g * 4 + k < n; ++k) out[g * 4 + k] = v[k];
        }
    }
}

__global__ void step_advance_kernel(unsigned long long* step) { *step += 1ULL; }

}  // namespace

extern "C" int sb_prep_stereo_pairs(const uint8_t* left, const uint8_t* right, int B, int H, int W, double scale,
                                    int rgb_input, const int* flip, float* out_left, float* out_right,
                                    sb_stream_t stream) {
    int Ho = 0, Wo = 0;
    if (!left || !right || !flip || !out_left || !out_right || B < 1 || B > kMaxPrepPairs ||
        sb_prep_image_size(H, W, scale, &Ho, &Wo) != SB_OK || Ho < 1 || Wo < 1)
        return SB_EINVAL;
    prep_stereo_pair_kernel<<<dim3(sb_div_up(Wo, 256), Ho, 2 * B), 256, 0, sb_cs(stream)>>>(
        left, right, H, W, 1.0 / scale, rgb_input, flip, out_left, out_right, Ho, Wo);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" int sb_prep_stereo_pair(const uint8_t* left, const uint8_t* right, int H, int W, double scale,
                                   int rgb_input, const int* flip, float* out_left, float* out_right,
                                   sb_stream_t stream) {
    return sb_prep_stereo_pairs(left, right, 1, H, W, scale, rgb_input, flip, out_left, out_right, stream);
}

extern "C" int sb_train_gt(const float* boxes_left, const float* boxes_right, const float* boxes_merge,
                           const int* gt_classes, const float* dim_orien, const float* kpts, const int* n_rows,
                           const unsigned* words, int B, int N, float im_scale, int im_width, float* gt_left,
                           float* gt_right, float* gt_merge, float* gt_dim_orien, float* gt_kpts, int* num_boxes,
                           sb_stream_t stream) {
    if (!boxes_left || !boxes_right || !boxes_merge || !gt_classes || !dim_orien || !kpts || !n_rows || !words ||
        !gt_left || !gt_right || !gt_merge || !gt_dim_orien || !gt_kpts || !num_boxes)
        return SB_EINVAL;
    if (B < 1 || N < 1 || N > kMaxGtRows || !(im_scale > 0.f) || !isfinite(im_scale) || im_width < 1) return SB_EINVAL;
    train_gt_kernel<<<B, 256, 0, sb_cs(stream)>>>(boxes_left, boxes_right, boxes_merge, gt_classes, dim_orien, kpts,
                                                  n_rows, words, N, im_scale, im_width, gt_left, gt_right, gt_merge,
                                                  gt_dim_orien, gt_kpts, num_boxes);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" int sb_random_words(unsigned long long seed, const unsigned long long* step, unsigned stream_id,
                               unsigned* out, size_t n, sb_stream_t stream) {
    if (!step || !out || n < 1) return SB_EINVAL;
    const size_t groups = (n + 3) / 4;
    const int blocks = (int)(groups < (size_t)(8 * 256 * 132) ? (groups + 255) / 256 : 8 * 132);
    random_words_kernel<<<blocks, 256, 0, sb_cs(stream)>>>(seed, step, stream_id, out, n,
                                                           ((uintptr_t)out & 15) == 0);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" int sb_step_advance(unsigned long long* step, sb_stream_t stream) {
    if (!step) return SB_EINVAL;
    step_advance_kernel<<<1, 1, 0, sb_cs(stream)>>>(step);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}
