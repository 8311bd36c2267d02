// proposal.cu -- the stereo RPN proposal layer, fully on device (sm_90a).
//
// Replaces lib/model/rpn/proposal_layer.py:42-145 (+ generate_anchors.py:112-173,
// bbox_transform.py:79-104,177-185, nms_wrapper/nms_gpu, np.intersect1d).
// Reference schedule: numpy anchors on the host every forward, ~20 elementwise kernels over
// all 298 476 anchors x 2 sides, torch.sort of everything, two synchronous NMS calls with
// a 4.5 MB mask read-back each, a CPU intersect1d round trip.
// This schedule (per image, no host sync, caller-owned workspace):
//   1. 3-pass radix select of the pre_nms_top_n-th largest score (11+11+10 bits)
//   2. ordered compaction of the survivors (ties broken by ascending anchor index --
//      the total order the oracle pins; the reference leaves ties to torch.sort)
//   3. rank sort of the <= 16384 unique (score, index) keys (K^2 compare-adds over K/64 CTAs)
//   4. anchors generated in fp64 *for survivors only* (bit-equal to the numpy table),
//      left/right decode + clip with the shared deterministic expf
//   5. upper-triangle bitmask NMS for both sides in one launch + lock-step greedy
//      reduction with on-the-fly intersection and early exit at post_nms_top_n
//   6. gather + zero padding into rois_left / rois_right
// Memory-bound: reads scores (A*8 B) 4x from L2, deltas only for survivors.
#include <climits>
#include <cuda_fp16.h>
#include "common.cuh"

int sb_nms_launch(const float* boxes0, const float* boxes1, int stride, int n, float thresh,
                  unsigned long long* mask0, unsigned long long* mask1, int max_out, int* keep,
                  int* num_out, cudaStream_t st);

namespace {

constexpr int kMaxLevels = 8;
constexpr int kMaxRatios = 4;
constexpr int kChunk = 2048;  // elements per block in the compaction kernels (256 thr x 8)

struct AnchorCfg {
    int n_levels, n_ratios;
    int start[kMaxLevels + 1];  // first anchor index of each level
    int width[kMaxLevels];
    int stride[kMaxLevels];
    double aw[kMaxLevels][kMaxRatios];  // scale * sqrt(ratio)
    double ah[kMaxLevels][kMaxRatios];  // scale / sqrt(ratio)
};

struct SelState {
    unsigned int prefix;  // high bits fixed so far
    int remaining;        // how many still to take from inside the prefix bucket
    int n_gt;             // (final) number of keys strictly greater than the threshold
    int gt_counter;       // running slot counter for > threshold
};

// inverse of sb_score_key (common.cuh) on the keys it returns: every NaN comes back as 0x7f800001, -0.0 as +0.0
__device__ __forceinline__ float key_to_float(unsigned int k) {
    unsigned int b = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    return __uint_as_float(b);
}

// scores[i] = cls_prob[i*2+1]
__global__ void __launch_bounds__(256)
select_hist_kernel(const float* __restrict__ prob, int A, int pass, const SelState* __restrict__ st,
                   int* __restrict__ hist) {
    __shared__ int sh[2048];
    for (int i = threadIdx.x; i < 2048; i += 256) sh[i] = 0;
    __syncthreads();
    const int shift = pass == 0 ? 21 : (pass == 1 ? 10 : 0);
    const int nbits = pass == 2 ? 10 : 11;
    const unsigned int prefix = st->prefix;
    for (int i = blockIdx.x * 256 + threadIdx.x; i < A; i += gridDim.x * 256) {
        unsigned int k = sb_score_key(prob[2 * (size_t)i + 1]);
        bool match = pass == 0 || (k >> (shift + nbits)) == prefix;
        if (match) atomicAdd(&sh[(k >> shift) & ((1u << nbits) - 1)], 1);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 2048; i += 256)
        if (sh[i]) atomicAdd(&hist[i], sh[i]);
}

// one warp: walk the histogram from the top bin down until `remaining` is covered
__global__ void select_scan_kernel(int* __restrict__ hist, int pass, SelState* __restrict__ st) {
    const int nb = pass == 2 ? 1024 : 2048;
    const int lane = threadIdx.x;
    const int seg = nb / 32;
    // lane 0 owns the TOP segment
    const int hi = nb - 1 - lane * seg;
    int sum = 0;
    for (int j = 0; j < seg; ++j) sum += hist[hi - j];
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int v = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += v;
    }
    const int excl = incl - sum;
    // lane 0 reads the state once and broadcasts it: the owning lane rewrites st->remaining / st->prefix below, and
    // under independent thread scheduling a late reader must not see the updated values
    int remaining = 0;
    unsigned prefix0 = 0;
    if (lane == 0) { remaining = st->remaining; prefix0 = st->prefix; }
    remaining = __shfl_sync(0xffffffffu, remaining, 0);
    prefix0 = __shfl_sync(0xffffffffu, prefix0, 0);
    const bool mine = excl < remaining && remaining <= incl;
    if (mine) {
        int acc = excl;
        int bin = hi;
        for (int j = 0; j < seg; ++j) {
            int h = hist[hi - j];
            if (acc + h >= remaining) { bin = hi - j; break; }
            acc += h;
        }
        const int nbits = pass == 2 ? 10 : 11;
        st->prefix = pass == 0 ? (unsigned)bin : ((prefix0 << nbits) | (unsigned)bin);
        st->remaining = remaining - acc;
        if (pass == 2) { st->n_gt = 0; }
    }
    __syncwarp();
    // reset the histogram for the next pass
    for (int j = lane; j < 2048; j += 32) hist[j] = 0;
}

__global__ void __launch_bounds__(256)
count_eq_kernel(const float* __restrict__ prob, int A, const SelState* __restrict__ st,
                int* __restrict__ block_eq, int* __restrict__ block_gt) {
    const unsigned int T = st->prefix;
    const int base = blockIdx.x * kChunk + threadIdx.x * 8;
    int ce = 0, cg = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        int i = base + j;
        if (i < A) {
            unsigned int k = sb_score_key(prob[2 * (size_t)i + 1]);
            ce += (k == T);
            cg += (k > T);
        }
    }
    __shared__ int se[8], sg[8];
    for (int o = 16; o > 0; o >>= 1) {
        ce += __shfl_xor_sync(0xffffffffu, ce, o);
        cg += __shfl_xor_sync(0xffffffffu, cg, o);
    }
    if ((threadIdx.x & 31) == 0) { se[threadIdx.x >> 5] = ce; sg[threadIdx.x >> 5] = cg; }
    __syncthreads();
    if (threadIdx.x == 0) {
        int a = 0, b = 0;
        for (int w = 0; w < 8; ++w) { a += se[w]; b += sg[w]; }
        block_eq[blockIdx.x] = a;
        block_gt[blockIdx.x] = b;
    }
}

// exclusive scan of the per-block counts (single CTA, nblocks <= 4096)
__global__ void __launch_bounds__(1024)
block_scan_kernel(int* __restrict__ block_eq, int* __restrict__ block_gt, int nblocks,
                  SelState* __restrict__ st) {
    __shared__ int buf[2][1024];
    __shared__ int carry[2];
    if (threadIdx.x < 2) carry[threadIdx.x] = 0;
    __syncthreads();
    for (int base = 0; base < nblocks; base += 1024) {
        int i = base + threadIdx.x;
        int ve = i < nblocks ? block_eq[i] : 0;
        int vg = i < nblocks ? block_gt[i] : 0;
        buf[0][threadIdx.x] = ve;
        buf[1][threadIdx.x] = vg;
        __syncthreads();
        for (int o = 1; o < 1024; o <<= 1) {
            int a = threadIdx.x >= o ? buf[0][threadIdx.x - o] : 0;
            int b = threadIdx.x >= o ? buf[1][threadIdx.x - o] : 0;
            __syncthreads();
            buf[0][threadIdx.x] += a;
            buf[1][threadIdx.x] += b;
            __syncthreads();
        }
        if (i < nblocks) {
            block_eq[i] = carry[0] + buf[0][threadIdx.x] - ve;
            block_gt[i] = carry[1] + buf[1][threadIdx.x] - vg;
        }
        __syncthreads();
        if (threadIdx.x == 1023) { carry[0] += buf[0][1023]; carry[1] += buf[1][1023]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) st->n_gt = carry[1];
}

// candidates: key64 = (ordered score << 32) | (0xFFFFFFFF - index): sorting descending gives
// score desc, index asc.
__global__ void __launch_bounds__(256)
compact_kernel(const float* __restrict__ prob, int A, const SelState* __restrict__ st,
               const int* __restrict__ block_eq, const int* __restrict__ block_gt,
               unsigned long long* __restrict__ cand, int K) {
    const unsigned int T = st->prefix;
    const int need_eq = st->remaining;
    const int n_gt = st->n_gt;
    const int base = blockIdx.x * kChunk + threadIdx.x * 8;
    unsigned int keys[8];
    int ce = 0, cg = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        int i = base + j;
        keys[j] = 0;
        if (i < A) {
            keys[j] = sb_score_key(prob[2 * (size_t)i + 1]);
            ce += (keys[j] == T);
            cg += (keys[j] > T);
        }
    }
    // block exclusive scan of (ce, cg) in thread order == index order
    __shared__ int we[8], wg[8];
    int ie = ce, ig = cg;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        int a = __shfl_up_sync(0xffffffffu, ie, o);
        int b = __shfl_up_sync(0xffffffffu, ig, o);
        if (lane >= o) { ie += a; ig += b; }
    }
    if (lane == 31) { we[warp] = ie; wg[warp] = ig; }
    __syncthreads();
    int oe = 0, og = 0;
    for (int w = 0; w < warp; ++w) { oe += we[w]; og += wg[w]; }
    int re = block_eq[blockIdx.x] + oe + ie - ce;  // rank among == T (index order)
    int rg = block_gt[blockIdx.x] + og + ig - cg;  // slot among  > T
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        int i = base + j;
        if (i >= A) break;
        unsigned long long k64 = ((unsigned long long)keys[j] << 32) | (unsigned long long)(0xFFFFFFFFu - (unsigned)i);
        if (keys[j] > T) {
            if (rg < K) cand[rg] = k64;
            ++rg;
        } else if (keys[j] == T) {
            if (re < need_eq && n_gt + re < K) cand[n_gt + re] = k64;
            ++re;
        }
    }
}

// Rank sort of the K unique 64-bit keys (descending): rank(i) = #{j : key_j > key_i}.  K^2 = 36 M
// compare-adds spread over ceil(K/64) CTAs replace the 91 barrier-separated steps of a single-CTA bitonic
// sort; keys are streamed through shared memory as broadcast reads.  Four threads share one key, each
// counting a quarter of every tile (the per-thread compare chain was the launch's whole latency: 54 us at
// K = 6000 with one thread per key), and their counts meet in shared memory.
__global__ void __launch_bounds__(256)
rank_sort_kernel(const unsigned long long* __restrict__ cand, int K, int* __restrict__ order,
                 float* __restrict__ score) {
    __shared__ unsigned long long tile[2048];
    __shared__ int part[4][64];
    const int kk = threadIdx.x & 63, q = threadIdx.x >> 6;
    const int i = blockIdx.x * 64 + kk;
    const unsigned long long my = i < K ? cand[i] : ~0ULL;
    int rank = 0;
    for (int base = 0; base < K; base += 2048) {
        const int cnt = min(2048, K - base);
        for (int j = threadIdx.x; j < 2048; j += 256) tile[j] = j < cnt ? cand[base + j] : 0ULL;   // 0 never outranks
        __syncthreads();
        const int j0 = q * 512;
#pragma unroll 16
        for (int j = 0; j < 512; ++j) rank += tile[j0 + j] > my;
        __syncthreads();
    }
    part[q][kk] = rank;
    __syncthreads();
    if (q == 0 && i < K) {
        rank = part[0][kk] + part[1][kk] + part[2][kk] + part[3][kk];
        order[rank] = (int)(0xFFFFFFFFu - (unsigned)(my & 0xFFFFFFFFu));
        score[rank] = key_to_float((unsigned)(my >> 32));
    }
}

__global__ void __launch_bounds__(256)
decode_kernel(const int* __restrict__ order, int K, const float* __restrict__ deltas /*[A,6]*/,
              const float* __restrict__ im_info /*[3]*/, AnchorCfg cfg,
              float4* __restrict__ prop_l, float4* __restrict__ prop_r) {
    int k = blockIdx.x * 256 + threadIdx.x;
    if (k >= K) return;
    const int idx = order[k];
    int l = 0;
    while (l + 1 < cfg.n_levels && idx >= cfg.start[l + 1]) ++l;
    const int r0 = idx - cfg.start[l];
    const int ratio = r0 % cfg.n_ratios;
    const int cell = r0 / cfg.n_ratios;
    const int x = cell % cfg.width[l], y = cell / cfg.width[l];
    // generate_anchors.py:131-154: fp64 centre -/+ 0.5*size, then .type_as(scores)
    const double cx = (double)x * cfg.stride[l], cy = (double)y * cfg.stride[l];
    const double hw = 0.5 * cfg.aw[l][ratio], hh = 0.5 * cfg.ah[l][ratio];
    float4 a = make_float4((float)(cx - hw), (float)(cy - hh), (float)(cx + hw), (float)(cy + hh));
    const float* d = deltas + (size_t)idx * 6;
    const float xmax = __fsub_rn(im_info[1], 1.0f), ymax = __fsub_rn(im_info[0], 1.0f);
    prop_l[k] = sb_decode_clip(a, d[0], d[1], d[2], d[3], xmax, ymax);
    prop_r[k] = sb_decode_clip(a, d[4], d[1], d[5], d[3], xmax, ymax);  // Q8
}

__global__ void __launch_bounds__(256)
write_rois_kernel(const float4* __restrict__ prop_l, const float4* __restrict__ prop_r,
                  const int* __restrict__ keep, const int* __restrict__ num, int post_n, float batch,
                  float* __restrict__ rois_l, float* __restrict__ rois_r) {
    int j = blockIdx.x * 256 + threadIdx.x;
    if (j >= post_n) return;
    float4 l = make_float4(0, 0, 0, 0), r = l;
    if (j < *num) { l = prop_l[keep[j]]; r = prop_r[keep[j]]; }
    float* o = rois_l + (size_t)j * 5;
    o[0] = batch; o[1] = l.x; o[2] = l.y; o[3] = l.z; o[4] = l.w;
    o = rois_r + (size_t)j * 5;
    o[0] = batch; o[1] = r.x; o[2] = r.y; o[3] = r.z; o[4] = r.w;
}

__global__ void init_state_kernel(SelState* st, int K, int* hist) {
    if (threadIdx.x == 0 && blockIdx.x == 0) { st->prefix = 0; st->remaining = K; st->n_gt = 0; st->gt_counter = 0; }
    for (int j = threadIdx.x; j < 2048; j += blockDim.x) hist[j] = 0;
}

// stereo_rpn.py:52-60,81-95: softmax over channel pairs (c, c+3), then NHWC flatten to
// [A,2] (channels 2a, 2a+1) and [A,6]
__global__ void __launch_bounds__(256)
rpn_head_epilogue_kernel(const float* __restrict__ head, long long total_pix, int ld,
                         float* __restrict__ cls_prob, float* __restrict__ bbox_pred) {
    long long p = (long long)blockIdx.x * 256 + threadIdx.x;
    if (p >= total_pix) return;
    const float* h = head + p * ld;
    float c[6], pr[6];
#pragma unroll
    for (int i = 0; i < 6; ++i) c[i] = h[i];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        float m = fmaxf(c[i], c[i + 3]);
        float ea = expf(c[i] - m), eb = expf(c[i + 3] - m);
        float s = ea + eb;
        pr[i] = ea / s;
        pr[i + 3] = eb / s;
    }
    float* cp = cls_prob + p * 6;
#pragma unroll
    for (int i = 0; i < 6; ++i) cp[i] = pr[i];
    float* bp = bbox_pred + p * 18;
#pragma unroll
    for (int i = 0; i < 18; ++i) bp[i] = h[6 + i];
}

// stereo_rpn.py:89,116-119: the raw class scores the RPN loss reads, each pixel's six channels as three consecutive
// pairs (c0,c1), (c2,c3), (c4,c5) -> rpn_cls_score [A,2]
__global__ void __launch_bounds__(256)
rpn_head_scores_kernel(const float* __restrict__ head, long long total_pix, int ld, float* __restrict__ score) {
    const long long e = (long long)blockIdx.x * 256 + threadIdx.x;
    if (e >= total_pix * 6) return;
    const long long p = e / 6;
    score[e] = head[p * ld + (e - p * 6)];
}

// backward of the fused head's outputs: dhead[p][0..5] = s * d_cls[p*6 ..], dhead[p][6..23] = s * d_box[p*18 ..],
// columns 24..63 zero (K padding of the head's data gradient and Cout padding of its weight gradient)
__global__ void __launch_bounds__(256)
rpn_head_grad_kernel(const float* __restrict__ d_cls, const float* __restrict__ d_box, long long total_pix,
                     float grad_scale, __half* __restrict__ dhead16, float* __restrict__ dhead32) {
    const long long e = (long long)blockIdx.x * 256 + threadIdx.x;
    if (e >= total_pix * 64) return;
    const long long p = e >> 6;
    const int c = (int)(e & 63);
    float v = 0.f;
    if (c < 6) v = grad_scale * __ldg(d_cls + p * 6 + c);
    else if (c < 24) v = grad_scale * __ldg(d_box + p * 18 + (c - 6));
    dhead16[e] = __float2half_rn(v);
    if (dhead32) dhead32[e] = v;
}

struct WsLayout {
    size_t state, hist, block_eq, block_gt, cand, order, score, prop_l, prop_r, mask0, mask1, keep, num, total;
};

WsLayout ws_layout(int A, int K) {
    WsLayout w;
    size_t off = 0;
    auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
    int nblocks = (A + kChunk - 1) / kChunk;
    int Kpad = 1; while (Kpad < K) Kpad <<= 1;
    size_t cb = (size_t)(K + 63) / 64;
    w.state = take(sizeof(SelState));
    w.hist = take(2048 * sizeof(int));
    w.block_eq = take((size_t)nblocks * sizeof(int));
    w.block_gt = take((size_t)nblocks * sizeof(int));
    w.cand = take((size_t)Kpad * 8);
    w.order = take((size_t)K * 4);
    w.score = take((size_t)K * 4);
    w.prop_l = take((size_t)K * 16);
    w.prop_r = take((size_t)K * 16);
    w.mask0 = take((size_t)K * cb * 8);
    w.mask1 = take((size_t)K * cb * 8);
    w.keep = take((size_t)K * 4);
    w.num = take(4);
    w.total = off;
    return w;
}

// generate_anchors.py:112-173 for every anchor of the pyramid (the train-time target layer needs the whole table; the
// proposal layer only decodes the survivors): fp64 centre -/+ 0.5 * size, cast to fp32 (`.type_as(scores)`)
__global__ void __launch_bounds__(256)
anchors_kernel(AnchorCfg cfg, int A, float4* __restrict__ out) {
    const int idx = blockIdx.x * 256 + threadIdx.x;
    if (idx >= A) return;
    int l = 0;
    while (l + 1 < cfg.n_levels && idx >= cfg.start[l + 1]) ++l;
    const int r0 = idx - cfg.start[l];
    const int ratio = r0 % cfg.n_ratios;
    const int cell = r0 / cfg.n_ratios;
    const int x = cell % cfg.width[l], y = cell / cfg.width[l];
    const double cx = (double)x * cfg.stride[l], cy = (double)y * cfg.stride[l];
    const double hw = 0.5 * cfg.aw[l][ratio], hh = 0.5 * cfg.ah[l][ratio];
    out[idx] = make_float4((float)(cx - hw), (float)(cy - hh), (float)(cx + hw), (float)(cy + hh));
}

// the pyramid fields of cfg: 1..8 levels, each with a positive shape, scale and stride, and 1..4 finite positive
// ratios, for at most INT_MAX anchors in all -> true when make_anchor_cfg may read them
bool anchor_cfg_ok(const sb_proposal_cfg* pc) {
    if (!pc || pc->n_levels < 1 || pc->n_levels > kMaxLevels || pc->n_ratios < 1 || pc->n_ratios > kMaxRatios)
        return false;
    for (int r = 0; r < pc->n_ratios; ++r)
        if (!(pc->ratios[r] > 0.0) || !isfinite(pc->ratios[r])) return false;
    long long tot = 0;
    for (int l = 0; l < pc->n_levels; ++l) {
        if (pc->shapes[l][0] < 1 || pc->shapes[l][1] < 1 || pc->anchor_scales[l] < 1 || pc->feat_strides[l] < 1)
            return false;
        const long long cells = (long long)pc->shapes[l][0] * pc->shapes[l][1];
        if (cells > INT_MAX) return false;
        tot += cells * pc->n_ratios;
        if (tot > INT_MAX) return false;
    }
    return true;
}

int make_anchor_cfg(const sb_proposal_cfg* pc, AnchorCfg* ac) {
    ac->n_levels = pc->n_levels;
    ac->n_ratios = pc->n_ratios;
    int tot = 0;
    for (int l = 0; l < pc->n_levels; ++l) {
        ac->start[l] = tot;
        ac->width[l] = pc->shapes[l][1];
        ac->stride[l] = pc->feat_strides[l];
        tot += pc->shapes[l][0] * pc->shapes[l][1] * pc->n_ratios;
        for (int r = 0; r < pc->n_ratios; ++r) {
            // generate_anchors.py:122-128: heights = scales / sqrt(ratios), widths = scales * sqrt(ratios)
            ac->aw[l][r] = (double)pc->anchor_scales[l] * sqrt(pc->ratios[r]);
            ac->ah[l][r] = (double)pc->anchor_scales[l] / sqrt(pc->ratios[r]);
        }
    }
    ac->start[pc->n_levels] = tot;
    return tot;
}

}  // namespace

extern "C" int sb_generate_anchors(const sb_proposal_cfg* pc, int A, float* anchors, sb_stream_t stream) {
    if (!anchor_cfg_ok(pc) || !anchors || (reinterpret_cast<uintptr_t>(anchors) & 15)) return SB_EINVAL;
    AnchorCfg ac;
    if (make_anchor_cfg(pc, &ac) != A) return SB_EINVAL;
    anchors_kernel<<<sb_div_up(A, 256), 256, 0, sb_cs(stream)>>>(ac, A, reinterpret_cast<float4*>(anchors));
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" size_t sb_proposal_workspace_bytes(int B, int A, int pre_nms_top_n) {
    (void)B;
    int K = (pre_nms_top_n > 0 && pre_nms_top_n < A) ? pre_nms_top_n : A;
    return ws_layout(A, K).total;
}

extern "C" int sb_proposal_layer(const float* cls_prob, const float* bbox_pred_lr, const float* im_info,
                                 int B, int A, const sb_proposal_cfg* pc, float* rois_left,
                                 float* rois_right, void* workspace, size_t workspace_bytes,
                                 sb_stream_t stream) {
    // post_nms_top_n sizes the caller's RoI buffers, so it must be positive (the reference allocates that many rows)
    if (!anchor_cfg_ok(pc) || !isfinite(pc->nms_thresh) || pc->post_nms_top_n < 1 || B < 0) return SB_EINVAL;
    if (B > 0 && (!cls_prob || !bbox_pred_lr || !im_info || !rois_left || !rois_right)) return SB_EINVAL;
    AnchorCfg ac;
    if (make_anchor_cfg(pc, &ac) != A) return SB_EINVAL;
    const int K = (pc->pre_nms_top_n > 0 && pc->pre_nms_top_n < A) ? pc->pre_nms_top_n : A;
    const int post_n = pc->post_nms_top_n;
    if (K > 16384 || A > kChunk * 4096) return SB_EINVAL;
    WsLayout w = ws_layout(A, K);
    if (workspace_bytes < w.total || !workspace) return SB_EINVAL;
    char* ws = (char*)workspace;
    cudaStream_t st = sb_cs(stream);
    SelState* state = (SelState*)(ws + w.state);
    int* hist = (int*)(ws + w.hist);
    int* block_eq = (int*)(ws + w.block_eq);
    int* block_gt = (int*)(ws + w.block_gt);
    unsigned long long* cand = (unsigned long long*)(ws + w.cand);
    int* order = (int*)(ws + w.order);
    float* score = (float*)(ws + w.score);
    float4* prop_l = (float4*)(ws + w.prop_l);
    float4* prop_r = (float4*)(ws + w.prop_r);
    unsigned long long* mask0 = (unsigned long long*)(ws + w.mask0);
    unsigned long long* mask1 = (unsigned long long*)(ws + w.mask1);
    int* keep = (int*)(ws + w.keep);
    int* num = (int*)(ws + w.num);
    const int nblocks = (A + kChunk - 1) / kChunk;
    int Kpad = 1; while (Kpad < K) Kpad <<= 1;
    for (int b = 0; b < B; ++b) {
        const float* prob = cls_prob + (size_t)b * A * 2;
        const float* deltas = bbox_pred_lr + (size_t)b * A * 6;
        init_state_kernel<<<1, 256, 0, st>>>(state, K, hist); SB_LAUNCHED();
        const int hb = min(148 * 4, (A + 255) / 256);
        for (int pass = 0; pass < 3; ++pass) {
            select_hist_kernel<<<hb, 256, 0, st>>>(prob, A, pass, state, hist); SB_LAUNCHED();
            select_scan_kernel<<<1, 32, 0, st>>>(hist, pass, state); SB_LAUNCHED();
        }
        count_eq_kernel<<<nblocks, 256, 0, st>>>(prob, A, state, block_eq, block_gt); SB_LAUNCHED();
        block_scan_kernel<<<1, 1024, 0, st>>>(block_eq, block_gt, nblocks, state); SB_LAUNCHED();
        compact_kernel<<<nblocks, 256, 0, st>>>(prob, A, state, block_eq, block_gt, cand, K); SB_LAUNCHED();
        rank_sort_kernel<<<(K + 63) / 64, 256, 0, st>>>(cand, K, order, score); SB_LAUNCHED();
        decode_kernel<<<(K + 255) / 256, 256, 0, st>>>(order, K, deltas, im_info + 3 * b, ac, prop_l, prop_r);
        SB_LAUNCHED();
        SB_CHECK_LAUNCH();
        int rc = sb_nms_launch((const float*)prop_l, (const float*)prop_r, 4, K, pc->nms_thresh, mask0, mask1,
                               post_n, keep, num, st);
        if (rc) return rc;
        write_rois_kernel<<<(post_n + 255) / 256, 256, 0, st>>>(prop_l, prop_r, keep, num, post_n, (float)b,
                                                              rois_left + (size_t)b * post_n * 5,
                                                              rois_right + (size_t)b * post_n * 5);
        SB_LAUNCHED();
        SB_CHECK_LAUNCH();
    }
    return SB_OK;
}

extern "C" int sb_rpn_head_epilogue(const float* head, int B, int P, int ld, float* cls_prob,
                                    float* bbox_pred, sb_stream_t stream) {
    long long total = (long long)B * P;
    if (total <= 0) return total == 0 ? SB_OK : SB_EINVAL;
    rpn_head_epilogue_kernel<<<sb_div_up(total, 256), 256, 0, sb_cs(stream)>>>(head, total, ld, cls_prob, bbox_pred);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" int sb_rpn_head_scores(const float* head, int B, int P, int ld, float* rpn_cls_score, sb_stream_t stream) {
    const long long total = (long long)B * P;
    if (B < 0 || P < 0 || ld < 6 || (total > 0 && (!head || !rpn_cls_score))) return SB_EINVAL;
    if (total == 0) return SB_OK;
    rpn_head_scores_kernel<<<sb_div_up(total * 6, 256), 256, 0, sb_cs(stream)>>>(head, total, ld, rpn_cls_score);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" int sb_rpn_head_grad(const float* d_cls_score, const float* d_bbox_pred, int B, int P, float grad_scale,
                                void* dhead16, float* dhead32, sb_stream_t stream) {
    const long long total = (long long)B * P;
    if (B < 0 || P < 0 || (total > 0 && (!d_cls_score || !d_bbox_pred || !dhead16))) return SB_EINVAL;
    if ((reinterpret_cast<uintptr_t>(dhead16) & 1) || (reinterpret_cast<uintptr_t>(dhead32) & 3)) return SB_EINVAL;
    if (total == 0) return SB_OK;
    rpn_head_grad_kernel<<<sb_div_up(total * 64, 256), 256, 0, sb_cs(stream)>>>(
        d_cls_score, d_bbox_pred, total, grad_scale, reinterpret_cast<__half*>(dhead16), dhead32);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}
