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
//     sb_conv2d_tc_rows runs fp16 3x3 convs on flat tiles of 128 consecutive output pixels instead: a TMA im2col map
//     loads them shifted by the tap (zero-filled halo at every row and image edge, inside a tile too), so no MMA row
//     is spent on pixels past the edge of a map; the shared-memory tile is that of a 1x1 conv's flat rows.
//     The stem variant builds its A tile in the kernel instead (patch gather warps, see below).
//   * warp-specialised persistent CTAs (one per SM): warps 0..7 are two consumer warpgroups -- each issues the
//     m64nNk16 (k8 for tf32) wgmma of 64 of the tile's 128 rows and owns their fp32 accumulators -- and warp 8 is
//     the TMA producer.  One mbarrier ring (full / empty) of stages sized so that nearly all shared memory holds
//     operands (4 stages of 48 KB for 256-wide tiles, 6 of 32 KB for 128-wide ones); the producer runs ahead into
//     the next tile while the consumers finish the epilogue of the current one.
//   * ping-pong schedule (fp16 operands, no residual, tiles of at most 128 columns -- 64 with the upsample-add or an fp32 TMA box
//     -- and a launch where some CTA gets a second tile): the CTA's j-th tile belongs to warpgroup j & 1, which
//     issues two m64nNk16 wgmma per k16 (one per 64-row half of the A stage) and owns all 128 rows' accumulators.  The mainloops take turns (a pair of
//     mbarriers: a warpgroup starts a tile once the other has issued its previous tile's last K-step), so each
//     tile's register epilogue runs under the other warpgroup's MMAs.  Each stage is consumed by one warpgroup; it
//     finds the ring position of its tile from the K-steps before it, j * num_k_blocks.  Every output element sums
//     the same K-steps in the same order as under the cooperative schedule, so the results are bit-identical.
//   * fused epilogue straight out of the accumulator registers: folded frozen-BN scale/shift or bias, residual add,
//     FPN bilinear (align_corners) upsample-add, ReLU, the TF32 store modes, fp32 and/or fp16 ("twin") stores with
//     arbitrary n/h/w strides and channel offset (RPN L|R concat, deconv scatter).  All loads of a column step (both
//     rows: residual, the four upsample taps, scale / shift) are issued before its first store.
//   * residual epilogue by TMA (fp16 operands, forward: conv3 of every bottleneck, HBM-bound): per consumer warpgroup
//     a ring of slots with its own full / empty mbarriers, each slot one 32-column chunk of the warpgroup's 64 rows --
//     an fp32 box of 64 x 32 (residual in, result out in place, 128-byte swizzle) and an fp16 box of 64 x 32 (the
//     twin, 64-byte swizzle).  Warps 9 and 10 are the residual producers of the two warpgroups: each loads its
//     warpgroup's chunks in (tile, chunk) order as soon as a slot is empty, so the next tile's residual streams in
//     under this tile's last chunks and the next main loop; the operand producer never waits on the ring.  Per chunk
//     the consumers add the accumulators in place, write the twin, fence the async proxy and sync the warpgroup
//     (named barrier); one thread issues the chunk's bulk tensor stores as one group and returns the previous chunk's
//     slot once its group has read it (cp.async.bulk.wait_group.read 1; the last chunk of a tile is returned under
//     the next tile's first MMAs).  Both sides step through every chunk of every tile, stored or not (rows past M,
//     columns past Cout, a warpgroup without rows in the last tile).  Shared memory of a 128-wide residual tile: 4
//     operand stages of 32 KB + 2 warpgroups x 4 slots x 12 KB = 96 KB of rings (64-wide: 6 x 24 KB + 2 x 3 x 12 KB;
//     32-wide: 7 x 20 KB + 2 x 3 x 12 KB).  The TF32 mode and the data-gradient variants keep the register epilogue.
//   * plain outputs by TMA (fp16 operands, forward, no residual or upsample-add, flat output rows that a 2-D [ld, M]
//     map expresses): the same per-warpgroup rings without the residual producers -- the consumers take a slot once
//     the stores of its previous entry have read it.  Slots hold both boxes when the conv writes fp32 (kEpiTma) and
//     the fp16 box alone otherwise (kEpiTma16, 4 KB: 4 slots per warpgroup beside the register variants' stages).  A
//     ping-pong warpgroup streams its 128 rows as two 64-row entries per chunk.
//   * programmatic dependent launch: the prologue (barrier init, descriptor prefetch) overlaps the previous
//     kernel's tail; dependents are released after the CTA's last operand loads are issued.
//   * optional per-CTA phase trace (sb_conv_trace) for tools/conv_trace.py: timestamps, the schedule and the tiles
//     each consumer warpgroup computed.
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdlib.h>
#include <string.h>

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
    int rows;             // 1 (patch 0): 3x3 / pad 1 on flat rows of 128 output pixels, A by TMA im2col
    long long M;
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
// Trace words of a CTA: [0..5] %globaltimer and [8..13] clock64 at entry, after griddepcontrol.wait, first operand
// stage landed, last operand load issued, first tile's epilogue done, exit; [6] SM id; [7] schedule (0 cooperative,
// 1 ping-pong); [14 + g] tiles computed by consumer warpgroup g (counted once per tile, outside the K loop).
constexpr int kTraceWords = 16, kTraceCtas = 304;
constexpr int kTraceSched = 7, kTraceTiles = 14;

// TMA residual epilogue (fp16-operand forward with a residual): per consumer warpgroup, a ring of epi_slots(BLOCK_N)
// slots, each one 32-column chunk of the warpgroup's 64 tile rows: an fp32 box [64 rows][32 columns] (residual in,
// fp32 result out, in place; 128-byte rows, 128-byte swizzle) and an fp16 box [64 rows][32 columns] (the twin; 64-byte
// rows, 64-byte swizzle).  Warps 9 and 10 are the residual producers of warpgroups 0 and 1.
// The plain TMA epilogue (fp16-operand forward without a residual, flat output rows) uses the same rings without the
// residual producers: the consumers own the slots.  Its slots hold both boxes when the conv writes an fp32 output
// (kEpiTma) and the fp16 box alone when it writes the twin only (kEpiTma16: 4 KB slots, so 4 per warpgroup fit beside
// the register-epilogue instantiations' operand stages).
constexpr uint32_t kEpiBox = 64 * 128, kTwinBox = 64 * 64, kSlotBytes = kEpiBox + kTwinBox;
enum : int { kEpiRegs = 0, kEpiTma = 1, kEpiTma16 = 2 };
constexpr int kResProducerWarps = 2;
constexpr int kResThreads = kThreads + 32 * kResProducerWarps;
constexpr uint32_t epi_slot_bytes(int epi) { return epi == kEpiTma16 ? kTwinBox : kSlotBytes; }
constexpr int epi_slots(int block_n, int epi) { return epi == kEpiRegs ? 0 : (epi == kEpiTma16 || block_n == 128) ? 4 : 3; }
constexpr bool res_ring(bool has_res, int epi) { return has_res && epi != kEpiRegs; }    // residual producer warps
constexpr int conv_threads(bool stem, bool res_producers) { return stem ? kStemThreads : res_producers ? kResThreads : kThreads; }
// instantiations that have a ping-pong twin: fp16 operands, no residual (its ring has one producer per 64-row
// warpgroup half), and a warpgroup's 128 x BLOCK_N accumulators and its epilogue state fit the register budget without
// spills -- 168 per thread at 288 threads and one CTA per SM (nine warps on four 16K-register SM sub-partitions).  At
// 128 columns the upsample-add epilogue does not (2.4 KB of spill stores), nor does the TMA epilogue with an fp32 box
// (4-24 bytes, however its ring counters are kept), so those stay cooperative.
constexpr bool pingpong_ok(int block_n, bool has_res, bool has_up, bool in16, bool stem, bool mask, int epi) {
    return in16 && !has_res && !stem && !mask && block_n <= (has_up || epi == kEpiTma ? 64 : 128);
}

// operand stages, then (slots > 0) both warpgroups' epilogue rings, the 1024-byte alignment pad and the mbarriers
// (operand ring, epilogue rings, the residual producers' start, the two ping-pong turns)
constexpr size_t conv_smem(int block_n, int stages, int slots, uint32_t slot_bytes) {
    return (size_t)stages * (BLOCK_M * kRowBytes + block_n * kRowBytes) + (size_t)2 * slots * slot_bytes + 1024 +
           (2 * stages + 4 * slots + 3) * 8;
}

// EPI: kEpiRegs (epilogue from registers), kEpiTma or kEpiTma16 (through the per-warpgroup rings, stored by TMA)
template <int BLOCK_N, int kStages, bool HAS_RES, bool HAS_UP, bool IN16, bool STEM = false, bool MASK = false,
          bool PP = false, int EPI = kEpiRegs>
__global__ void __launch_bounds__(conv_threads(STEM, res_ring(HAS_RES, EPI)), 1)
conv_tc_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
               const __grid_constant__ CUtensorMap map_r, const __grid_constant__ CUtensorMap map_o,
               const __grid_constant__ CUtensorMap map_o16, const TcParams p) {
    static_assert(!STEM || (IN16 && !HAS_RES && !HAS_UP), "stem variant");
    static_assert(!MASK || (IN16 && !HAS_UP && !STEM), "mask variant");
    static_assert(!PP || pingpong_ok(BLOCK_N, HAS_RES, HAS_UP, IN16, STEM, MASK, EPI), "ping-pong variant");
    static_assert(EPI == kEpiRegs || (IN16 && !STEM && !MASK && !HAS_UP), "TMA epilogue: fp16-operand forward");
    static_assert(!HAS_RES || !IN16 || MASK || EPI == kEpiTma, "the fp16 forward residual runs through the ring");
    constexpr bool kTmaEpi = EPI != kEpiRegs;
    constexpr bool kResRing = res_ring(HAS_RES, EPI);
    static_assert(!kResRing || BLOCK_N <= 128, "residual layers use tiles of at most 128 columns");
    constexpr uint32_t kABytes = BLOCK_M * kRowBytes, kBBytes = BLOCK_N * kRowBytes;
    constexpr int BLOCK_K = IN16 ? 64 : 32;     // elements per K-step
    constexpr uint32_t kStageBytes = kABytes + kBBytes;
    constexpr int kSlots = epi_slots(BLOCK_N, EPI);              // epilogue ring slots per consumer warpgroup
    constexpr uint32_t kSlotB = epi_slot_bytes(EPI), kTwinOff = EPI == kEpiTma16 ? 0 : kEpiBox;
    constexpr int kChunks = BLOCK_N / 32;                        // 32-column chunks per tile
    // a chunk's slot is released while the next chunk is processed, so a second slot must be free to fill
    static_assert(!kTmaEpi || kSlots >= 2, "epilogue ring of at least two slots");
    extern __shared__ uint8_t smem_raw[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
    uint8_t* epi = smem + kStages * kStageBytes;                  // [2 warpgroups][kSlots][kSlotB]
    uint64_t* full = reinterpret_cast<uint64_t*>(epi + 2 * kSlots * kSlotB);
    uint64_t* empty = full + kStages;
    uint64_t* slot_full = empty + kStages;         // [2][kSlots]: the chunk's residual box has landed
    uint64_t* slot_empty = slot_full + 2 * kSlots; // [2][kSlots]: the output stores of the slot's last chunk have read it
    uint64_t* res_go = slot_empty + 2 * kSlots;    // the first tile's first operand loads are issued
    uint64_t* turn = res_go + 1;                   // [2] (PP): warpgroup g may start its next tile's K loop

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const sb_conv_desc& d = p.d;
    unsigned long long* tr = p.trace ? p.trace + (size_t)blockIdx.x * kTraceWords : nullptr;
    if (tr && threadIdx.x == 0) {
        unsigned smid;
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        tr[0] = gtimer(); tr[8] = clock64(); tr[6] = smid;
        tr[kTraceSched] = PP ? 1 : 0;
        tr[kTraceTiles] = tr[kTraceTiles + 1] = 0;     // counted below by the warpgroups' thread 0
    }
    if (warp == kProducerWarp && lane == 0) {
        if (!STEM) prefetch_tmap(&map_a);
        prefetch_tmap(&map_b);
        if (kResRing) prefetch_tmap(&map_r);
        // STEM: a stage is full when the weight tile has landed (1 expect_tx arrival) and the gather threads have
        // written their patch rows.  A stage is empty when the MMAs on it of every consumer warp that reads it
        // (all eight; PP: the four of the tile's warpgroup) have completed.
        for (int i = 0; i < kStages; ++i) {
            mbar_init(&full[i], STEM ? 1 + 32 * kStemGatherWarps : 1);
            mbar_init(&empty[i], PP ? kConsumerWarps / 2 : kConsumerWarps);
        }
        if (PP) {
            mbar_init(&turn[0], kConsumerWarps / 2);     // lane 0 of each warp of the other warpgroup
            mbar_init(&turn[1], kConsumerWarps / 2);
        }
        for (int i = 0; i < 2 * kSlots; ++i) {
            mbar_init(&slot_full[i], 1);         // the residual producer's expect_tx arrival
            mbar_init(&slot_empty[i], 1);        // the warpgroup's store thread
        }
        if (kResRing) mbar_init(res_go, 1);
        fence_barrier_init();
    }
    __syncthreads();
    // Programmatic dependent launch: everything above (barrier init, descriptor prefetch) overlapped the previous
    // kernel's tail.  Wait for the producers of our activations; the producer warp releases the next kernel below.
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
                } else if (!STEM && p.rows) {      // the tile's first output pixel
                    const unsigned m0 = (unsigned)mt * BLOCK_M, hw = (unsigned)(d.Ho * d.Wo);
                    n_img = (int)(m0 / hw);
                    const unsigned rem = m0 - (unsigned)n_img * hw;
                    h0 = (int)(rem / (unsigned)d.Wo);
                    w0 = (int)(rem - (unsigned)h0 * (unsigned)d.Wo);
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
                        } else if (p.rows) {
                            // the bounding box holds the taps' origins (output pixel - pad); each tap is an offset
                            const int r = tap / d.kw, s = tap - r * d.kw;
                            tma_load_im2col_4d(&map_a, &full[stage], sa, c0, w0 - d.pad, h0 - d.pad, n_img,
                                               (uint16_t)s, (uint16_t)r);
                        } else {
                            tma_load_2d(&map_a, &full[stage], sa, c0, mt * BLOCK_M);
                        }
                    }
                    tma_load_2d(&map_b, &full[stage], sa + kABytes, tap * d.Cin + c0, nt * BLOCK_N);
                    if (++stage == kStages) { stage = 0; phase ^= 1; }
                    // the residual producers start once the first tile's first min(K-steps, stages) operand loads
                    // are issued: with the residual loads issued alongside, the first operand stage landed ~10 k
                    // cycles after griddepcontrol.wait instead of ~3 k (H100, layers 1-4 conv3)
                    if (kResRing && tile == (int)blockIdx.x && kb == min(p.num_k_blocks, kStages) - 1) mbar_arrive(res_go);
                }
            }
            // release the dependent launch once this CTA's last operand loads are issued: an earlier release lets the
            // next kernel's CTAs sit in griddepcontrol.wait on SMs the other stream's chain could be using
            asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
            if (tr) { tr[3] = gtimer(); tr[11] = clock64(); }
        }
    } else if (kResRing && warp > kProducerWarp) {
        // ===================== residual producer of warpgroup g (warps 9, 10) =====================
        // Loads the warpgroup's residual chunks in (tile, chunk) order into its ring as soon as a slot is empty, so
        // the next tile's chunks stream in under this tile's last chunks and the next main loop.  Every chunk of
        // every tile is loaded, also rows past M and columns past Cout (zero-filled, still counted in the bytes), so
        // that both sides step through the ring alike.
        if (lane == 0) {
            const int g = warp - kProducerWarp - 1;
            int slot = 0;
            uint32_t sphase = 0;
            mbar_wait(res_go, 0);
            for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
                const int mt = tile / p.num_n_tiles, nt = tile - mt * p.num_n_tiles;
                for (int c = 0; c < kChunks; ++c) {
                    uint64_t* bar = &slot_full[g * kSlots + slot];
                    mbar_wait(&slot_empty[g * kSlots + slot], sphase ^ 1);
                    mbar_expect_tx(bar, kEpiBox);
                    tma_load_2d(&map_r, bar, epi + (g * kSlots + slot) * kSlotB, nt * BLOCK_N + 32 * c,
                                mt * BLOCK_M + 64 * g);
                    if (++slot == kSlots) { slot = 0; sphase ^= 1; }
                }
            }
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
        // Cooperative: warpgroup wg computes rows 64*wg .. 64*wg+63 of every tile against all BLOCK_N columns; this
        // thread holds rows r_lo and r_lo + 8, columns 8*j + cq + {0,1} for j < BLOCK_N/8 (wgmma.cuh: fragment
        // layout).  PP: warpgroup wg computes all 128 rows of the CTA's tiles j = wg, wg + 2, ..., as two 64-row
        // halves; this thread holds rows r_lo, r_lo + 8, r_lo + 64 and r_lo + 72 (accumulators of the second half at
        // kAcc + ...).
        const int wg = warp >> 2;
        constexpr int kHalves = PP ? 2 : 1;
        constexpr int kRows = 2 * kHalves;
        const int r_lo = (PP ? 0 : 64 * wg) + 16 * (warp & 3) + (lane >> 2);
        const int cq = 2 * (lane & 3);
        constexpr int kAcc = BLOCK_N / 2;      // per 64-row half
        float acc[kHalves * kAcc];
#pragma unroll
        for (int i = 0; i < kHalves * kAcc; ++i) acc[i] = 0.f;
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
        // epilogue ring (kTmaEpi): the next slot and its phase, and the slot of the previous tile's last chunk, whose
        // stores may still be reading it (-1: none)
        int slot = 0, held = -1;
        uint32_t sphase = 0;
        const bool store_thread = (threadIdx.x & 127) == 0;
        // the CTA's jt-th tile (PP: jt = wg, wg + 2, ...)
        for (int tile = blockIdx.x + (PP ? wg * (int)gridDim.x : 0), jt = PP ? wg : 0; tile < num_tiles;
             tile += (PP ? 2 : 1) * gridDim.x, jt += PP ? 2 : 1) {
            const int mt = tile / p.num_n_tiles, nt = tile - mt * p.num_n_tiles;
            if (PP) {
                // ring position of the tile's first K-step: the tiles before it took jt * num_k_blocks stages, the
                // last of them by the other warpgroup (num_k_blocks need not divide kStages)
                const unsigned ks = (unsigned)jt * (unsigned)p.num_k_blocks;
                stage = (int)(ks % kStages);
                phase = (ks / kStages) & 1u;
                // wait for the turn: the other warpgroup has issued tile jt - 1's last K-step, so every K-step before
                // this tile has landed (no `full` wait below is a phase behind) and the two mainloops alternate
                if (jt > 0) mbar_wait(&turn[wg], ((unsigned)(jt - 1) >> 1) & 1u);
            }
            int prev = 0;
            for (int kb = 0; kb < p.num_k_blocks; ++kb) {
                mbar_wait(&full[stage], phase);
                if (tr && threadIdx.x == 0 && kb == 0 && tile == (int)blockIdx.x) { tr[2] = gtimer(); tr[10] = clock64(); }
                const uint32_t sa = smem_u32(smem + stage * kStageBytes);
                const uint64_t db = make_smem_desc(sa + kABytes);
#pragma unroll
                for (int i = 0; i < kHalves * kAcc; ++i) reg_fence(acc[i]);
                wgmma_fence();
#pragma unroll
                for (int k = 0; k < 4; ++k) {  // advance 32 bytes (16 fp16 / 8 tf32) inside the 128-byte swizzle row
#pragma unroll
                    for (int hf = 0; hf < kHalves; ++hf) {
                        const uint64_t da = make_smem_desc(sa + (PP ? hf : wg) * (kABytes / 2));
                        Wgmma<BLOCK_N, IN16>::mma(acc + hf * kAcc, da + (uint64_t)(k * 2), db + (uint64_t)(k * 2),
                                                  (kb | k) != 0);
                    }
                }
                wgmma_commit();
#pragma unroll
                for (int i = 0; i < kHalves * kAcc; ++i) reg_fence(acc[i]);
                if (PP && kb == p.num_k_blocks - 1 && lane == 0) mbar_arrive(&turn[wg ^ 1]);     // pass the turn
                // keep one K-step of MMAs in flight: the previous step's are complete, its stage may be refilled
                wgmma_wait<1>();
                if (kb > 0 && lane == 0) mbar_arrive(&empty[prev]);
                prev = stage;
                if (++stage == kStages) { stage = 0; phase ^= 1; }
                if (kTmaEpi && held >= 0) {
                    // the previous tile's last chunk, stored at the end of its epilogue, is released here, under
                    // this tile's first MMAs, instead of stalling that epilogue on its read
                    if (store_thread) {
                        bulk_wait_read<0>();
                        mbar_arrive(&slot_empty[wg * kSlots + held]);
                    }
                    held = -1;
                }
            }
            wgmma_wait<0>();
#pragma unroll
            for (int i = 0; i < kHalves * kAcc; ++i) reg_fence(acc[i]);
            if (lane == 0) mbar_arrive(&empty[prev]);

            if constexpr (kTmaEpi) {
                // ---- TMA epilogue through the warpgroup's ring, one box of 64 rows x 32 columns per ring entry: a
                // cooperative warpgroup streams its 64 rows chunk by chunk, a ping-pong warpgroup all 128 rows as two
                // 64-row entries per chunk (the slots, tensor maps and ring accounting stay those of the 64-row
                // residual ring).  With a residual, its producer has loaded the entry's residual rows into the slot's
                // fp32 box and every thread adds its accumulator pairs to them in place; without, the slot is taken
                // once the stores of its previous entry have read it.  Every thread writes its values (and the fp16
                // twin) into the slot, then one thread stores the boxes by TMA (rows past M and columns past Cout
                // are clipped) as one bulk group.  The slot of the entry before is handed back once its group has
                // read it, so the warpgroup goes straight on to the next entry and the global writes drain under the
                // next entries and the next tile's MMAs.
                const int rl = 16 * (warp & 3) + (lane >> 2);     // rows rl and rl + 8 of the entry's 64
#pragma unroll
                for (int e = 0; e < kChunks * kHalves; ++e) {
                    const int ch = e / kHalves, hf = e % kHalves;
                    const int row0 = mt * BLOCK_M + 64 * (PP ? hf : wg);
                    const uint32_t rbuf = smem_u32(epi) + (wg * kSlots + slot) * kSlotB, tbuf = rbuf + kTwinOff;
                    if (kResRing) mbar_wait(&slot_full[wg * kSlots + slot], sphase);
                    else mbar_wait(&slot_empty[wg * kSlots + slot], sphase ^ 1);
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) {
                        const int j = 4 * ch + jj;
                        const int cl = 8 * j + cq;                // column in the tile
                        const int c = nt * BLOCK_N + cl;
                        const int cs = c < d.Cout ? c : 0;        // past Cout: any in-bounds column, never stored
                        const float2 sc = d.scale ? __ldg(reinterpret_cast<const float2*>(d.scale + cs)) : make_float2(1.f, 1.f);
                        const float2 sh = d.shift ? __ldg(reinterpret_cast<const float2*>(d.shift + cs)) : make_float2(0.f, 0.f);
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const uint32_t row = (uint32_t)(rl + 8 * h);
                            const uint32_t ra = rbuf + swz128(row * 128 + (cl & 31) * 4);
                            const int ai = hf * kAcc + 4 * j + 2 * h;
                            float x0 = fmaf(acc[ai], sc.x, sh.x);
                            float x1 = fmaf(acc[ai + 1], sc.y, sh.y);
                            if (kResRing) {
                                float2 r = lds64f(ra);
                                if (res_biased) { r.x = sb_unbias_tf32(r.x); r.y = sb_unbias_tf32(r.y); }
                                x0 += r.x; x1 += r.y;
                            }
                            if (relu) { x0 = fmaxf(x0, 0.f); x1 = fmaxf(x1, 0.f); }
                            if (out_mode == 1) { x0 = sb_round_tf32(x0); x1 = sb_round_tf32(x1); }
                            else if (out_mode == 2) { x0 = sb_bias_tf32(x0); x1 = sb_bias_tf32(x1); }
                            if (EPI == kEpiTma) sts64f(ra, x0, x1);
                            if (d.out16) {   // fp16 twin (round to nearest) for the next tensor-core consumer
                                if (out_mode == 2) { x0 = sb_unbias_tf32(x0); x1 = sb_unbias_tf32(x1); }
                                const __half2 hv = __floats2half2_rn(x0, x1);
                                sts32u(tbuf + swz64(row * 64 + (cl & 31) * 2), *reinterpret_cast<const uint32_t*>(&hv));
                            }
                        }
                    }
                    fence_proxy_async();                  // generic-proxy writes -> visible to the TMA stores
                    named_bar_sync(1 + wg, 128);
                    if (store_thread) {
                        const int col = nt * BLOCK_N + 32 * ch;
                        if (row0 < p.M && col < d.Cout) {
                            if (EPI == kEpiTma && d.out) tma_store_2d(&map_o, rbuf, col, row0);
                            if (d.out16) tma_store_2d(&map_o16, tbuf, col, row0);
                        }
                        bulk_commit();                    // one group per entry, empty or not
                        if (e > 0) {
                            bulk_wait_read<1>();          // all groups but this entry's have read their slots
                            mbar_arrive(&slot_empty[wg * kSlots + held]);
                        }
                    }
                    held = slot;
                    if (++slot == kSlots) { slot = 0; sphase ^= 1; }
                }
            } else {
                // ---- epilogue from registers: per row {output offset, residual row, upsample source + weights}, then
                // per column pair.  Row h is r_lo + 8 * (h & 1) + 64 * (h >> 1), its accumulators at
                // (h >> 1) * kAcc + 4 * j + 2 * (h & 1) + {0, 1}.
                long long ooff[kRows];
                bool valid[kRows];
                long long rrow[kRows];
                int uoff[kRows];
                float uly[kRows], ulx[kRows];
                bool by[kRows], bx[kRows];
#pragma unroll
                for (int h = 0; h < kRows; ++h) {
                    const int row = r_lo + 8 * (h & 1) + 64 * (h >> 1);
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
                    const bool cv = c < d.Cout;
                    const int cs = cv ? c : 0;                    // past Cout: any in-bounds column, never stored
                    // every load of the column step, for all rows, is issued before its first store (addresses of
                    // invalid rows and columns are clamped into the tensors instead of branching around the loads)
                    const float2 sc = d.scale ? __ldg(reinterpret_cast<const float2*>(d.scale + cs)) : make_float2(1.f, 1.f);
                    const float2 sh = d.shift ? __ldg(reinterpret_cast<const float2*>(d.shift + cs)) : make_float2(0.f, 0.f);
                    float2 rv[kRows], ua[kRows], ub[kRows], ug[kRows], uh[kRows];
#pragma unroll
                    for (int h = 0; h < kRows; ++h) {
                        if (HAS_RES) rv[h] = __ldg(reinterpret_cast<const float2*>(d.residual + rrow[h] + cs));
                        if (HAS_UP) {
                            const float* u00 = d.up_src + uoff[h] + cs;
                            const long long dx = bx[h] ? d.Cout : 0;
                            const long long dy = by[h] ? (long long)d.UW * d.Cout : 0;
                            ua[h] = __ldg(reinterpret_cast<const float2*>(u00));
                            ub[h] = __ldg(reinterpret_cast<const float2*>(u00 + dx));
                            ug[h] = __ldg(reinterpret_cast<const float2*>(u00 + dy));
                            uh[h] = __ldg(reinterpret_cast<const float2*>(u00 + dy + dx));
                        }
                    }
#pragma unroll
                    for (int h = 0; h < kRows; ++h) {
                        if (!cv || !valid[h]) continue;
                        const int ai = (h >> 1) * kAcc + 4 * j + 2 * (h & 1);
                        float x0 = fmaf(acc[ai], sc.x, sh.x);
                        float x1 = fmaf(acc[ai + 1], sc.y, sh.y);
                        if (HAS_RES) {
                            float2 r = rv[h];
                            if (res_biased) { r.x = sb_unbias_tf32(r.x); r.y = sb_unbias_tf32(r.y); }
                            x0 += r.x; x1 += r.y;
                        }
                        if (HAS_UP) {
                            const float2 a = ua[h], bq = ub[h], g = ug[h], hh = uh[h];
                            const float ly1 = uly[h], ly0 = 1.f - ly1, lx1 = ulx[h], lx0 = 1.f - lx1;
                            x0 += ly0 * (lx0 * a.x + lx1 * bq.x) + ly1 * (lx0 * g.x + lx1 * hh.x);
                            x1 += ly0 * (lx0 * a.y + lx1 * bq.y) + ly1 * (lx0 * g.y + lx1 * hh.y);
                        }
                        if (MASK && p.mask16) {     // dgrad without a mask (a residual add only) has mask16 == NULL
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
            }
            if (tr && threadIdx.x == 0 && tile == (int)blockIdx.x) { tr[4] = gtimer(); tr[12] = clock64(); }
            if (tr && store_thread) atomicAdd(tr + kTraceTiles + wg, 1ull);
        }
        if (kTmaEpi && (threadIdx.x & 127) == 0) bulk_wait<0>();     // the last tile's stores have completed
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
              const cuuint32_t* box, bool f16, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUresult r = enc(m, f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, const_cast<void*>(base), dims,
                     strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle,
                     CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS;
}

typedef CUresult (*EncodeIm2colFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                   const cuuint64_t*, const int*, const int*, cuuint32_t, cuuint32_t, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                   CUtensorMapFloatOOBfill);

EncodeIm2colFn get_encode_im2col() {
    static EncodeIm2colFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeIm2col", &p, cudaEnableDefault, &qres) != cudaSuccess ||
            qres != cudaDriverEntryPointSuccess)
            return nullptr;
        fn = (EncodeIm2colFn)p;
    }
    return fn;
}

// im2col map of a 3x3 / pad 1 / stride 1 conv over fp16 NHWC activations [N, H, W, in_ld] (channels [0, Cin) used):
// a load brings the BLOCK_M pixels that follow its start coordinate in (n, h, w) order, 64 channels (128 bytes) each,
// 128-byte swizzled -- the layout of the flat 2-D [M, Cin] box of a 1x1 conv.  The bounding box holds the origins of
// the taps, output pixel - pad: w in [-1, W - 2] (lower corner -1, upper corner W - 1 + (-1)), h alike; the tap
// offsets (s, r) in 0..2 shift every pixel, and what lands outside [0, W) x [0, H) is zero-filled.
bool make_map_im2col3x3(CUtensorMap* m, const sb_conv_desc* d) {
    EncodeIm2colFn enc = get_encode_im2col();
    if (!enc) return false;
    const cuuint64_t dims[4] = {(cuuint64_t)d->Cin, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)d->N};
    const cuuint64_t strides[3] = {(cuuint64_t)d->in_ld * 2, (cuuint64_t)d->W * d->in_ld * 2,
                                   (cuuint64_t)d->H * d->W * d->in_ld * 2};
    const int lower[2] = {-d->pad, -d->pad}, upper[2] = {d->pad - (d->kw - 1), d->pad - (d->kh - 1)};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(static_cast<const void*>(d->in)), dims,
                     strides, lower, upper, 64, BLOCK_M, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
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

// operands (a, b); residual in, fp32 and fp16 outputs (r, o, o16: the TMA residual epilogue only, zero otherwise)
struct TcMaps {
    CUtensorMap a, b, r, o, o16;
};

// PP: the ping-pong schedule.  An instantiation that has a ping-pong twin runs it when some CTA gets a second tile.
// With one tile per CTA there is no other tile's epilogue to hide, and a warpgroup alone would run all 128 rows'.

template <int BN, int ST, bool RES, bool UP, bool IN16, bool STEM = false, bool MASK = false, bool PP = false,
          int EPI = kEpiRegs>
int launch_t(const TcMaps& m, const TcParams& p, cudaStream_t st) {
    const int tiles = p.num_m_tiles * p.num_n_tiles;
    int slots = sb_num_sms();
    if (p.d.max_ctas > 0 && p.d.max_ctas < slots) slots = p.d.max_ctas;
    const int grid = tiles < slots ? tiles : slots;
    if constexpr (!PP && pingpong_ok(BN, RES, UP, IN16, STEM, MASK, EPI)) {
        if (tiles > grid) return launch_t<BN, ST, RES, UP, IN16, STEM, MASK, true, EPI>(m, p, st);
    }
    constexpr size_t smem = conv_smem(BN, ST, epi_slots(BN, EPI), epi_slot_bytes(EPI));
    static_assert(smem <= 227 * 1024, "smem budget");
    auto kern = conv_tc_kernel<BN, ST, RES, UP, IN16, STEM, MASK, PP, EPI>;
    static bool attr_done[kSbMaxDevices] = {false};
    bool& attr = attr_done[sb_cur_device()];
    if (!attr) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
        attr = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid);
    cfg.blockDim = dim3(conv_threads(STEM, res_ring(RES, EPI)));
    cfg.dynamicSmemBytes = smem;
    cfg.stream = st;
    cudaLaunchAttribute attrs[1];
    attrs[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attrs[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attrs;
    cfg.numAttrs = 1;
    cudaError_t le = cudaLaunchKernelEx(&cfg, kern, m.a, m.b, m.r, m.o, m.o16, p);
    SB_LAUNCHED();
    if (le != cudaSuccess) return (int)le;
    SB_CHECK_LAUNCH();
    return SB_OK;
}

// ST: operand stages beside no ring or 4 KB slots (kEpiTma16); ST_EPI: operand stages beside the 12 KB slots of
// kEpiTma (the residual, fp32 outputs)
template <int BN, int ST, int ST_EPI>
int launch(const TcMaps& m, const TcParams& p, bool dgrad, int epi, cudaStream_t st) {
    const bool res = p.d.residual != nullptr, up = p.d.up_src != nullptr;   // never both (supported())
    if (dgrad && (p.mask16 || res))     // fp16 operands, never an upsample source (sb_conv2d_tc_dgrad)
        return res ? launch_t<BN, ST, true, false, true, false, true>(m, p, st)
                   : launch_t<BN, ST, false, false, true, false, true>(m, p, st);
    if (p.d.in_dtype == 1) {
        if (up) return launch_t<BN, ST, false, true, true>(m, p, st);
        if (res) {
            if constexpr (BN <= 128) return launch_t<BN, ST_EPI, true, false, true, false, false, false, kEpiTma>(m, p, st);
            return SB_EINVAL;
        }
        if (epi == kEpiTma) return launch_t<BN, ST_EPI, false, false, true, false, false, false, kEpiTma>(m, p, st);
        if (epi == kEpiTma16) return launch_t<BN, ST, false, false, true, false, false, false, kEpiTma16>(m, p, st);
        return launch_t<BN, ST, false, false, true>(m, p, st);
    }
    if (up) return launch_t<BN, ST, false, true, false>(m, p, st);
    return res ? launch_t<BN, ST, true, false, false>(m, p, st) : launch_t<BN, ST, false, false, false>(m, p, st);
}

// The fp16-operand forward TMA epilogue moves the residual and both outputs as 2-D [ld, M] TMA boxes: output
// pixels must be contiguous rows (m * out_w_stride), and row strides and bases 16-byte aligned.  The twin's rows must
// also be a whole number of 16-byte units (Cout % 8 == 0): with Cout = 36 or 100 the bulk tensor store was measured
// to write fp16 columns past Cout, into the neighbouring channels of a wider row (H100, CUDA 12.9).
bool tma_epilogue_layout_ok(const sb_conv_desc* d) {
    const long long ws = d->out_w_stride;
    if (d->Ho > 1 && d->out_h_stride != (long long)d->Wo * ws) return false;
    if (d->N > 1 && d->out_n_stride != (long long)d->Ho * d->Wo * ws) return false;
    if (d->out16 && ((ws & 7) || (d->out_coff & 7) || (d->Cout & 7) || (reinterpret_cast<uintptr_t>(d->out16) & 15)))
        return false;
    return true;   // fp32 rows: out_w_stride, out_coff % 4 == 0 and the 16-byte aligned base are checked for every conv
}

// dgrad: the data-gradient entry point, whose residual (and mask) epilogue runs from registers and takes any layout
int supported(const sb_conv_desc* d, bool dgrad) {
    if (!d || !d->in || !d->wgt) return 0;
    const int bk = d->in_dtype == 1 ? 64 : 32;
    if (d->in_dtype != 0 && d->in_dtype != 1) return 0;
    if (d->stride != 1 || d->Cin % bk != 0 || d->in_ld % (d->in_dtype == 1 ? 8 : 4) != 0) return 0;
    if (d->in_ld < d->Cin) return 0;      // a shorter row would read the next pixel's channels (past the end on the last)
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
    if (d->residual && d->in_dtype == 1 && !dgrad && !tma_epilogue_layout_ok(d)) return 0;
    return 1;
}

}  // namespace

extern "C" int sb_conv2d_tc_supported(const sb_conv_desc* d) { return supported(d, false); }

// ---- optional phase trace (tools/conv_trace.py): 16 words per CTA, kTraceCtas CTAs per launch
namespace {
unsigned long long* g_trace = nullptr;
int g_trace_cap = 0, g_trace_n = 0;
struct TraceInfo { int v[12]; };
TraceInfo g_trace_info[4096];
int g_trace_epi[4096];
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
extern "C" int sb_conv_trace_epilogue(int id) { return id < 0 || id >= g_trace_n ? SB_EINVAL : g_trace_epi[id]; }

namespace {
// rows: flat 128-pixel tiles loaded by TMA im2col for a 3x3 conv (sb_conv2d_tc_rows; the caller has checked the
// descriptor)
int conv2d_tc(const sb_conv_desc* d, const __half* mask16, bool dgrad, bool rows, sb_stream_t stream) {
    if (!supported(d, dgrad)) return SB_EINVAL;
    TcParams p;
    p.d = *d;
    p.mask16 = mask16;
    p.trace = nullptr;
    p.stem_im = nullptr;
    p.sH = p.sW = 0;
    // spatial 8x16 tiles for 3x3 convs, and for the FPN laterals so that the bilinear upsample taps of a tile
    // (5x9 source pixels) stay in L1 instead of being re-fetched from L2 for every output row
    p.patch = !rows && (d->kh == 3 || d->up_src) ? 1 : 0;
    p.rows = rows ? 1 : 0;
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
    if (const char* e = getenv("SB_TC_BLOCK_N")) { int v = atoi(e); if ((v == 128 || v == 256) && d->Cout >= 256) BN = v; }
    // residual layers are HBM-bound: the narrower tile keeps more CTAs busy, and its epilogue buffers fit beside
    // the operand stages
    if (d->residual && BN == 256) BN = 128;
    p.num_n_tiles = (d->Cout + BN - 1) / BN;
    // the TMA epilogue: fp16-operand forward on flat rows (1x1, or 3x3 through the rows entry) whose outputs are 2-D
    // [ld, M] maps.  The TF32 mode, the data gradient, the upsample-add and 8x16 patches keep the register epilogue.
    int epi = kEpiRegs;
    if (f16 && !dgrad && !d->up_src && !p.patch && tma_epilogue_layout_ok(d))
        epi = d->out || d->residual ? kEpiTma : kEpiTma16;
    if (epi == kEpiTma && !d->residual && BN == 128) {
        // no ping-pong twin (pingpong_ok): where a CTA gets a second tile, the register epilogue's ping-pong hides
        // the epilogue under the other warpgroup's MMAs, which a cooperative TMA epilogue cannot
        int ctas = sb_num_sms();
        if (d->max_ctas > 0 && d->max_ctas < ctas) ctas = d->max_ctas;
        if ((long long)p.num_m_tiles * p.num_n_tiles > ctas) epi = kEpiRegs;
    }
    if (g_trace && g_trace_n < g_trace_cap) {
        const int id = g_trace_n++;
        p.trace = g_trace + (size_t)id * kTraceCtas * kTraceWords;
        int* v = g_trace_info[id].v;
        v[0] = d->Cin; v[1] = d->Cout; v[2] = d->kh; v[3] = (int)p.M; v[4] = BN; v[5] = p.num_m_tiles * p.num_n_tiles;
        v[6] = p.num_k_blocks; v[7] = d->residual ? 1 : 0; v[8] = d->up_src ? 1 : 0;
        v[9] = (f16 ? 1 : 0) | (dgrad ? 2 : 0) | (mask16 ? 4 : 0);     // operand type and entry point
        v[10] = d->max_ctas; v[11] = d->N;
        g_trace_epi[id] = epi != kEpiRegs ? 1 : 0;
    }
    TcMaps m;
    memset(&m, 0, sizeof(m));
    CUtensorMap &ma = m.a, &mb = m.b;
    if (p.rows) {
        if (!make_map_im2col3x3(&ma, d)) return SB_EINVAL;
    } else if (p.patch) {
        cuuint64_t dims[4] = {(cuuint64_t)d->Cin, (cuuint64_t)d->W, (cuuint64_t)d->H, (cuuint64_t)d->N};
        cuuint64_t strides[3] = {(cuuint64_t)d->in_ld * esz, (cuuint64_t)d->W * d->in_ld * esz,
                                 (cuuint64_t)d->H * d->W * d->in_ld * esz};
        cuuint32_t box[4] = {(cuuint32_t)BLOCK_K, TW, TH, 1};
        if (!make_map(&ma, d->in, 4, dims, strides, box, f16)) return SB_EINVAL;
    } else {
        cuuint64_t dims[2] = {(cuuint64_t)d->Cin, (cuuint64_t)p.M};
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
    if (epi != kEpiRegs) {
        // TMA epilogue: [Cout, M] boxes of 64 rows and 32 columns, one ring entry each; the fp16 box has 64-byte rows,
        // so it is 64-byte swizzled
        const cuuint64_t dims[2] = {(cuuint64_t)d->Cout, (cuuint64_t)p.M};
        const cuuint32_t box32[2] = {32, 64};
        const cuuint64_t rs[1] = {(cuuint64_t)d->res_ld * 4};
        if (d->residual && !make_map(&m.r, d->residual, 2, dims, rs, box32, false)) return SB_EINVAL;
        const cuuint64_t os[1] = {(cuuint64_t)d->out_w_stride * 4}, os16[1] = {(cuuint64_t)d->out_w_stride * 2};
        if (d->out && !make_map(&m.o, d->out + d->out_coff, 2, dims, os, box32, false)) return SB_EINVAL;
        if (d->out16 && !make_map(&m.o16, reinterpret_cast<const __half*>(d->out16) + d->out_coff, 2, dims, os16,
                                  box32, true, CU_TENSOR_MAP_SWIZZLE_64B))
            return SB_EINVAL;
    }
    cudaStream_t st = sb_cs(stream);
    switch (BN) {        // <BN, operand stages, operand stages beside the 12 KB-slot rings>
        case 32: return launch<32, 9, 7>(m, p, dgrad, epi, st);
        case 64: return launch<64, 8, 6>(m, p, dgrad, epi, st);
        case 256: return launch<256, 4, 3>(m, p, dgrad, epi, st);
        default: return launch<128, 6, 4>(m, p, dgrad, epi, st);
    }
}
}  // namespace

extern "C" int sb_conv2d_tc(const sb_conv_desc* d, sb_stream_t stream) {
    return conv2d_tc(d, nullptr, false, false, stream);
}

// A 3x3 conv on 8x16 patches issues all 128 MMA rows of a patch that runs past the right or bottom edge of its map
// (a 14x14 map takes two patches, 256 rows for 196 pixels).  Flat tiles of 128 consecutive output pixels, loaded
// by TMA im2col one tap at a time, issue only the rows of the last tile past M.  Per output pixel the A values and
// the K order (tap-major, then Cin chunks) are those of the patch path, so the results are bit-identical to
// sb_conv2d_tc's.  Same kernel instantiations, epilogue of the flat rows (any out strides).
extern "C" int sb_conv2d_tc_rows(const sb_conv_desc* d, sb_stream_t stream) {
    if (!d || d->in_dtype != 1 || d->kh != 3 || d->kw != 3 || d->pad != 1 || d->stride != 1 || d->residual ||
        d->up_src)
        return SB_EINVAL;
    return conv2d_tc(d, nullptr, false, true, stream);
}

// Data gradient of a convolution as the forward implicit GEMM on transposed weights (the caller packs them
// [Cin][kh][kw][Cout], taps flipped, frozen-BN scale folded in), with the ReLU mask of a saved tensor applied after
// the optional residual add.  mask16 has the output's element layout (out strides and channel offset).
extern "C" int sb_conv2d_tc_dgrad(const sb_conv_desc* d, const void* mask16, sb_stream_t stream) {
    if (!d || d->in_dtype != 1 || d->up_src || d->relu || d->out_mode != 0) return SB_EINVAL;
    if (reinterpret_cast<uintptr_t>(mask16) & 3) return SB_EINVAL;
    return conv2d_tc(d, reinterpret_cast<const __half*>(mask16), true, false, stream);
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
    p.stem_im = im_nchw; p.sH = H; p.sW = W;
    p.mask16 = nullptr;
    TcMaps m;
    memset(&m, 0, sizeof(m));
    {
        cuuint64_t dims[2] = {192, 64};
        cuuint64_t strides[1] = {192 * 2};
        cuuint32_t box[2] = {64, 64};
        if (!make_map(&m.b, wgt16, 2, dims, strides, box, true)) return SB_EINVAL;
    }
    return launch_t<64, 8, false, false, true, true>(m, p, sb_cs(stream));
}
