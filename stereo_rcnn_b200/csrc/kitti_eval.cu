// kitti_eval.cu -- the KITTI object devkit's evaluate_object (Car) on the device: per (detection, ground truth) pair
// the 2D, bird's-eye (BEV) and 3D overlaps, then per configuration (metric, IoU bar, difficulty) the devkit's greedy
// matching over every image -- once to collect the true-positive scores, once per recall threshold for the
// precision / recall / orientation curves -- and the average precision.  The restatement of the devkit that this
// follows, and oracle/kitti_eval.py with it, is DESIGN.md §9.
//
// Every floating-point operation of the overlaps is an explicit fp64 round-to-nearest intrinsic in the oracle's order
// (no contraction), so the device and the oracle make the same decisions bit for bit.  Sums over images run in image
// order, so the results are identical run to run.
#include <math.h>

#include "common.cuh"

namespace {

// row fields (SB_KITTI_ROW doubles per row)
constexpr int kTrunc = 0, kOcc = 1, kAlpha = 2, kX1 = 3, kY1 = 4, kX2 = 5, kY2 = 6, kH = 7, kW = 8, kL = 9, kX = 10,
              kY = 11, kZ = 12, kCos = 13, kSin = 14, kScore = 15;
constexpr int kRow = SB_KITTI_ROW;
constexpr int kT = SB_KITTI_MAX_THRESHOLDS;     // 41 recall sample points
constexpr int kDontCare = 2;
constexpr int kMaxPoly = 16;                    // clipped polygon capacity (8 in exact arithmetic)
constexpr int kStageBytes = 8192;               // per-(configuration, image) shared-memory staging
constexpr double kNoMatch = -10000000.0;

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }

// ------------------------------------------------------------------------------------------------ overlaps ----
__device__ void bev_corners(const double* r, double* px, double* pz) {
    const double hl = dmul(r[kL], 0.5), hw = dmul(r[kW], 0.5), c = r[kCos], s = r[kSin];
    const double dx[4] = {hl, hl, -hl, -hl}, dz[4] = {hw, -hw, -hw, hw};
    double x[4], z[4];
    for (int k = 0; k < 4; ++k) {
        x[k] = dadd(r[kX], dadd(dmul(c, dx[k]), dmul(s, dz[k])));
        z[k] = dadd(r[kZ], dsub(dmul(c, dz[k]), dmul(s, dx[k])));
    }
    double a = 0.0;
    for (int k = 0; k < 4; ++k) {
        const int k1 = (k + 1) & 3;
        a = dadd(a, dsub(dmul(x[k], z[k1]), dmul(x[k1], z[k])));
    }
    const int order[2][4] = {{0, 1, 2, 3}, {0, 3, 2, 1}};      // counter-clockwise
    for (int k = 0; k < 4; ++k) {
        px[k] = x[order[a < 0.0][k]];
        pz[k] = z[order[a < 0.0][k]];
    }
}

__device__ __forceinline__ double edge_side(double ax, double az, double ex, double ez, double x, double z) {
    return dsub(dmul(ex, dsub(z, az)), dmul(ez, dsub(x, ax)));
}

// area of the intersection of the two BEV rectangles: det clipped by gt (Sutherland-Hodgman), shoelace area
__device__ double bev_intersection(const double* d, const double* g) {
    // circumscribed circles apart: disjoint
    const double cx = dsub(d[kX], g[kX]), cz = dsub(d[kZ], g[kZ]);
    const double rd = dmul(__dsqrt_rn(dadd(dmul(d[kL], d[kL]), dmul(d[kW], d[kW]))), 0.5);
    const double rg = dmul(__dsqrt_rn(dadd(dmul(g[kL], g[kL]), dmul(g[kW], g[kW]))), 0.5);
    const double rr = dadd(rd, rg);
    if (dadd(dmul(cx, cx), dmul(cz, cz)) > dmul(rr, rr)) return 0.0;
    double qx[4], qz[4];
    double px[2][kMaxPoly], pz[2][kMaxPoly];
    bev_corners(g, qx, qz);
    bev_corners(d, px[0], pz[0]);
    int n = 4, cur = 0;
    for (int e = 0; e < 4 && n > 0; ++e) {
        const double ax = qx[e], az = qz[e];
        const double ex = dsub(qx[(e + 1) & 3], ax), ez = dsub(qz[(e + 1) & 3], az);
        const double* sx = px[cur];
        const double* sz = pz[cur];
        double* ox = px[cur ^ 1];
        double* oz = pz[cur ^ 1];
        int m = 0;
        for (int k = 0; k < n; ++k) {
            const int kp = k == 0 ? n - 1 : k - 1;
            const double cc = edge_side(ax, az, ex, ez, sx[k], sz[k]);
            const double cp = edge_side(ax, az, ex, ez, sx[kp], sz[kp]);
            if ((cc >= 0.0) != (cp >= 0.0) && m < kMaxPoly) {
                const double t = ddiv(cp, dsub(cp, cc));
                ox[m] = dadd(sx[kp], dmul(t, dsub(sx[k], sx[kp])));
                oz[m] = dadd(sz[kp], dmul(t, dsub(sz[k], sz[kp])));
                ++m;
            }
            if (cc >= 0.0 && m < kMaxPoly) {
                ox[m] = sx[k];
                oz[m] = sz[k];
                ++m;
            }
        }
        n = m;
        cur ^= 1;
    }
    if (n < 3) return 0.0;
    double a = 0.0;
    for (int k = 0; k < n; ++k) {
        const int k1 = k + 1 == n ? 0 : k + 1;
        a = dadd(a, dsub(dmul(px[cur][k], pz[cur][k1]), dmul(px[cur][k1], pz[cur][k])));
    }
    return dmul(fabs(a), 0.5);
}

// crit 0: intersection / area(det); otherwise intersection / union.  A zero denominator gives 0.
__device__ __forceinline__ double ratio(double inter, double area_d, double area_g, int crit0) {
    const double den = crit0 ? area_d : dsub(dadd(area_d, area_g), inter);
    return den == 0.0 ? 0.0 : ddiv(inter, den);
}

__device__ double overlap_2d(const double* d, const double* g, int crit0) {
    const double iw = dsub(fmin(d[kX2], g[kX2]), fmax(d[kX1], g[kX1]));
    const double ih = dsub(fmin(d[kY2], g[kY2]), fmax(d[kY1], g[kY1]));
    if (!(iw > 0.0 && ih > 0.0)) return 0.0;
    const double inter = dmul(iw, ih);
    return ratio(inter, dmul(dsub(d[kX2], d[kX1]), dsub(d[kY2], d[kY1])),
                 dmul(dsub(g[kX2], g[kX1]), dsub(g[kY2], g[kY1])), crit0);
}

__global__ void __launch_bounds__(256)
overlaps_kernel(const double* __restrict__ gt, const int* __restrict__ gt_code, const double* __restrict__ det,
                const long long* __restrict__ gt_off, const long long* __restrict__ det_off,
                const long long* __restrict__ pair_off, int n_images, long long n_pairs, double* __restrict__ ov_2d,
                double* __restrict__ ov_bev, double* __restrict__ ov_3d) {
    const long long p = (long long)blockIdx.x * 256 + threadIdx.x;
    if (p >= n_pairs) return;
    int lo = 0, hi = n_images;                    // last image with pair_off[img] <= p
    while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (pair_off[mid] <= p) lo = mid; else hi = mid;
    }
    const long long ng = gt_off[lo + 1] - gt_off[lo];
    const long long q = p - pair_off[lo];
    const long long gi = gt_off[lo] + q % ng, dj = det_off[lo] + q / ng;
    const double* g = gt + gi * kRow;
    const double* d = det + dj * kRow;
    const int crit0 = gt_code[gi] == kDontCare;
    ov_2d[p] = overlap_2d(d, g, crit0);
    const double inter = bev_intersection(d, g);
    ov_bev[p] = ratio(inter, dmul(d[kL], d[kW]), dmul(g[kL], g[kW]), crit0);
    const double ih = fmax(0.0, dsub(fmin(d[kY], g[kY]), fmax(dsub(d[kY], d[kH]), dsub(g[kY], g[kH]))));
    ov_3d[p] = ratio(dmul(inter, ih), dmul(dmul(d[kH], d[kW]), d[kL]), dmul(dmul(g[kH], g[kW]), g[kL]), crit0);
}

// ------------------------------------------------------------------------------------------------ matching ----
struct Bars {
    double v[SB_KITTI_MAX_BARS];
};

struct Config {
    int metric, d;
    double bar;
};

__device__ __forceinline__ Config config(int cfg, int n_bars, const Bars& bars) {
    Config c;
    c.d = cfg % 3;
    c.bar = bars.v[(cfg / 3) % n_bars];
    c.metric = cfg / (3 * n_bars);
    return c;
}

// ground-truth flag: 0 counted, 1 ignored (Van, or a Car outside the difficulty), -1 not a gt of this class
__device__ __forceinline__ int gt_flag(const double* g, int code, int d) {
    const double min_h[3] = {40.0, 25.0, 25.0}, max_occ[3] = {0.0, 1.0, 2.0}, max_trunc[3] = {0.15, 0.30, 0.50};
    if (code == 1) return 1;
    if (code != 0) return -1;
    const bool hard = g[kOcc] > max_occ[d] || g[kTrunc] > max_trunc[d] || dsub(g[kY2], g[kY1]) <= min_h[d];
    return hard ? 1 : 0;
}

// detection flag: 1 too short for the difficulty, 0 a Car detection, -1 another class
__device__ __forceinline__ int det_flag(const double* r, int code, int d) {
    const double min_h[3] = {40.0, 25.0, 25.0};
    if (dsub(r[kY2], r[kY1]) < min_h[d]) return 1;
    return code == 0 ? 0 : -1;
}

// One image's matching state for one warp: the image's overlap matrix [nd][ng] of the configuration's metric and
// per-lane "assigned" bit rows (word w of lane L at asg[w * 32 + L]), in shared memory when both fit, else read from
// the global matrix and the warp's slice of the workspace.
struct ImageView {
    const double* ov;
    unsigned* asg;
    int ng, nd;
};

__device__ ImageView stage_image(int cfg, int img, const Config& c, const long long* gt_off, const long long* det_off,
                                 const long long* pair_off, const double* const* ov3, long long n_det_rows,
                                 int n_images, unsigned* ws_asg, double* smem) {
    const int lane = threadIdx.x;
    ImageView v;
    v.ng = (int)(gt_off[img + 1] - gt_off[img]);
    v.nd = (int)(det_off[img + 1] - det_off[img]);
    const long long n_ov = (long long)v.ng * v.nd;
    const int words = (v.nd + 31) / 32;
    const double* g_ov = ov3[c.metric] + pair_off[img];
    if (n_ov * 8 + (long long)words * 32 * 4 <= kStageBytes) {
        for (int k = lane; k < n_ov; k += 32) smem[k] = g_ov[k];
        v.ov = smem;
        v.asg = reinterpret_cast<unsigned*>(smem + n_ov);
    } else {
        v.ov = g_ov;
        v.asg = ws_asg + (long long)cfg * (n_det_rows + 32LL * n_images) + det_off[img] + 32LL * img;
    }
    __syncwarp();
    return v;
}

__device__ __forceinline__ bool asg_get(const unsigned* asg, int j) {
    return (asg[(j >> 5) * 32 + threadIdx.x] >> (j & 31)) & 1u;
}
__device__ __forceinline__ void asg_set(unsigned* asg, int j) { asg[(j >> 5) * 32 + threadIdx.x] |= 1u << (j & 31); }

// pass 1 (compute_fp = false): lane 0 runs the greedy; the image's true-positive scores go to its gt rows' slots
__global__ void __launch_bounds__(32)
match_tp_kernel(const double* __restrict__ gt, const int* __restrict__ gt_code, const double* __restrict__ det,
                const int* __restrict__ det_code, const long long* __restrict__ gt_off,
                const long long* __restrict__ det_off, const long long* __restrict__ pair_off, int n_images,
                long long n_gt_rows, long long n_det_rows, const double* __restrict__ ov_2d,
                const double* __restrict__ ov_bev, const double* __restrict__ ov_3d, Bars bars, int n_bars, unsigned* __restrict__ ws_asg, int* __restrict__ ntp, int* __restrict__ ngt,
                double* __restrict__ tp_scores) {
    extern __shared__ double smem[];
    const int img = blockIdx.x, cfg = blockIdx.y;
    const Config c = config(cfg, n_bars, bars);
    const double* ov3[3] = {ov_2d, ov_bev, ov_3d};
    const ImageView v = stage_image(cfg, img, c, gt_off, det_off, pair_off, ov3, n_det_rows, n_images, ws_asg, smem);
    if (threadIdx.x != 0) return;
    gt += gt_off[img] * kRow; gt_code += gt_off[img];
    det += det_off[img] * kRow; det_code += det_off[img];
    for (int w = 0; w < (v.nd + 31) / 32; ++w) v.asg[w * 32] = 0u;
    double* scores = tp_scores + (long long)cfg * n_gt_rows + gt_off[img];
    int n_tp = 0, n_gt = 0;
    for (int i = 0; i < v.ng; ++i) {
        const int ig = gt_flag(gt + i * kRow, gt_code[i], c.d);
        n_gt += ig == 0;
        if (ig == -1) continue;
        int best = -1;
        double valid = kNoMatch;
        for (int j = 0; j < v.nd; ++j) {
            if (det_flag(det + j * kRow, det_code[j], c.d) == -1 || asg_get(v.asg, j)) continue;
            const double o = v.ov[(long long)j * v.ng + i], s = det[j * kRow + kScore];
            if (o > c.bar && s > valid) {
                best = j;
                valid = s;
            }
        }
        if (valid == kNoMatch) continue;
        if (ig == 0 && det_flag(det + best * kRow, det_code[best], c.d) != 1) scores[n_tp++] = valid;
        asg_set(v.asg, best);
    }
    ntp[(long long)cfg * n_images + img] = n_tp;
    ngt[(long long)cfg * n_images + img] = n_gt;
}

// per configuration: the true-positive scores of all images in image order (compact), their count, n_gt, and which
// ranks of the descending order become thresholds (the devkit's getThresholds)
__global__ void __launch_bounds__(1024)
thresholds_scan_kernel(const long long* __restrict__ gt_off, int n_images, long long n_gt_rows,
                       const int* __restrict__ ntp, const int* __restrict__ ngt, const double* __restrict__ tp_scores,
                       double* __restrict__ compact, long long* __restrict__ n_tp_total, int* __restrict__ sel,
                       int* __restrict__ n_thresholds, double* __restrict__ thresholds, long long* __restrict__ n_gt_out) {
    __shared__ long long s_warp[32][2];
    __shared__ long long s_base[2];
    const int cfg = blockIdx.x, t = threadIdx.x, lane = t & 31, warp = t >> 5;
    ntp += (long long)cfg * n_images;
    ngt += (long long)cfg * n_images;
    tp_scores += (long long)cfg * n_gt_rows;
    compact += (long long)cfg * n_gt_rows;
    if (t == 0) s_base[0] = s_base[1] = 0;
    if (t < kT) thresholds[cfg * kT + t] = 0.0;
    __syncthreads();
    for (int c0 = 0; c0 < n_images; c0 += 1024) {
        const int img = c0 + t;
        const long long a = img < n_images ? ntp[img] : 0, b = img < n_images ? ngt[img] : 0;
        long long ia = a, ib = b;                           // inclusive warp scan
        for (int o = 1; o < 32; o <<= 1) {
            const long long ua = __shfl_up_sync(0xffffffffu, ia, o), ub = __shfl_up_sync(0xffffffffu, ib, o);
            if (lane >= o) { ia += ua; ib += ub; }
        }
        if (lane == 31) { s_warp[warp][0] = ia; s_warp[warp][1] = ib; }
        __syncthreads();
        if (warp == 0) {
            long long wa = s_warp[lane][0], wb = s_warp[lane][1];
            for (int o = 1; o < 32; o <<= 1) {
                const long long ua = __shfl_up_sync(0xffffffffu, wa, o), ub = __shfl_up_sync(0xffffffffu, wb, o);
                if (lane >= o) { wa += ua; wb += ub; }
            }
            s_warp[lane][0] = wa;
            s_warp[lane][1] = wb;
        }
        __syncthreads();
        const long long off = s_base[0] + (warp ? s_warp[warp - 1][0] : 0) + ia - a;
        for (int k = 0; k < a; ++k) compact[off + k] = tp_scores[gt_off[img] + k];
        __syncthreads();
        if (t == 0) { s_base[0] += s_warp[31][0]; s_base[1] += s_warp[31][1]; }
        __syncthreads();
    }
    if (t != 0) return;
    const long long n = s_base[0], n_gt = s_base[1];
    n_tp_total[cfg] = n;
    n_gt_out[cfg] = n_gt;
    int nt = 0;
    double cur = 0.0;
    for (long long i = 0; i < n && nt < kT; ++i) {
        const double l = ddiv((double)(i + 1), (double)n_gt);
        const double r = i < n - 1 ? ddiv((double)(i + 2), (double)n_gt) : l;
        if (dsub(r, cur) < dsub(cur, l) && i < n - 1) continue;
        sel[cfg * kT + nt++] = (int)i;
        cur = dadd(cur, 1.0 / 40.0);
    }
    n_thresholds[cfg] = nt;
}

// the selected ranks of the descending order: each thread ranks one score by counting (value, index) predecessors
__global__ void __launch_bounds__(256)
thresholds_rank_kernel(const double* __restrict__ compact, long long n_gt_rows,
                       const long long* __restrict__ n_tp_total, const int* __restrict__ sel,
                       const int* __restrict__ n_thresholds, double* __restrict__ thresholds) {
    __shared__ double s_v[256];
    __shared__ int s_sel[kT];
    const int cfg = blockIdx.y, t = threadIdx.x;
    const long long n = n_tp_total[cfg];
    const long long e = (long long)blockIdx.x * 256 + t;
    if ((long long)blockIdx.x * 256 >= n) return;
    const int nt = n_thresholds[cfg];
    if (t < nt) s_sel[t] = sel[cfg * kT + t];
    compact += (long long)cfg * n_gt_rows;
    const double v = e < n ? compact[e] : 0.0;
    long long rank = 0;
    for (long long b = 0; b < n; b += 256) {
        __syncthreads();
        if (b + t < n) s_v[t] = compact[b + t];
        __syncthreads();
        const int m = (int)min(256LL, n - b);
        for (int k = 0; k < m; ++k) {
            const double u = s_v[k];
            rank += u > v || (u == v && b + k < e);
        }
    }
    if (e >= n) return;
    for (int k = 0; k < nt; ++k)
        if (s_sel[k] == rank) thresholds[cfg * kT + k] = v;
}

// pass 2 (compute_fp = true): lane L runs the greedy at thresholds L and L + 32; per-image counts to the workspace
__global__ void __launch_bounds__(32)
match_curve_kernel(const double* __restrict__ gt, const int* __restrict__ gt_code, const double* __restrict__ det,
                   const int* __restrict__ det_code, const long long* __restrict__ gt_off,
                   const long long* __restrict__ det_off, const long long* __restrict__ pair_off, int n_images,
                   long long n_det_rows, const double* __restrict__ ov_2d, const double* __restrict__ ov_bev,
                   const double* __restrict__ ov_3d, Bars bars, int n_bars,
                   const double* __restrict__ thresholds, const int* __restrict__ n_thresholds,
                   unsigned* __restrict__ ws_asg, int4* __restrict__ counts, double* __restrict__ sims) {
    extern __shared__ double smem[];
    const int img = blockIdx.x, cfg = blockIdx.y, lane = threadIdx.x;
    const Config c = config(cfg, n_bars, bars);
    const double* ov3[3] = {ov_2d, ov_bev, ov_3d};
    const ImageView v = stage_image(cfg, img, c, gt_off, det_off, pair_off, ov3, n_det_rows, n_images, ws_asg, smem);
    gt += gt_off[img] * kRow; gt_code += gt_off[img];
    det += det_off[img] * kRow; det_code += det_off[img];
    const int nt = n_thresholds[cfg];
    for (int t = lane; t < nt; t += 32) {
        const double thr = thresholds[cfg * kT + t];
        for (int w = 0; w < (v.nd + 31) / 32; ++w) v.asg[w * 32 + lane] = 0u;
        int tp = 0, fp = 0, fn = 0;
        double sim = 0.0;
        for (int i = 0; i < v.ng; ++i) {
            const double* g = gt + i * kRow;
            const int ig = gt_flag(g, gt_code[i], c.d);
            if (ig == -1) continue;
            int best = -1;
            double valid = kNoMatch, max_iou = 0.0;
            bool took_ignored = false;
            for (int j = 0; j < v.nd; ++j) {
                const int id = det_flag(det + j * kRow, det_code[j], c.d);
                if (id == -1 || asg_get(v.asg, j) || det[j * kRow + kScore] < thr) continue;
                const double o = v.ov[(long long)j * v.ng + i];
                if (o > c.bar && (o > max_iou || took_ignored) && id == 0) {
                    max_iou = o;
                    best = j;
                    valid = 1.0;
                    took_ignored = false;
                } else if (o > c.bar && valid == kNoMatch && id == 1) {
                    best = j;
                    valid = 1.0;
                    took_ignored = true;
                }
            }
            if (valid == kNoMatch) {
                fn += ig == 0;
                continue;
            }
            if (ig == 0 && det_flag(det + best * kRow, det_code[best], c.d) != 1) {
                ++tp;
                sim = dadd(sim, dmul(dadd(1.0, cos(dsub(g[kAlpha], det[best * kRow + kAlpha]))), 0.5));
            }
            asg_set(v.asg, best);
        }
        for (int j = 0; j < v.nd; ++j)
            fp += !asg_get(v.asg, j) && det_flag(det + j * kRow, det_code[j], c.d) == 0 && !(det[j * kRow + kScore] < thr);
        for (int i = 0; i < v.ng; ++i) {
            if (gt_code[i] != kDontCare) continue;
            for (int j = 0; j < v.nd; ++j) {
                if (asg_get(v.asg, j) || det_flag(det + j * kRow, det_code[j], c.d) != 0 || det[j * kRow + kScore] < thr)
                    continue;
                if (v.ov[(long long)j * v.ng + i] > c.bar) {
                    asg_set(v.asg, j);
                    --fp;
                }
            }
        }
        const long long o = ((long long)cfg * kT + t) * n_images + img;
        counts[o] = make_int4(tp, fp, fn, 0);
        sims[o] = sim;
    }
}

// per configuration: the sums over images in image order, the curves, their suffix maxima and the AP (R11, R40)
__global__ void __launch_bounds__(64)
curves_kernel(int n_images, const int4* __restrict__ counts, const double* __restrict__ sims,
              const int* __restrict__ n_thresholds, long long* __restrict__ tp_out, long long* __restrict__ fp_out,
              long long* __restrict__ fn_out, double* __restrict__ sim_out, double* __restrict__ precision,
              double* __restrict__ recall, double* __restrict__ aos, double* __restrict__ ap) {
    const int cfg = blockIdx.x, t = threadIdx.x;
    const int nt = n_thresholds[cfg];
    const long long o = (long long)cfg * kT + t;
    if (t < kT) {
        long long tp = 0, fp = 0, fn = 0;
        double sim = 0.0;
        if (t < nt) {
            for (int img = 0; img < n_images; ++img) {
                const int4 k = counts[o * n_images + img];
                tp += k.x; fp += k.y; fn += k.z;
                sim = dadd(sim, sims[o * n_images + img]);
            }
        }
        tp_out[o] = tp; fp_out[o] = fp; fn_out[o] = fn; sim_out[o] = sim;
        const double tf = (double)(tp + fp), tn = (double)(tp + fn);
        precision[o] = tp + fp == 0 ? 0.0 : ddiv((double)tp, tf);
        recall[o] = tp + fn == 0 ? 0.0 : ddiv((double)tp, tn);
        aos[o] = tp + fp == 0 ? 0.0 : ddiv(sim, tf);
    }
    __syncthreads();
    if (t != 0) return;
    precision += (long long)cfg * kT;
    aos += (long long)cfg * kT;
    for (int k = kT - 2; k >= 0; --k) {
        precision[k] = fmax(precision[k], precision[k + 1]);
        aos[k] = fmax(aos[k], aos[k + 1]);
    }
    double p11 = 0.0, a11 = 0.0, p40 = 0.0, a40 = 0.0;
    for (int k = 0; k < kT; k += 4) { p11 = dadd(p11, precision[k]); a11 = dadd(a11, aos[k]); }
    for (int k = 1; k < kT; ++k) { p40 = dadd(p40, precision[k]); a40 = dadd(a40, aos[k]); }
    ap[cfg * 4 + 0] = dmul(ddiv(p11, 11.0), 100.0);
    ap[cfg * 4 + 1] = dmul(ddiv(p40, 40.0), 100.0);
    ap[cfg * 4 + 2] = dmul(ddiv(a11, 11.0), 100.0);
    ap[cfg * 4 + 3] = dmul(ddiv(a40, 40.0), 100.0);
}

// ------------------------------------------------------------------------------------------------ workspace ----
struct Ws {
    size_t ov, asg, ntp, ngt, scores, compact, n_tp, sel, counts, sims, total;
};

static size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

static Ws ws_layout(int n_images, long long n_gt_rows, long long n_det_rows, long long n_pairs, int n_bars) {
    const size_t C = 9 * (size_t)n_bars, I = (size_t)n_images;
    Ws w;
    size_t o = 0;
    w.ov = o;      o = align256(o + 3 * (size_t)n_pairs * sizeof(double));
    w.asg = o;     o = align256(o + C * ((size_t)n_det_rows + 32 * I) * sizeof(unsigned));
    w.ntp = o;     o = align256(o + C * I * sizeof(int));
    w.ngt = o;     o = align256(o + C * I * sizeof(int));
    w.scores = o;  o = align256(o + C * (size_t)n_gt_rows * sizeof(double));
    w.compact = o; o = align256(o + C * (size_t)n_gt_rows * sizeof(double));
    w.n_tp = o;    o = align256(o + C * sizeof(long long));
    w.sel = o;     o = align256(o + C * kT * sizeof(int));
    w.counts = o;  o = align256(o + C * kT * I * sizeof(int4));
    w.sims = o;    o = align256(o + C * kT * I * sizeof(double));
    w.total = o;
    return w;
}

static bool sizes_ok(int n_images, long long n_gt_rows, long long n_det_rows, long long n_pairs) {
    return n_images >= 1 && n_gt_rows >= 0 && n_det_rows >= 0 && n_pairs >= 0 && n_gt_rows < (1LL << 40) &&
           n_det_rows < (1LL << 40) && n_pairs < (1LL << 40);
}

static int launch_overlaps(const double* gt, const int* gt_code, const double* det, const long long* gt_off,
                           const long long* det_off, const long long* pair_off, int n_images, long long n_pairs,
                           double* ov_2d, double* ov_bev, double* ov_3d, cudaStream_t s) {
    if (n_pairs == 0) return SB_OK;
    overlaps_kernel<<<(unsigned)((n_pairs + 255) / 256), 256, 0, s>>>(gt, gt_code, det, gt_off, det_off, pair_off,
                                                                       n_images, n_pairs, ov_2d, ov_bev, ov_3d);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

}  // namespace

extern "C" int sb_kitti_overlaps(const double* gt, const int* gt_code, const double* det, const long long* gt_off,
                                 const long long* det_off, const long long* pair_off, int n_images, long long n_pairs,
                                 double* ov_2d, double* ov_bev, double* ov_3d, sb_stream_t stream) {
    if (!gt_off || !det_off || !pair_off || !sizes_ok(n_images, 0, 0, n_pairs)) return SB_EINVAL;
    if (n_pairs > 0 && (!gt || !gt_code || !det || !ov_2d || !ov_bev || !ov_3d)) return SB_EINVAL;
    return launch_overlaps(gt, gt_code, det, gt_off, det_off, pair_off, n_images, n_pairs, ov_2d, ov_bev, ov_3d,
                           sb_cs(stream));
}

extern "C" size_t sb_kitti_eval_workspace_bytes(int n_images, long long n_gt_rows, long long n_det_rows,
                                                long long n_pairs, int n_bars) {
    if (!sizes_ok(n_images, n_gt_rows, n_det_rows, n_pairs) || n_bars < 1 || n_bars > SB_KITTI_MAX_BARS) return 0;
    return ws_layout(n_images, n_gt_rows, n_det_rows, n_pairs, n_bars).total;
}

extern "C" int sb_kitti_eval(const double* gt, const int* gt_code, const double* det, const int* det_code,
                             const long long* gt_off, const long long* det_off, const long long* pair_off,
                             int n_images, long long n_gt_rows, long long n_det_rows, long long n_pairs,
                             const double* bars, int n_bars, void* workspace, size_t workspace_bytes,
                             double* thresholds, int* n_thresholds, long long* tp, long long* fp, long long* fn,
                             double* sim, double* precision, double* recall, double* aos, double* ap,
                             long long* n_gt, sb_stream_t stream) {
    if (!gt_off || !det_off || !pair_off || !bars || !workspace || !thresholds || !n_thresholds || !tp || !fp || !fn ||
        !sim || !precision || !recall || !aos || !ap || !n_gt)
        return SB_EINVAL;
    if ((n_gt_rows > 0 && (!gt || !gt_code)) || (n_det_rows > 0 && (!det || !det_code))) return SB_EINVAL;
    if (!sizes_ok(n_images, n_gt_rows, n_det_rows, n_pairs) || n_bars < 1 || n_bars > SB_KITTI_MAX_BARS)
        return SB_EINVAL;
    for (int b = 0; b < n_bars; ++b)
        if (!(bars[b] >= 0.0 && bars[b] <= 1.0)) return SB_EINVAL;
    const Ws L = ws_layout(n_images, n_gt_rows, n_det_rows, n_pairs, n_bars);
    if (workspace_bytes < L.total || ((uintptr_t)workspace & 255)) return SB_EINVAL;
    const cudaStream_t s = sb_cs(stream);
    char* w = static_cast<char*>(workspace);
    double* ov = reinterpret_cast<double*>(w + L.ov);
    unsigned* asg = reinterpret_cast<unsigned*>(w + L.asg);
    int* ntp = reinterpret_cast<int*>(w + L.ntp);
    int* ngt = reinterpret_cast<int*>(w + L.ngt);
    double* scores = reinterpret_cast<double*>(w + L.scores);
    double* compact = reinterpret_cast<double*>(w + L.compact);
    long long* n_tp = reinterpret_cast<long long*>(w + L.n_tp);
    int* sel = reinterpret_cast<int*>(w + L.sel);
    int4* counts = reinterpret_cast<int4*>(w + L.counts);
    double* sims = reinterpret_cast<double*>(w + L.sims);
    Bars d_bars = {};
    for (int b = 0; b < n_bars; ++b) d_bars.v[b] = bars[b];
    const int C = 9 * n_bars;
    double* ov_2d = ov;
    double* ov_bev = ov + n_pairs;
    double* ov_3d = ov + 2 * n_pairs;
    int rc = launch_overlaps(gt, gt_code, det, gt_off, det_off, pair_off, n_images, n_pairs, ov_2d, ov_bev, ov_3d, s);
    if (rc != SB_OK) return rc;
    const dim3 grid_ic(n_images, C);
    match_tp_kernel<<<grid_ic, 32, kStageBytes, s>>>(gt, gt_code, det, det_code, gt_off, det_off, pair_off, n_images,
                                                     n_gt_rows, n_det_rows, ov_2d, ov_bev, ov_3d, d_bars, n_bars, asg,
                                                     ntp, ngt, scores);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    thresholds_scan_kernel<<<C, 1024, 0, s>>>(gt_off, n_images, n_gt_rows, ntp, ngt, scores, compact, n_tp, sel,
                                              n_thresholds, thresholds, n_gt);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    if (n_gt_rows > 0) {
        thresholds_rank_kernel<<<dim3((unsigned)((n_gt_rows + 255) / 256), C), 256, 0, s>>>(compact, n_gt_rows, n_tp,
                                                                                            sel, n_thresholds,
                                                                                            thresholds);
        SB_LAUNCHED();
        SB_CHECK_LAUNCH();
    }
    match_curve_kernel<<<grid_ic, 32, kStageBytes, s>>>(gt, gt_code, det, det_code, gt_off, det_off, pair_off,
                                                        n_images, n_det_rows, ov_2d, ov_bev, ov_3d, d_bars, n_bars,
                                                        thresholds, n_thresholds, asg, counts, sims);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    curves_kernel<<<C, 64, 0, s>>>(n_images, counts, sims, n_thresholds, tp, fp, fn, sim, precision, recall, aos, ap);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}
