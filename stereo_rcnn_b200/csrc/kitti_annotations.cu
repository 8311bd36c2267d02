// kitti_annotations.cu -- the training ground truth of a KITTI split on the device: kitti_utils.read_obj_data's
// projection of every 3D box into both cameras (left, right and merged 2D boxes, four bottom-corner keypoints),
// kitti.remove_occluded_keypoints' occlusion reasoning along a 1260-column depth line (left camera, then right camera
// on the left pass's survivors) and _load_kitti_annotation's final filter.  One CTA per image; the restatement it
// follows, and oracle/kitti_annotations.py with it, is DESIGN.md §10.
//
// Every floating-point operation is an explicit fp64 round-to-nearest intrinsic in the oracle's order (no
// contraction), `int()` is round-toward-zero and Python's min / max are `b < a ? b : a` / `b > a ? b : a`, so the
// device and the oracle make the same decisions and write the same bits.
#include <limits.h>
#include <math.h>

#include "common.cuh"

namespace {

// input row fields (SB_KITTI_ANN_IN doubles per used label line)
constexpr int kTrunc = 0, kOcc = 1, kAlpha = 2, kW = 3, kH = 4, kL = 5, kX = 6, kY = 7, kZ = 8, kCos = 9, kSin = 10;
constexpr int kIn = SB_KITTI_ANN_IN;
constexpr int kOut = SB_KITTI_ANN_OUT;
constexpr int kCalib = SB_KITTI_ANN_CALIB;
constexpr int kCols = SB_KITTI_DEPTH_COLS;       // the reference's depth line, whatever the image width
// per-object state in the workspace (doubles): box[side][4], box_merge[4], kp[side][4], (vl, vr)[side], pos z
constexpr int kSBox = 0, kSMerge = 8, kSKp = 12, kSVis = 20, kSZ = 24, kState = 32;
constexpr int kThreads = 256, kWarps = kThreads / 32;

__device__ __forceinline__ double dmul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double dadd(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double dsub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double ddiv(double a, double b) { return __ddiv_rn(a, b); }
// Python's min(a, b) / max(a, b): the second argument only when strictly smaller / larger
__device__ __forceinline__ double pymin(double a, double b) { return b < a ? b : a; }
__device__ __forceinline__ double pymax(double a, double b) { return b > a ? b : a; }

// read_obj_data for one object: corners, both projections, boxes, keypoints and the merged box, into its state
__device__ void project_object(const double* r, const double* cal, int H, int W, double* st) {
    const double px = dadd(r[kX], cal[24]), py = dadd(r[kY], 0.0), pz = dadd(r[kZ], 0.0);
    const double c = r[kCos], s = r[kSin], w = r[kW], h = r[kH], l = r[kL];
    double cx[8], cy[8], cz[8];
    for (int k = 0; k < 8; ++k) {
        const double vx = (k & 3) < 2 ? -w : w;
        const double vz = ((k & 3) == 0 || (k & 3) == 3) ? -l : l;
        const double vy = k < 4 ? 0.0 : dmul(-2.0, h);
        // R = [[c, 0, s], [0, 1, 0], [-s, 0, c]]; R.v as (r0 vx + r1 vy) + r2 vz, then / 2, then + pos
        const double rx = dadd(dadd(dmul(c, vx), dmul(0.0, vy)), dmul(s, vz));
        const double ry = dadd(dadd(dmul(0.0, vx), dmul(1.0, vy)), dmul(0.0, vz));
        const double rz = dadd(dadd(dmul(-s, vx), dmul(0.0, vy)), dmul(c, vz));
        cx[k] = dadd(px, ddiv(rx, 2.0));
        cy[k] = dadd(py, ddiv(ry, 2.0));
        cz[k] = dadd(pz, ddiv(rz, 2.0));
    }
    for (int j = 0; j < 2; ++j) {
        const double* P = cal + 12 * j;
        double b0 = 10000.0, b1 = 10000.0, b2 = 0.0, b3 = 0.0;
        double kp[4] = {-1.0, -1.0, -1.0, -1.0};
        for (int k = 0; k < 8; ++k) {
            if (cz[k] < 0.0) continue;
            double n[3];
            for (int q = 0; q < 3; ++q)
                n[q] = dadd(dadd(dadd(dmul(P[4 * q], cx[k]), dmul(P[4 * q + 1], cy[k])), dmul(P[4 * q + 2], cz[k])),
                            P[4 * q + 3]);
            const double u = ddiv(n[0], n[2]), v = ddiv(n[1], n[2]);
            if (k < 4) kp[k] = u;
            b0 = pymin(b0, u);
            b1 = pymin(b1, v);
            b2 = pymax(b2, u);
            b3 = pymax(b3, v);
        }
        b0 = pymax(b0, 0.0);
        b1 = pymax(b1, 0.0);
        b2 = pymin(b2, (double)(W - 1));
        b3 = pymin(b3, (double)(H - 1));
        double lk = 5000.0, rk = 0.0;
        int li = -1, ri = -1;
        for (int k = 0; k < 4; ++k) {
            if (kp[k] < lk) { lk = kp[k]; li = k; }
            if (kp[k] > rk) { rk = kp[k]; ri = k; }
        }
        for (int k = 0; k < 4; ++k)
            if (k != li && k != ri && cz[k] > pz) kp[k] = -1.0;
        st[kSBox + 4 * j + 0] = b0;
        st[kSBox + 4 * j + 1] = b1;
        st[kSBox + 4 * j + 2] = b2;
        st[kSBox + 4 * j + 3] = b3;
        for (int k = 0; k < 4; ++k) st[kSKp + 4 * j + k] = kp[k];
    }
    for (int q = 0; q < 2; ++q) st[kSMerge + q] = pymin(st[kSBox + 4 + q], st[kSBox + q]);
    for (int q = 2; q < 4; ++q) st[kSMerge + q] = pymax(st[kSBox + 4 + q], st[kSBox + q]);
    st[kSZ] = pz;
}

// stable block-wide compaction of in[0..m) by pred(row) into out; every thread of the CTA calls it
template <class Pred>
__device__ int compact(const int* in, int m, int* out, Pred pred, int* s_warp) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int total = 0;
    for (int c0 = 0; c0 < m; c0 += kThreads) {
        const int k = c0 + threadIdx.x;
        const bool f = k < m && pred(in[k]);
        const unsigned b = __ballot_sync(0xffffffffu, f);
        if (lane == 0) s_warp[warp] = __popc(b);
        __syncthreads();
        int before = total, chunk = 0;
        for (int q = 0; q < kWarps; ++q) {
            if (q < warp) before += s_warp[q];
            chunk += s_warp[q];
        }
        if (f) out[before + __popc(b & ((1u << lane) - 1u))] = in[k];
        total += chunk;
        __syncthreads();
    }
    return total;
}

__global__ void __launch_bounds__(kThreads) annotations_kernel(
    const double* __restrict__ rows, const int* __restrict__ codes, const long long* __restrict__ obj_off,
    const double* __restrict__ calib, const int* __restrict__ image_hw, double* __restrict__ state, int* list_a,
    int* list_b, float* __restrict__ out, int* __restrict__ n_kept, int* __restrict__ status) {
    __shared__ double depth[kCols];
    __shared__ int s_warp[kWarps];
    __shared__ int s_fail[2];
    const int img = blockIdx.x;
    const long long base = obj_off[img];
    const int n = (int)(obj_off[img + 1] - base);
    const int H = image_hw[2 * img], W = image_hw[2 * img + 1];
    const double* cal = calib + (size_t)img * kCalib;
    double* st = state + (size_t)base * kState;
    const double* in = rows + (size_t)base * kIn;
    int* la = list_a + base;
    int* lb = list_b + base;
    float* o = out + (size_t)base * kOut;
    int m = 0, st_code = 0;
    if (H <= 0 || W <= 0) {
        st_code = -1;
    } else {
        for (int j = threadIdx.x; j < n; j += kThreads) {
            project_object(in + (size_t)j * kIn, cal, H, W, st + (size_t)j * kState);
            la[j] = j;
        }
        m = n;
        __syncthreads();
        int* lists[2] = {la, lb};
        for (int side = 0; side < 2 && st_code == 0; ++side) {
            const int* cur = lists[side];
            int* nxt = lists[side ^ 1];
            // the reference's IndexError: painting runs first over every object, then the two end lookups
            if (threadIdx.x < 2) s_fail[threadIdx.x] = INT_MAX;
            __syncthreads();
            for (int k = threadIdx.x; k < m; k += kThreads) {
                const double* so = st + (size_t)cur[k] * kState + kSBox + 4 * side;
                // int() of the untruncated ends (x1 in [0, 10000], x2 in [0, W - 1]): a box wholly right of the line
                // (x1 > x2 >= 1260) paints nothing and fails only at its end lookups
                const double c1 = trunc(so[0]), c2 = trunc(so[2]);
                if (c1 <= c2 && c2 >= (double)kCols) atomicMin(&s_fail[0], cur[k]);
                if (c1 >= (double)kCols || c2 >= (double)kCols) atomicMin(&s_fail[1], cur[k]);
            }
            __syncthreads();
            const int fail = s_fail[0] != INT_MAX ? s_fail[0] : s_fail[1];
            if (fail != INT_MAX) {
                st_code = 1 + fail;
                break;
            }
            // painting: threads own columns and walk the objects in order
            for (int col = threadIdx.x; col < kCols; col += kThreads) {
                double d = 0.0;
                for (int k = 0; k < m; ++k) {
                    const double* so = st + (size_t)cur[k] * kState;
                    const int c1 = (int)so[kSBox + 4 * side], c2 = (int)so[kSBox + 4 * side + 2];
                    if (col < c1 || col > c2) continue;
                    const double z = so[kSZ];
                    if (d == 0.0) d = z;
                    else if (z < d) d = ddiv(dadd(z, d), 2.0);
                }
                depth[col] = d;
            }
            __syncthreads();
            // visible range: one warp per object, the last matching column wins
            const int lane = threadIdx.x & 31;
            for (int k = threadIdx.x >> 5; k < m; k += kWarps) {
                double* so = st + (size_t)cur[k] * kState;
                const double x1 = so[kSBox + 4 * side], x2 = so[kSBox + 4 * side + 2], z = so[kSZ];
                const int c1 = (int)x1, c2 = (int)x2;
                const bool lv = !(depth[c1] < z), rv = !(depth[c2] < z);
                int best_r = -1, best_l = -1;
                for (int col = c1 + lane; col <= c2; col += 32) {
                    const double d = depth[col];
                    const bool a = lv && d >= z;
                    if (a) best_r = col;
                    else if (rv && d < z) best_l = col;
                }
                for (int sh = 16; sh > 0; sh >>= 1) {
                    best_r = max(best_r, __shfl_xor_sync(0xffffffffu, best_r, sh));
                    best_l = max(best_l, __shfl_xor_sync(0xffffffffu, best_l, sh));
                }
                if (lane == 0) {
                    double vl = x1, vr = x2;
                    if (!lv && !rv) {
                        vr = x1;
                        for (int q = 0; q < 4; ++q) so[kSKp + 4 * side + q] = -1.0;
                    }
                    if (best_r >= 0) vr = (double)best_r;
                    if (best_l >= 0) vl = (double)best_l;
                    so[kSVis + 2 * side] = vl;
                    so[kSVis + 2 * side + 1] = vr;
                }
            }
            __syncthreads();
            m = compact(cur, m, nxt, [&](int r) {
                const double* kp = st + (size_t)r * kState + kSKp + 4 * side;
                return dadd(dadd(dadd(kp[0], kp[1]), kp[2]), kp[3]) > -4.0;
            }, s_warp);
            // keypoint pruning on the survivors
            for (int k = threadIdx.x; k < m; k += kThreads) {
                double* so = st + (size_t)nxt[k] * kState;
                double* kp = so + kSKp + 4 * side;
                const double vl = so[kSVis + 2 * side], vr = so[kSVis + 2 * side + 1];
                double lk = 5000.0, rk = 0.0;
                for (int q = 0; q < 4; ++q)
                    if (kp[q] != -1.0) {
                        if (kp[q] < lk) lk = kp[q];
                        if (kp[q] > rk) rk = kp[q];
                    }
                for (int q = 0; q < 4; ++q)
                    if (kp[q] != -1.0 && (kp[q] < dsub(vl, 5.0) || kp[q] > dadd(vr, 5.0) || kp[q] < dadd(lk, 3.0) ||
                                          kp[q] > dsub(rk, 3.0)))
                        kp[q] = -1.0;
            }
            __syncthreads();
        }
        if (st_code == 0) {
            // _load_kitti_annotation's filter over the right pass's survivors (list_a), kept rows into list_b
            m = compact(la, m, lb, [&](int r) {
                const double* ro = in + (size_t)r * kIn;
                const double* so = st + (size_t)r * kState;
                return ro[kTrunc] < 0.98 && ro[kOcc] < 3.0 && dsub(so[kSBox + 3], so[kSBox + 1]) > 10.0 &&
                       codes[base + r] == 0 && dsub(so[kSVis + 1], so[kSVis]) > 3.0 &&
                       dsub(so[kSVis + 3], so[kSVis + 2]) > 3.0;
            }, s_warp);
        } else {
            m = 0;
        }
    }
    // kept rows in label order, then zeros up to the image's row count
    for (int k = threadIdx.x; k < n; k += kThreads) {
        float* d = o + (size_t)k * kOut;
        if (k < m) {
            const int r = lb[k];
            const double* ro = in + (size_t)r * kIn;
            const double* so = st + (size_t)r * kState;
            for (int q = 0; q < 12; ++q) d[q] = __double2float_rn(so[kSBox + q]);   // left, right, merge
            d[12] = __double2float_rn(ro[kW]);
            d[13] = __double2float_rn(ro[kH]);
            d[14] = __double2float_rn(ro[kL]);
            d[15] = __double2float_rn(ro[kAlpha]);
            for (int j = 0; j < 2; ++j) {
                for (int q = 0; q < 4; ++q) d[16 + 6 * j + q] = __double2float_rn(so[kSKp + 4 * j + q]);
                d[20 + 6 * j] = __double2float_rn(so[kSVis + 2 * j]);
                d[21 + 6 * j] = __double2float_rn(so[kSVis + 2 * j + 1]);
            }
            d[28] = __double2float_rn(ro[kTrunc]);
            d[29] = __double2float_rn(ro[kOcc]);
        } else {
            for (int q = 0; q < kOut; ++q) d[q] = 0.0f;
        }
    }
    if (threadIdx.x == 0) {
        n_kept[img] = m;
        status[img] = st_code;
    }
}

struct Ws {
    size_t state, list_a, list_b, total;
};

static size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

static Ws ws_layout(long long n_rows) {
    Ws w;
    size_t o = 0;
    w.state = o;  o = align256(o + (size_t)n_rows * kState * sizeof(double));
    w.list_a = o; o = align256(o + (size_t)n_rows * sizeof(int));
    w.list_b = o; o = align256(o + (size_t)n_rows * sizeof(int));
    w.total = o > 256 ? o : 256;                    // nonzero for a split without used rows
    return w;
}

static bool sizes_ok(int n_images, long long n_rows) { return n_images >= 1 && n_rows >= 0 && n_rows < (1LL << 31); }

}  // namespace

extern "C" size_t sb_kitti_annotations_workspace_bytes(int n_images, long long n_rows) {
    if (!sizes_ok(n_images, n_rows)) return 0;
    return ws_layout(n_rows).total;
}

extern "C" int sb_kitti_annotations(const double* rows, const int* codes, const long long* obj_off,
                                    const double* calib, const int* image_hw, int n_images, long long n_rows,
                                    void* workspace, size_t workspace_bytes, float* out, int* n_kept, int* status,
                                    sb_stream_t stream) {
    if (!obj_off || !calib || !image_hw || !workspace || !n_kept || !status || !sizes_ok(n_images, n_rows))
        return SB_EINVAL;
    if (n_rows > 0 && (!rows || !codes || !out)) return SB_EINVAL;
    const Ws L = ws_layout(n_rows);
    if (workspace_bytes < L.total || ((uintptr_t)workspace & 255)) return SB_EINVAL;
    char* w = static_cast<char*>(workspace);
    annotations_kernel<<<n_images, kThreads, 0, sb_cs(stream)>>>(
        rows, codes, obj_off, calib, image_hw, reinterpret_cast<double*>(w + L.state),
        reinterpret_cast<int*>(w + L.list_a), reinterpret_cast<int*>(w + L.list_b), out, n_kept, status);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}
