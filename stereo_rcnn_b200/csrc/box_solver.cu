// box_solver.cu -- the CPU stage between the network and dense_align, on the device (SURVEY 8f-1).
//
// Replaces, per image, test_net.py:262-325's Python loop:
//   infer_boundary            (lib/model/utils/kitti_utils.py:398-437)     -> infer_boundary_kernel
//   keypoint border fix-up    (test_net.py:263-266)                        \
//   solve_x_y_z_theta_from_kpt (box_estimator.py:169-385, scipy Newton-CG)  > box_solve_kernel (+ ordered compaction
//   boxes_all / kpts_all / poses_all concatenation (test_net.py:281-303)   /   of the solved detections)
//   solve_x_y_theta_from_kpt  (box_estimator.py:387-545) after dense_align -> box_rectify_kernel
// so that dense_align consumes the solver's poses without a device->host->device round trip and without ~2 x D scipy
// calls on the host.  The numerics (problem set-up, residuals, Levenberg-Marquardt in fp64) live in
// box_solver_core.h, shared with a host harness that checks them against scipy and the reference goldens.
// One thread per detection: D <= 512 and each solve is a few dozen 4x4 systems -- latency, not throughput.
#include "box_solver_core.h"
#include "common.cuh"

namespace {

constexpr int kMaxDet = 512;
constexpr int kMaxWidth = 4094;      // depth_line lives in static shared memory (KITTI frames are 1242 wide)

// depth_line painting is order dependent across detections (kept order = score desc) but independent per column:
// thread per column walks the detections; then thread per detection derives its visible span.
__global__ void __launch_bounds__(1024)
infer_boundary_kernel(const float* __restrict__ boxes /*[R, ld]*/, int ld, int coff, const int* __restrict__ keep,
                      const int* __restrict__ num, int im_w, float* __restrict__ left_right /*[R,2] by kept index*/) {
    __shared__ double depth_line[kMaxWidth + 2];
    const int n = min(*num, kMaxDet);
    for (int col = threadIdx.x; col <= im_w; col += blockDim.x) {
        double dl = 0.0;
        for (int i = 0; i < n; ++i) {
            const float* b = boxes + (size_t)keep[i] * ld + coff;
            if (col < (int)b[0] || col > (int)b[2]) continue;
            const double depth = 1050.0 / (double)b[3];
            if (dl == 0.0) dl = depth;
            else if (depth < dl) dl = (depth + dl) / 2.0;
        }
        depth_line[col] = dl;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float* b = boxes + (size_t)keep[i] * ld + coff;
        const double depth = 1050.0 / (double)b[3];
        float l0 = b[0], l1 = b[2];
        const int c0 = (int)b[0], c1 = (int)b[2];
        const bool left_visible = !(depth_line[c0] < depth), right_visible = !(depth_line[c1] < depth);
        if (!right_visible && !left_visible) l1 = b[0];
        for (int col = c0; col <= c1; ++col) {
            if (left_visible && depth_line[col] >= depth) l1 = (float)col;
            else if (right_visible && depth_line[col] < depth) l0 = (float)col;
        }
        left_right[2 * i] = l0;
        left_right[2 * i + 1] = l1;
    }
}

struct SolveArgs {
    const float *scores, *boxes_l, *boxes_r, *dim_orien, *kpts;   // [R,nc], [R,4nc], [R,4nc], [R,5nc], [R,5]
    const int *keep, *num;
    const float* inferred;       // [R,2] or null
    int nc, cls, im_h, im_w;
    double p2[12], p3[12];
    float eval_thresh;
};

// DEV_CALIB: the calibration is read from device memory, `calib` = P2 then P3 (24 row-major doubles), so that a
// captured launch uses whatever was last written there; otherwise it is a.p2 / a.p3 (kernel arguments).
// one CTA: thread i solves kept detection i, then the solved ones are compacted in order
template <bool DEV_CALIB>
__global__ void __launch_bounds__(kMaxDet)
box_solve_kernel(SolveArgs a, int cap, float* __restrict__ boxes_all /*[cap,5]*/, float* __restrict__ kpts_all /*[cap,5]*/,
                 float* __restrict__ poses_all /*[cap,8]*/, int* __restrict__ src_index /*[cap]*/, int* __restrict__ n_out,
                 const double* __restrict__ calib /*[24], DEV_CALIB only*/) {
    __shared__ int warp_cnt[kMaxDet / 32];
    const int i = threadIdx.x;
    const int n = min(*a.num, kMaxDet);
    bool ok = false;
    float box[5], kp[5], pose[8];
    int r = -1;
    if (i < n) {
        r = a.keep[i];
        const float score = a.scores[(size_t)r * a.nc + a.cls];
        const float* bl = a.boxes_l + (size_t)r * 4 * a.nc + 4 * a.cls;
        const float* br = a.boxes_r + (size_t)r * 4 * a.nc + 4 * a.cls;
        const float* dm = a.dim_orien + (size_t)r * 5 * a.nc + 5 * a.cls;
#pragma unroll
        for (int q = 0; q < 5; ++q) kp[q] = a.kpts[(size_t)r * 5 + q];
        if (a.inferred) {        // test_net.py:263-266
            const float i0 = a.inferred[2 * i], i1 = a.inferred[2 * i + 1];
            if (__fsub_rn(kp[4], kp[3]) < __fmul_rn(0.5f, __fsub_rn(i1, i0))) { kp[3] = i0; kp[4] = i1; }
        }
        box[0] = bl[0]; box[1] = bl[1]; box[2] = bl[2]; box[3] = bl[3]; box[4] = score;
        if (score > a.eval_thresh && !sb_box_rejected(box, kp)) {
            const double alpha = atan2((double)dm[3], (double)dm[4]);
            const double dim[3] = {dm[0], dm[1], dm[2]};
            const double bld[4] = {box[0], box[1], box[2], box[3]}, brd[4] = {br[0], br[1], br[2], br[3]};
            const double kpd[5] = {kp[0], kp[1], kp[2], kp[3], kp[4]};
            SbBoxProblem pb;
            sb_box_problem(&pb, a.im_h, a.im_w, DEV_CALIB ? calib : a.p2, DEV_CALIB ? calib + 12 : a.p3, alpha, dim, bld, brd, kpd, 0, 0.0);
            double s[4];
            sb_box_init(pb, s);
            sb_box_lm(pb, s);
            ok = isfinite(s[0]) && isfinite(s[1]) && isfinite(s[2]) && isfinite(s[3]) && !(s[2] > 100);   // box_estimator.py:383-385
            pose[0] = (float)s[0]; pose[1] = (float)s[1]; pose[2] = (float)s[2];
            pose[3] = dm[0]; pose[4] = dm[1]; pose[5] = dm[2];
            pose[6] = (float)s[3]; pose[7] = (float)alpha;
        }
    }
    // ordered compaction (test_net.py:300-303 appends the solved detections in order)
    const unsigned bal = __ballot_sync(0xffffffffu, ok);
    const int lane = i & 31, warp = i >> 5;
    if (lane == 0) warp_cnt[warp] = __popc(bal);
    __syncthreads();
    int base = 0;
    for (int w = 0; w < warp; ++w) base += warp_cnt[w];
    const int slot = base + __popc(bal & ((1u << lane) - 1u));
    if (ok && slot < cap) {
#pragma unroll
        for (int q = 0; q < 5; ++q) { boxes_all[5 * slot + q] = box[q]; kpts_all[5 * slot + q] = kp[q]; }
#pragma unroll
        for (int q = 0; q < 8; ++q) poses_all[8 * slot + q] = pose[q];
        src_index[slot] = r;
    }
    if (i == 0) {
        int tot = 0;
        for (int w = 0; w < kMaxDet / 32; ++w) tot += warp_cnt[w];
        *n_out = min(tot, cap);
    }
}

// after dense_align: rectified pose per solved detection (test_net.py:311-325); DEV_CALIB as in box_solve_kernel
template <bool DEV_CALIB>
__global__ void __launch_bounds__(128)
box_rectify_kernel(const float* __restrict__ boxes_all, const float* __restrict__ kpts_all,
                   const float* __restrict__ poses_all, const float* __restrict__ succ, const float* __restrict__ dis,
                   const int* __restrict__ n_in, int im_h, int im_w, SolveArgs a, double* __restrict__ final_out /*[cap,13]*/,
                   const double* __restrict__ calib /*[24], DEV_CALIB only*/) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *n_in) return;
    double* o = final_out + (size_t)i * 13;
    o[0] = 0.0;
    if (!(succ[i] > 0.f)) return;
    const float* b = boxes_all + 5 * i;
    const float* kp = kpts_all + 5 * i;
    const float* ps = poses_all + 8 * i;
    const double dim[3] = {ps[3], ps[4], ps[5]};
    const double bld[4] = {b[0], b[1], b[2], b[3]};
    const double kpd[5] = {kp[0], kp[1], kp[2], kp[3], kp[4]};
    SbBoxProblem pb;
    sb_box_problem(&pb, im_h, im_w, DEV_CALIB ? calib : a.p2, DEV_CALIB ? calib + 12 : a.p3, (double)ps[7], dim, bld, bld, kpd, 1, (double)dis[i]);
    double s[4];
    sb_box_init(pb, s);
    sb_box_lm(pb, s);
    o[0] = 1.0; o[1] = b[4];
    o[2] = b[0]; o[3] = b[1]; o[4] = b[2]; o[5] = b[3];
    o[6] = s[0]; o[7] = s[1]; o[8] = pb.z_fixed;
    o[9] = dim[0]; o[10] = dim[1]; o[11] = dim[2];
    o[12] = s[3];
}

void fill_args(SolveArgs* a, const double* p2, const double* p3) {
    for (int i = 0; i < 12; ++i) { a->p2[i] = p2[i]; a->p3[i] = p3[i]; }
}

}  // namespace

extern "C" int sb_infer_boundary(const float* boxes, int ld, int col_offset, const int* keep, const int* num, int im_w,
                                 float* left_right, sb_stream_t stream) {
    if (!boxes || !keep || !num || !left_right || im_w < 1 || im_w > kMaxWidth || ld < col_offset + 4) return SB_EINVAL;
    infer_boundary_kernel<<<1, 1024, 0, sb_cs(stream)>>>(boxes, ld, col_offset, keep, num, im_w, left_right);
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

// host-calibrated (p2, p3) or device-calibrated (dcalib) launches share the argument checks and the launch
static int box_solve_launch(const float* scores, const float* boxes_left, const float* boxes_right,
                            const float* dim_orien, const float* kpts, const int* keep, const int* num,
                            const float* inferred, int n_classes, int cls, int im_h, int im_w, const double* p2,
                            const double* p3, const double* dcalib, float eval_thresh, int cap, float* boxes_all,
                            float* kpts_all, float* poses_all, int* src_index, int* n_out, sb_stream_t stream) {
    if (!scores || !boxes_left || !boxes_right || !dim_orien || !kpts || !keep || !num || !boxes_all ||
        !kpts_all || !poses_all || !src_index || !n_out || cap < 1 || cls < 0 || cls >= n_classes)
        return SB_EINVAL;
    SolveArgs a = {};
    a.scores = scores; a.boxes_l = boxes_left; a.boxes_r = boxes_right; a.dim_orien = dim_orien; a.kpts = kpts;
    a.keep = keep; a.num = num; a.inferred = inferred; a.nc = n_classes; a.cls = cls; a.im_h = im_h; a.im_w = im_w;
    a.eval_thresh = eval_thresh;
    if (dcalib) {
        box_solve_kernel<true><<<1, kMaxDet, 0, sb_cs(stream)>>>(a, cap, boxes_all, kpts_all, poses_all, src_index,
                                                                 n_out, dcalib);
    } else {
        fill_args(&a, p2, p3);
        box_solve_kernel<false><<<1, kMaxDet, 0, sb_cs(stream)>>>(a, cap, boxes_all, kpts_all, poses_all, src_index,
                                                                  n_out, nullptr);
    }
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

static int box_rectify_launch(const float* boxes_all, const float* kpts_all, const float* poses_all, const float* succ,
                              const float* best_dis, const int* n, int cap, int im_h, int im_w, const double* p2,
                              const double* p3, const double* dcalib, double* final_out, sb_stream_t stream) {
    if (!boxes_all || !kpts_all || !poses_all || !succ || !best_dis || !n || !final_out || cap < 1)
        return SB_EINVAL;
    SolveArgs a = {};
    if (dcalib) {
        box_rectify_kernel<true><<<sb_div_up(cap, 128), 128, 0, sb_cs(stream)>>>(
            boxes_all, kpts_all, poses_all, succ, best_dis, n, im_h, im_w, a, final_out, dcalib);
    } else {
        fill_args(&a, p2, p3);
        box_rectify_kernel<false><<<sb_div_up(cap, 128), 128, 0, sb_cs(stream)>>>(
            boxes_all, kpts_all, poses_all, succ, best_dis, n, im_h, im_w, a, final_out, nullptr);
    }
    SB_LAUNCHED();
    SB_CHECK_LAUNCH();
    return SB_OK;
}

extern "C" int sb_box_solve(const float* scores, const float* boxes_left, const float* boxes_right,
                            const float* dim_orien, const float* kpts, const int* keep, const int* num,
                            const float* inferred, int n_classes, int cls, int im_h, int im_w, const double* p2,
                            const double* p3, float eval_thresh, int cap, float* boxes_all, float* kpts_all,
                            float* poses_all, int* src_index, int* n_out, sb_stream_t stream) {
    if (!p2 || !p3) return SB_EINVAL;
    return box_solve_launch(scores, boxes_left, boxes_right, dim_orien, kpts, keep, num, inferred, n_classes, cls, im_h,
                            im_w, p2, p3, nullptr, eval_thresh, cap, boxes_all, kpts_all, poses_all, src_index, n_out,
                            stream);
}

extern "C" int sb_box_solve_devcalib(const float* scores, const float* boxes_left, const float* boxes_right,
                                     const float* dim_orien, const float* kpts, const int* keep, const int* num,
                                     const float* inferred, int n_classes, int cls, int im_h, int im_w,
                                     const double* calib, float eval_thresh, int cap, float* boxes_all,
                                     float* kpts_all, float* poses_all, int* src_index, int* n_out,
                                     sb_stream_t stream) {
    if (!calib) return SB_EINVAL;
    return box_solve_launch(scores, boxes_left, boxes_right, dim_orien, kpts, keep, num, inferred, n_classes, cls, im_h,
                            im_w, nullptr, nullptr, calib, eval_thresh, cap, boxes_all, kpts_all, poses_all, src_index,
                            n_out, stream);
}

extern "C" int sb_box_rectify(const float* boxes_all, const float* kpts_all, const float* poses_all, const float* succ,
                              const float* best_dis, const int* n, int cap, int im_h, int im_w, const double* p2,
                              const double* p3, double* final_out, sb_stream_t stream) {
    if (!p2 || !p3) return SB_EINVAL;
    return box_rectify_launch(boxes_all, kpts_all, poses_all, succ, best_dis, n, cap, im_h, im_w, p2, p3, nullptr,
                              final_out, stream);
}

extern "C" int sb_box_rectify_devcalib(const float* boxes_all, const float* kpts_all, const float* poses_all,
                                       const float* succ, const float* best_dis, const int* n, int cap, int im_h,
                                       int im_w, const double* calib, double* final_out, sb_stream_t stream) {
    if (!calib) return SB_EINVAL;
    return box_rectify_launch(boxes_all, kpts_all, poses_all, succ, best_dis, n, cap, im_h, im_w, nullptr, nullptr,
                              calib, final_out, stream);
}
