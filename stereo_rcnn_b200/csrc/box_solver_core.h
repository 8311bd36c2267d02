// box_solver_core.h -- the 3D box least-squares problems of lib/model/utils/box_estimator.py as plain
// host/device C++ (no CUDA dependencies), shared by the device kernels (box_solver.cu) and by a host test harness
// (tests/tools/box_solver_host.cpp, compiled with g++) that checks the numerics without a GPU.
//
//   solve_x_y_z_theta_from_kpt (box_estimator.py:169-385): states (x, y, z, theta), residuals
//       r0 left u, r1 right u, r2 keypoint u (x2), r3 bottom v, r4 top v, r5 viewpoint angle, r6 / r7 left / right u of
//       the right box; which ones are live depends on truncation (box_estimator.py:251-269).
//   solve_x_y_theta_from_kpt   (box_estimator.py:387-545): states (x, y, theta), z fixed by the aligned disparity,
//       residuals r0..r5.
//
// The reference minimises sum r_i^2 with scipy's Newton-CG and ITS analytic gradient j_kpt / j_rect, in which the
// keypoint term is 2*(2 rho)*rho' (box_estimator.py:236,292-297: res_uk is doubled before it is used, the factor of
// the doubling itself is not applied) -- the gradient of sum_{i != 2} r_i^2 + 2 rho^2.  Newton-CG iterates on that
// gradient, so its fixed points are the minima of THAT function; here it is minimised directly, by Levenberg-Marquardt
// on the residual vector with the keypoint residual scaled by sqrt(2), in fp64, to a tight tolerance (Newton-CG itself
// stops on a step-size test and its end point moves by centimetres with the rounding of its inputs).
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define SB_HD __host__ __device__ __forceinline__
#else
#define SB_HD inline
#endif

struct SbBoxProblem {
    double left_u, right_u, top_v, bottom_v, kpt_u, left_u_r, right_u_r;
    double alpha, bl, h, f;
    double vw[4], vl[4];     // (w, l) offsets of the left, right, bottom, keypoint vertices
    int on[8];               // live residuals
    int rect;                // 1: z fixed (solve_x_y_theta_from_kpt)
    int truncation;
    double z_fixed, disparity;
};

// box_estimator.py:187's rejection rules on the float32 box [x1,y1,x2,y2] and keypoints [.., left border, right
// border]: 1 = not solved.  test_net.py passes the box as a float32 numpy row and the keypoints as a float32 torch row,
// so each difference is rounded to float32 before it is compared: a difference just below the threshold can round up
// to it, and then the reference solves the detection.  __fsub_rn keeps the device from contracting or widening it.
SB_HD int sb_box_rejected(const float* box, const float* kp) {
#if defined(__CUDA_ARCH__)
    return __fsub_rn(kp[4], kp[3]) < 3.f || __fsub_rn(box[2], box[0]) < 10.f || __fsub_rn(box[3], box[1]) < 10.f;
#else
    return kp[4] - kp[3] < 3.f || box[2] - box[0] < 10.f || box[3] - box[1] < 10.f;
#endif
}

SB_HD int sb_bb2viewpoint(double alpha) {       // box_estimator.py:15-42
    const double kPi = 3.141592653589793;
    alpha = alpha * 180.0 / kPi;
    if (alpha > 360) alpha -= 360;
    else if (alpha < -360) alpha += 360;
    const double t = 4.0;
    if (alpha >= -90.0 - t && alpha <= -90.0 + t) return 0;
    if (alpha >= -180.0 + t && alpha <= -90.0 - t) return 1;
    if (alpha >= 180.0 - t || alpha <= -180.0 + t) return 2;
    if (alpha >= 90.0 + t && alpha <= 180.0 - t) return 3;
    if (alpha >= 90.0 - t && alpha <= 90.0 + t) return 4;
    if (alpha >= 0.0 + t && alpha <= 90.0 - t) return 5;
    if (alpha >= 0.0 - t && alpha <= 0.0 + t) return 6;
    if (alpha >= -90.0 + t && alpha <= 0.0 - t) return 7;
    return -1;
}

SB_HD double sb_kpt2alpha(double kpt_pos, int kpt_type, double box0, double box2) {    // box_estimator.py:148-167
    const double kPi = 3.141592653589793;
    double q = (kpt_pos - box0) / (box2 - box0);
    q = q > 1.0 ? 1.0 : (q < -1.0 ? -1.0 : q);
    const double r = asin(q);
    switch (kpt_type) {
        case 0: return -kPi / 2 - r;
        case 1: return kPi - r;
        case 2: return kPi / 2 - r;
        default: return -r;
    }
}

// im_h, im_w: the ORIGINAL image size (im2show_left.shape); p2 / p3: 3x4 row-major; alpha: viewpoint angle;
// dim (w,h,l); boxes [x1,y1,x2,y2]; kpts [u, type, conf, left border, right border]; disparity only for rect
SB_HD void sb_box_problem(SbBoxProblem* pb, int im_h, int im_w, const double* p2, const double* p3, double alpha,
                          const double* dim, const double* box_left, const double* box_right, const double* kpts,
                          int rect, double disparity) {
    const double tb = 10.0;                                   // truncate_border
    const int kpt_type = (int)kpts[1];
    const double w = dim[0], l = dim[2];
    const double ul = box_left[0], ur = box_left[2], vt = box_left[1], vb = box_left[3];
    const double f = p2[0], cx = p2[2], cy = p2[6];
    pb->f = f;
    pb->bl = (p2[3] - p3[3]) / f;
    pb->h = dim[1];
    pb->left_u = (ul - cx) / f;
    pb->right_u = (ur - cx) / f;
    pb->top_v = (vt - cy) / f;
    pb->bottom_v = (vb - cy) / f;
    pb->kpt_u = (kpts[0] - cx) / f;
    pb->truncation = (ul < 2.0 * tb || ur > im_w - 2.0 * tb) ? 1 : 0;
    pb->alpha = pb->truncation ? alpha : sb_kpt2alpha(kpts[0], kpt_type, box_left[0], box_left[2]);
    // viewpoint -> (left, right, bottom) vertices, box_estimator.py:93-123; signs of (w, l)
    const int vp = sb_bb2viewpoint(pb->alpha);
    int sg[3][2];
    switch (vp) {
        case 0: sg[0][0] = -1; sg[0][1] = -1; sg[1][0] = 1;  sg[1][1] = -1; sg[2][0] = 1;  sg[2][1] = -1; break;
        case 1: sg[0][0] = -1; sg[0][1] = 1;  sg[1][0] = 1;  sg[1][1] = -1; sg[2][0] = -1; sg[2][1] = -1; break;
        case 2: sg[0][0] = -1; sg[0][1] = 1;  sg[1][0] = -1; sg[1][1] = -1; sg[2][0] = -1; sg[2][1] = -1; break;
        case 3: sg[0][0] = 1;  sg[0][1] = 1;  sg[1][0] = -1; sg[1][1] = -1; sg[2][0] = -1; sg[2][1] = 1;  break;
        case 4: sg[0][0] = 1;  sg[0][1] = 1;  sg[1][0] = -1; sg[1][1] = 1;  sg[2][0] = -1; sg[2][1] = 1;  break;
        case 5: sg[0][0] = 1;  sg[0][1] = -1; sg[1][0] = -1; sg[1][1] = 1;  sg[2][0] = 1;  sg[2][1] = 1;  break;
        case 6: sg[0][0] = 1;  sg[0][1] = -1; sg[1][0] = 1;  sg[1][1] = 1;  sg[2][0] = 1;  sg[2][1] = 1;  break;
        default: sg[0][0] = -1; sg[0][1] = -1; sg[1][0] = 1; sg[1][1] = 1;  sg[2][0] = 1;  sg[2][1] = -1; break;
    }
    for (int i = 0; i < 3; ++i) { pb->vw[i] = sg[i][0] * w / 2; pb->vl[i] = sg[i][1] * l / 2; }
    const int ks[4][2] = {{-1, -1}, {-1, 1}, {1, 1}, {1, -1}};       // kpt2vertex, box_estimator.py:139-146
    const int kt = kpt_type < 0 ? 0 : (kpt_type > 3 ? 3 : kpt_type);
    pb->vw[3] = ks[kt][0] * w / 2;
    pb->vl[3] = ks[kt][1] * l / 2;
    pb->on[0] = !(ul < 2.0 * tb);
    pb->on[1] = !(ur > im_w - 2.0 * tb);
    pb->on[2] = !pb->truncation;
    pb->on[3] = !(vb > im_h - tb);
    pb->on[4] = !(vt < tb);
    pb->on[5] = pb->truncation;
    pb->on[6] = pb->on[7] = 0;
    pb->rect = rect;
    pb->left_u_r = pb->right_u_r = 0.0;
    pb->z_fixed = 0.0;
    pb->disparity = disparity;
    if (rect) {
        pb->z_fixed = f * pb->bl / disparity;
    } else {
        const double ul_r = box_right[0], ur_r = box_right[2];
        pb->left_u_r = (ul_r - cx) / f;
        pb->right_u_r = (ur_r - cx) / f;
        pb->on[6] = pb->truncation && !(ul_r < 2.0 * tb);
        pb->on[7] = pb->truncation && !(ur_r > im_w - 2.0 * tb);
        pb->disparity = (box_left[0] + box_left[2]) / 2 - (box_right[0] + box_right[2]) / 2;
    }
}

// residuals and Jacobian wrt (x, y, z, theta) at s = (x, y, z, theta); kpt_scale multiplies the keypoint residual
// (2 = the reference's objective f_kpt; sqrt 2 = the function whose gradient the reference's j_kpt is)
SB_HD void sb_box_residuals(const SbBoxProblem& pb, const double* s, double kpt_scale, double* r, double* J /*[8][4]*/) {
    const double kPi = 3.141592653589793;
    const double x = s[0], y = s[1], z = s[2], th = s[3];
    const double c = cos(th), sn = sin(th);
    for (int i = 0; i < 8; ++i) { r[i] = 0.0; J[4 * i] = J[4 * i + 1] = J[4 * i + 2] = J[4 * i + 3] = 0.0; }
    const int vert[8] = {0, 1, 3, -1, -1, -1, 0, 1};
    const double meas[8] = {pb.left_u, pb.right_u, pb.kpt_u, 0, 0, 0, pb.left_u_r, pb.right_u_r};
    for (int i = 0; i < 8; ++i) {
        if (vert[i] < 0 || !pb.on[i]) continue;
        const double vw = pb.vw[vert[i]], vl = pb.vl[vert[i]];
        const double sc = i == 2 ? kpt_scale : 1.0;
        const double xo = i >= 6 ? -pb.bl : 0.0;
        const double den = z - sn * vw + c * vl;
        const double num = x + xo + c * vw + sn * vl;
        r[i] = sc * (num / den - meas[i]);
        J[4 * i + 0] = sc / den;
        J[4 * i + 2] = -sc * num / (den * den);
        J[4 * i + 3] = sc * ((vl * c - vw * sn) / den + (vw * c + vl * sn) * num / (den * den));
    }
    const double bw = pb.vw[2], bl_ = pb.vl[2];
    if (pb.on[3]) {
        const double den = z - sn * bw + c * bl_;
        r[3] = y / den - pb.bottom_v;
        J[13] = 1.0 / den; J[14] = -y / (den * den); J[15] = y * (bw * c + bl_ * sn) / (den * den);
    }
    if (pb.on[4]) {
        const double den = z + sn * bw - c * bl_;
        r[4] = (y - pb.h) / den - pb.top_v;
        J[17] = 1.0 / den; J[18] = (pb.h - y) / (den * den); J[19] = (pb.h - y) * (bw * c + bl_ * sn) / (den * den);
    }
    if (pb.on[5]) {
        r[5] = th - kPi / 2 + atan2(-x, z) - pb.alpha;
        const double q = 1.0 / (1.0 + (x / z) * (x / z));
        J[20] = q * (-1.0 / z); J[22] = q * (x / (z * z)); J[23] = 1.0;
    }
}

SB_HD double sb_box_objective(const SbBoxProblem& pb, const double* s, double kpt_scale) {
    double r[8], J[32];
    sb_box_residuals(pb, s, kpt_scale, r, J);
    double f = 0.0;
    for (int i = 0; i < 8; ++i) f += r[i] * r[i];
    return f;
}

// initial state (box_estimator.py:376-379 / 540-542) -> s[4] (z = z_fixed for the rect problem)
SB_HD void sb_box_init(const SbBoxProblem& pb, double* s) {
    const double kPi = 3.141592653589793;
    const double z = pb.rect ? pb.z_fixed : pb.f * pb.bl / pb.disparity;
    s[0] = z * (pb.left_u + pb.right_u) / 2.0;
    s[1] = z * (pb.bottom_v + pb.top_v) / 2.0 + pb.h / 2.0;
    s[2] = z;
    s[3] = pb.alpha + kPi / 2 - atan2(-s[0], z);
}

// Levenberg-Marquardt on (x, y, [z,] theta); returns the number of iterations used.  s: in = start, out = solution.
SB_HD int sb_box_lm(const SbBoxProblem& pb, double* s, int max_iter = 200) {
    const double ks = 1.4142135623730951;         // see the header: the reference's gradient halves the keypoint term
    const int nv = pb.rect ? 3 : 4;
    const int var[4] = {0, 1, pb.rect ? 3 : 2, 3};   // state index of variable k
    double lam = 1e-3;
    double r[8], J[32];
    sb_box_residuals(pb, s, ks, r, J);
    double f = 0.0;
    for (int i = 0; i < 8; ++i) f += r[i] * r[i];
    int it = 0;
    for (; it < max_iter; ++it) {
        double A[16], g[4];
        for (int a = 0; a < nv; ++a) {
            g[a] = 0.0;
            for (int i = 0; i < 8; ++i) g[a] += J[4 * i + var[a]] * r[i];
            for (int b = 0; b < nv; ++b) {
                double v = 0.0;
                for (int i = 0; i < 8; ++i) v += J[4 * i + var[a]] * J[4 * i + var[b]];
                A[4 * a + b] = v;
            }
        }
        double gmax = 0.0;
        for (int a = 0; a < nv; ++a) gmax = fmax(gmax, fabs(g[a]));
        if (gmax < 1e-15) break;
        bool improved = false;
        for (int tries = 0; tries < 30 && !improved; ++tries) {
            // (A + lam * (diag(A) + eps)) d = -g by Gaussian elimination with partial pivoting
            double M[4][5];
            for (int a = 0; a < nv; ++a) {
                for (int b = 0; b < nv; ++b) M[a][b] = A[4 * a + b];
                M[a][a] += lam * (A[4 * a + a] + 1e-12);
                M[a][nv] = -g[a];
            }
            bool singular = false;
            for (int col = 0; col < nv; ++col) {
                int piv = col;
                for (int rr = col + 1; rr < nv; ++rr) if (fabs(M[rr][col]) > fabs(M[piv][col])) piv = rr;
                if (fabs(M[piv][col]) < 1e-300) { singular = true; break; }
                if (piv != col) for (int cc = 0; cc <= nv; ++cc) { const double t = M[col][cc]; M[col][cc] = M[piv][cc]; M[piv][cc] = t; }
                for (int rr = col + 1; rr < nv; ++rr) {
                    const double m = M[rr][col] / M[col][col];
                    for (int cc = col; cc <= nv; ++cc) M[rr][cc] -= m * M[col][cc];
                }
            }
            double d[4] = {0, 0, 0, 0};
            if (!singular) {
                for (int a = nv - 1; a >= 0; --a) {
                    double v = M[a][nv];
                    for (int b = a + 1; b < nv; ++b) v -= M[a][b] * d[b];
                    d[a] = v / M[a][a];
                }
            }
            double t[4] = {s[0], s[1], s[2], s[3]};
            for (int a = 0; a < nv; ++a) t[var[a]] += d[a];
            double r2[8], J2[32];
            sb_box_residuals(pb, t, ks, r2, J2);
            double f2 = 0.0;
            for (int i = 0; i < 8; ++i) f2 += r2[i] * r2[i];
            if (!singular && f2 <= f && isfinite(f2)) {
                double dmax = 0.0;
                for (int a = 0; a < nv; ++a) dmax = fmax(dmax, fabs(d[a]) / (1.0 + fabs(s[var[a]])));
                for (int a = 0; a < 4; ++a) s[a] = t[a];
                for (int i = 0; i < 8; ++i) r[i] = r2[i];
                for (int i = 0; i < 32; ++i) J[i] = J2[i];
                const double df = f - f2;
                f = f2;
                lam = fmax(lam / 3.0, 1e-15);
                improved = true;
                if (dmax < 1e-13 || df <= 1e-30 * (1.0 + f)) return it + 1;
            } else {
                lam *= 4.0;
            }
        }
        if (!improved) break;
    }
    return it;
}
