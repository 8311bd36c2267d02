// Host harness around stereo_rcnn_b200/csrc/box_solver_core.h (the numerics of the device box solver, plain C++):
// compiled with g++ by tests/test_box_solver.py so that the Levenberg-Marquardt solver is checked against the scipy
// oracle and the reference goldens without a GPU.
#include "../../stereo_rcnn_b200/csrc/box_solver_core.h"

extern "C" {

// in: im_h, im_w, p2[12], p3[12], alpha, dim[3], box_left[4], box_right[4], kpts[5], rect, disparity
// out: state[4], info[4] = {iterations, f_ref_objective(start), f_ref_objective(end), truncation}
int box_solve_host(int im_h, int im_w, const double* p2, const double* p3, double alpha, const double* dim,
                   const double* box_left, const double* box_right, const double* kpts, int rect, double disparity,
                   double* state, double* info) {
    SbBoxProblem pb;
    sb_box_problem(&pb, im_h, im_w, p2, p3, alpha, dim, box_left, box_right, kpts, rect, disparity);
    sb_box_init(pb, state);
    info[1] = sb_box_objective(pb, state, 2.0);
    const int it = sb_box_lm(pb, state);
    info[0] = it;
    info[2] = sb_box_objective(pb, state, 2.0);
    info[3] = pb.truncation;
    return 0;
}

// the status rules of box_estimator.py:187 on float32 inputs: 1 = rejected (box [4], kpts [5])
int box_rejected_host(const float* box, const float* kpts) { return sb_box_rejected(box, kpts); }

// objective (kpt_scale 2 = the reference's f) and the reference-style gradient (sum 2 r_i dr_i with the keypoint
// derivative halved) at a given state, for golden comparison
int box_eval_host(int im_h, int im_w, const double* p2, const double* p3, double alpha, const double* dim,
                  const double* box_left, const double* box_right, const double* kpts, int rect, double disparity,
                  const double* state, double* f_out, double* grad4) {
    SbBoxProblem pb;
    sb_box_problem(&pb, im_h, im_w, p2, p3, alpha, dim, box_left, box_right, kpts, rect, disparity);
    double s[4] = {state[0], state[1], rect ? pb.z_fixed : state[2], state[3]};
    double r[8], J[32];
    sb_box_residuals(pb, s, 2.0, r, J);
    double f = 0;
    for (int i = 0; i < 8; ++i) f += r[i] * r[i];
    *f_out = f;
    for (int a = 0; a < 4; ++a) {
        double g = 0;
        for (int i = 0; i < 8; ++i) g += 2.0 * r[i] * J[4 * i + a] * (i == 2 ? 0.5 : 1.0);
        grad4[a] = g;
    }
    return 0;
}
}
