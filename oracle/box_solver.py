"""CPU oracle of the 3D box solvers between the network and dense_align -- TEST INFRASTRUCTURE ONLY.

Restates lib/model/utils/box_estimator.py (SURVEY 8f-1):

* ``BB2Viewpoint``                  box_estimator.py:15-42
* ``viewpoint2vertex``              box_estimator.py:44-125
* ``kpt2vertex`` / ``kpt2alpha``    box_estimator.py:127-167
* ``solve_x_y_z_theta_from_kpt``    box_estimator.py:169-385  (8 residuals, 4 states)
* ``solve_x_y_theta_from_kpt``      box_estimator.py:387-545  (6 residuals, 3 states, z from the aligned disparity)
* ``infer_boundary``                kitti_utils.py:398-437
* ``kitti_result_line``             kitti_utils.py:440-460 (write_detection_results' format string)

The reference minimises the sum of squared residuals with scipy's Newton-CG and an analytic gradient
(box_estimator.py:381,544; scipy is third-party and unpinned there -- scipy 1.18 in this image).  The oracle keeps
that: `objective`/`gradient` below are the reference's f_kpt/j_kpt (f_rect/j_rect) written once over a residual
vector, and `solve_*` call scipy.optimize.minimize(method="Newton-CG") on them.  tests/golden/make_golden.py (10)
pins objective, gradient and solutions against the reference's own functions executed from /root/reference.
"""
import math as m

import numpy as np

TRUNCATE_BORDER = 10          # box_estimator.py:195,406


def bb2viewpoint(alpha):
    alpha = alpha * 180.0 / m.pi
    if alpha > 360:
        alpha = alpha - 360
    elif alpha < -360:
        alpha = alpha + 360
    t = 4.0
    if -90.0 - t <= alpha <= -90.0 + t:
        return 0
    if -180.0 + t <= alpha <= -90.0 - t:
        return 1
    if alpha >= 180.0 - t or alpha <= -180.0 + t:
        return 2
    if 90.0 + t <= alpha <= 180.0 - t:
        return 3
    if 90.0 - t <= alpha <= 90.0 + t:
        return 4
    if 0.0 + t <= alpha <= 90.0 - t:
        return 5
    if 0.0 - t <= alpha <= 0.0 + t:
        return 6
    if -90.0 + t <= alpha <= 0.0 - t:
        return 7
    return -1


# (left, right, bottom) vertex signs (w, l) per viewpoint, box_estimator.py:93-123; viewpoint -1 falls in `else`
_VP = {0: ((-1, -1), (1, -1), (1, -1)), 1: ((-1, 1), (1, -1), (-1, -1)), 2: ((-1, 1), (-1, -1), (-1, -1)),
       3: ((1, 1), (-1, -1), (-1, 1)), 4: ((1, 1), (-1, 1), (-1, 1)), 5: ((1, -1), (-1, 1), (1, 1)),
       6: ((1, -1), (1, 1), (1, 1))}
_VP_ELSE = ((-1, -1), (1, 1), (1, -1))
_KPT = {0: (-1, -1), 1: (-1, 1), 2: (1, 1), 3: (1, -1)}       # box_estimator.py:139-146


def kpt2alpha(kpt_pos, kpt_type, box):
    clamp = lambda n: max(min(1, n), -1)
    r = m.asin(clamp((kpt_pos - box[0]) / (box[2] - box[0])))
    return {0: -m.pi / 2 - r, 1: m.pi - r, 2: m.pi / 2 - r, 3: -r}[kpt_type]


class Problem(object):
    """everything both solvers share: normalised measurements, active-residual masks, the three box vertices"""

    def __init__(self, im_shape, p2, p3, alpha, dim, box_left, box_right, kpts, z_fixed=None):
        p2, p3 = np.asarray(p2, np.float64), np.asarray(p3, np.float64)
        self.kpt_type = int(kpts[1])
        h_max, w_max = im_shape[0], im_shape[1]
        self.w, self.h, self.l = float(dim[0]), float(dim[1]), float(dim[2])
        ul, ur, vt, vb = [float(v) for v in (box_left[0], box_left[2], box_left[1], box_left[3])]
        f = p2[0, 0]
        cx, cy = p2[0, 2], p2[1, 2]
        self.f, self.bl = f, (p2[0, 3] - p3[0, 3]) / f
        self.left_u, self.right_u = (ul - cx) / f, (ur - cx) / f
        self.top_v, self.bottom_v = (vt - cy) / f, (vb - cy) / f
        self.kpt_u = (float(kpts[0]) - cx) / f
        tb = TRUNCATE_BORDER
        self.truncation = ul < 2.0 * tb or ur > w_max - 2.0 * tb
        self.alpha = float(alpha) if self.truncation else kpt2alpha(float(kpts[0]), self.kpt_type, box_left)
        vp = bb2viewpoint(self.alpha)
        lv, rv, bv = _VP.get(vp, _VP_ELSE)
        kv = _KPT[self.kpt_type]
        hw, hl = self.w / 2, self.l / 2
        self.vert = np.array([[lv[0] * hw, lv[1] * hl], [rv[0] * hw, rv[1] * hl], [bv[0] * hw, bv[1] * hl],
                              [kv[0] * hw, kv[1] * hl]])                      # rows: left, right, bottom, kpt (w, l)
        # which residuals are live (box_estimator.py:251-269 / 462-474)
        self.on = dict(ul=not ul < 2.0 * tb, ur=not ur > w_max - 2.0 * tb, uk=not self.truncation,
                       vb=not vb > h_max - tb, vt=not vt < tb, alpha=self.truncation)
        self.z_fixed = z_fixed
        if z_fixed is None:
            ul_r, ur_r = float(box_right[0]), float(box_right[2])
            self.left_u_r, self.right_u_r = (ul_r - cx) / f, (ur_r - cx) / f
            self.on.update(ulr=self.truncation and not ul_r < 2.0 * tb, urr=self.truncation and not ur_r > w_max - 2.0 * tb)
            self.disparity = (box_left[0] + box_left[2]) / 2 - (box_right[0] + box_right[2]) / 2

    # ---- residuals r_i and their derivatives wrt (x, y, z, theta) ----
    def residuals(self, s):
        """-> r [8], dr [8,4]; entries of switched-off residuals are zero"""
        if self.z_fixed is None:
            x, y, z, th = s
        else:
            (x, y, th), z = s, self.z_fixed
        c, sn = np.cos(th), np.sin(th)
        r, dr = np.zeros(8), np.zeros((8, 4))

        def u_res(i, vw, vl, meas, x_off, scale):
            den = z - sn * vw + c * vl
            num = x + x_off + c * vw + sn * vl
            r[i] = scale * (num / den - meas)
            dr[i] = scale * np.array([1.0 / den, 0.0, -num / den ** 2,
                                      (vl * c - vw * sn) / den + (vw * c + vl * sn) * num / den ** 2])
        (lw, ll), (rw, rl), (bw, bl_), (kw, kl) = self.vert
        if self.on["ul"]:
            u_res(0, lw, ll, self.left_u, 0.0, 1.0)
        if self.on["ur"]:
            u_res(1, rw, rl, self.right_u, 0.0, 1.0)
        if self.on["uk"]:
            u_res(2, kw, kl, self.kpt_u, 0.0, 2.0)                       # res_uk = 2 * res_uk (box_estimator.py:236)
        if self.on["vb"]:
            den = z - sn * bw + c * bl_
            r[3] = y / den - self.bottom_v
            dr[3] = [0.0, 1.0 / den, -y / den ** 2, y * (bw * c + bl_ * sn) / den ** 2]
        if self.on["vt"]:
            den = z + sn * bw - c * bl_
            r[4] = (y - self.h) / den - self.top_v
            dr[4] = [0.0, 1.0 / den, (self.h - y) / den ** 2, (self.h - y) * (bw * c + bl_ * sn) / den ** 2]
        if self.on["alpha"]:
            r[5] = th - m.pi / 2 + m.atan2(-x, z) - self.alpha
            q = 1.0 / (1.0 + (-x / z) ** 2)
            dr[5] = [q * (-1.0 / z), 0.0, q * (x / (z * z)), 1.0]
        if self.z_fixed is None:
            if self.on["ulr"]:
                u_res(6, lw, ll, self.left_u_r, -self.bl, 1.0)
            if self.on["urr"]:
                u_res(7, rw, rl, self.right_u_r, -self.bl, 1.0)
        return r, dr

    def objective(self, s):
        r, _ = self.residuals(s)
        return float(np.dot(r, r))

    def gradient(self, s):
        """the reference's j_kpt / j_rect: sum_i 2 r_i dr_i, with ITS scaling of the keypoint term: res_uk is doubled
        before being used in 2*res_uk/den, and the derivative of the doubling itself is not applied
        (box_estimator.py:236,292-297), so d(res_uk^2) is half of the true derivative there"""
        r, dr = self.residuals(s)
        dr = dr.copy()
        dr[2] *= 0.5
        g = 2.0 * (r[:, None] * dr).sum(0)
        return g if self.z_fixed is None else g[[0, 1, 3]]

    def init(self):
        if self.z_fixed is None:
            z = self.f * self.bl / self.disparity
        else:
            z = self.z_fixed
        x = z * (self.left_u + self.right_u) / 2.0
        y = z * (self.bottom_v + self.top_v) / 2.0 + self.h / 2.0
        th = self.alpha + m.pi / 2 - m.atan2(-x, z)
        return np.array([x, y, z, th]) if self.z_fixed is None else np.array([x, y, th])


def rejected(box_left, kpts):
    """the rejection rules of box_estimator.py:187 as test_net.py:287-295 evaluates them: the box is a float32 numpy
    row and the keypoints a float32 torch row, so each difference is rounded to float32 before it is compared"""
    b, k = np.asarray(box_left, np.float32), np.asarray(kpts, np.float32)
    return bool(k[4] - k[3] < 3 or b[2] - b[0] < 10 or b[3] - b[1] < 10)


def solve_x_y_z_theta_from_kpt(im_shape, p2, p3, alpha, dim, box_left, box_right, kpts):
    """box_estimator.py:169-385 -> (status, state[4] or 0)"""
    from scipy.optimize import minimize
    if rejected(box_left, kpts):
        return 0, 0
    pb = Problem(im_shape, p2, p3, alpha, dim, box_left, box_right, kpts)
    res = minimize(pb.objective, pb.init(), method="Newton-CG", jac=pb.gradient, options={"disp": False})
    return (0 if res.x[2] > 100 else 1), res.x


def solve_x_y_theta_from_kpt(im_shape, p2, p3, alpha, dim, box_left, disparity, kpts):
    """box_estimator.py:387-545 -> (state[3], z)"""
    from scipy.optimize import minimize
    p2a, p3a = np.asarray(p2, np.float64), np.asarray(p3, np.float64)
    f = p2a[0, 0]
    z = f * ((p2a[0, 3] - p3a[0, 3]) / f) / float(disparity)
    pb = Problem(im_shape, p2, p3, alpha, dim, box_left, None, kpts, z_fixed=z)
    res = minimize(pb.objective, pb.init(), method="Newton-CG", jac=pb.gradient, options={"disp": False})
    return res.x, z


def infer_boundary(im_shape, boxes_left):
    """kitti_utils.py:398-437: occlusion borders from a 1-D depth buffer painted in detection order"""
    n = boxes_left.shape[0]
    left_right = np.zeros((n, 2), dtype=np.float32)
    depth_line = np.zeros(im_shape[1] + 1, dtype=float)
    # (under the reference's numpy 1.x, `1050.0 / np.float32` is a float64: restated with float())
    for i in range(n):
        depth = 1050.0 / float(boxes_left[i, 3])
        for col in range(int(boxes_left[i, 0]), int(boxes_left[i, 2]) + 1):
            pixel = depth_line[col]
            if pixel == 0.0:
                depth_line[col] = depth
            elif depth < depth_line[col]:
                depth_line[col] = (depth + pixel) / 2.0
    for i in range(n):
        depth = 1050.0 / float(boxes_left[i, 3])
        left_right[i, 0], left_right[i, 1] = boxes_left[i, 0], boxes_left[i, 2]
        left_visible = not depth_line[int(boxes_left[i, 0])] < depth
        right_visible = not depth_line[int(boxes_left[i, 2])] < depth
        if not right_visible and not left_visible:
            left_right[i, 1] = boxes_left[i, 0]
        for col in range(int(boxes_left[i, 0]), int(boxes_left[i, 2]) + 1):
            if left_visible and depth_line[col] >= depth:
                left_right[i, 1] = col
            elif right_visible and depth_line[col] < depth:
                left_right[i, 0] = col
    return left_right


def kitti_result_line(t_cam2_cam0_x, box_left, pos, dim, orien, score):
    """kitti_utils.py:440-460, the text of one detection"""
    alpha = orien - m.pi / 2 + m.atan2(-pos[0], pos[2])
    s = "Car -1 -1 "
    s += "%f %f %f %f %f " % (alpha, box_left[0], box_left[1], box_left[2], box_left[3])
    s += "%f %f %f %f %f %f %f %f \n" % (dim[1], dim[0], dim[2], pos[0] - t_cam2_cam0_x, pos[1], pos[2], orien - 1.57, score)
    return s
