"""Sequential restatement of sb_kitti_annotations (DESIGN.md §10), the checker of csrc/kitti_annotations.cu: the
reference's kitti_utils.read_obj_data, kitti.remove_occluded_keypoints (left camera, then right camera on the
survivors) and kitti._load_kitti_annotation's filter over the packed split of stereo_rcnn_b200.kitti_data.

Every fp64 operation is one Python float operation in the kernel's order: R.v as (r0 vx + r1 vy) + r2 vz with the
literal zero terms, the projection as ((p0 x + p1 y) + p2 z) + p3 and then the two divisions, `int()` toward zero, and
min / max as Python's builtins (the second argument only when strictly smaller / larger).  The reference's numpy
BLAS products may round differently in the last bit; with orientation exactly 0 and dyadic inputs every order gives
the same bits.
"""
import numpy as np

COLS = 1260                                   # the reference's depth line
IN, OUT, CALIB = 11, 30, 25
TRUNC, OCC, ALPHA, W_, H_, L_, X, Y, Z, COS, SIN = range(11)


def _div(a, b):
    """a / b in IEEE fp64: +-inf or NaN for b == 0, as numpy and __ddiv_rn give (Python's float division raises)"""
    if b != 0.0:
        return a / b
    with np.errstate(divide="ignore", invalid="ignore"):
        return float(np.float64(a) / np.float64(b))


class _Obj(object):
    __slots__ = ("row", "car", "box", "kp", "vis", "z", "merge")


def project(r, cal, H, W, car=True):
    """read_obj_data for one packed row -> _Obj (boxes, keypoints and merged box of both cameras, pos z)"""
    r = [float(v) for v in r]
    cal = [float(v) for v in cal]
    px, py, pz = r[X] + cal[24], r[Y] + 0.0, r[Z] + 0.0
    c, s, w, h, l = r[COS], r[SIN], r[W_], r[H_], r[L_]
    corners = []
    for k in range(8):
        vx = -w if (k & 3) < 2 else w
        vz = -l if (k & 3) in (0, 3) else l
        vy = 0.0 if k < 4 else -2.0 * h
        rx = (c * vx + 0.0 * vy) + s * vz
        ry = (0.0 * vx + 1.0 * vy) + 0.0 * vz
        rz = (-s * vx + 0.0 * vy) + c * vz
        corners.append((px + rx / 2.0, py + ry / 2.0, pz + rz / 2.0))
    o = _Obj()
    o.car, o.z, o.box, o.kp, o.vis = car, pz, [], [], [[0.0, 0.0], [0.0, 0.0]]
    for j in range(2):
        P = cal[12 * j:12 * j + 12]
        box = [10000.0, 10000.0, 0.0, 0.0]
        kp = [-1.0] * 4
        for k, (x, y, z) in enumerate(corners):
            if z < 0:
                continue
            n = [((P[4 * q] * x + P[4 * q + 1] * y) + P[4 * q + 2] * z) + P[4 * q + 3] for q in range(3)]
            u, v = _div(n[0], n[2]), _div(n[1], n[2])
            if k < 4:
                kp[k] = u
            box = [min(box[0], u), min(box[1], v), max(box[2], u), max(box[3], v)]
        box = [max(box[0], 0.0), max(box[1], 0.0), min(box[2], float(W - 1)), min(box[3], float(H - 1))]
        lk, rk, li, ri = 5000.0, 0.0, -1, -1
        for k in range(4):
            if kp[k] < lk:
                lk, li = kp[k], k
            if kp[k] > rk:
                rk, ri = kp[k], k
        for k in range(4):
            if k not in (li, ri) and corners[k][2] > pz:
                kp[k] = -1.0
        o.box.append(box)
        o.kp.append(kp)
    b0, b1 = o.box
    o.merge = [min(b1[0], b0[0]), min(b1[1], b0[1]), max(b1[2], b0[2]), max(b1[3], b0[3])]
    return o


def _fail(objs, ix):
    """the list position of the object the reference indexes the depth line out of range with, or None"""
    for p, o in enumerate(objs):                            # painting, object by object
        c1, c2 = int(o.box[ix][0]), int(o.box[ix][2])
        if c1 <= c2 and c2 >= COLS:
            return p
    for p, o in enumerate(objs):                            # then the two end lookups
        if int(o.box[ix][0]) >= COLS or int(o.box[ix][2]) >= COLS:
            return p
    return None


def occlusion_pass(objs, ix):
    """remove_occluded_keypoints(objs, left=(ix == 0)) -> survivors (the objects are updated in place)"""
    depth = [0.0] * COLS
    for o in objs:
        for col in range(int(o.box[ix][0]), int(o.box[ix][2]) + 1):
            pixel = depth[col]
            if pixel == 0.0:
                depth[col] = o.z
            elif o.z < depth[col]:
                depth[col] = (o.z + pixel) / 2.0
    for o in objs:
        x1, x2 = o.box[ix][0], o.box[ix][2]
        vl, vr = x1, x2
        lv = not depth[int(x1)] < o.z
        rv = not depth[int(x2)] < o.z
        if not lv and not rv:
            vr = x1
            o.kp[ix] = [-1.0] * 4
        for col in range(int(x1), int(x2) + 1):
            if lv and depth[col] >= o.z:
                vr = float(col)
            elif rv and depth[col] < o.z:
                vl = float(col)
        o.vis[ix] = [vl, vr]
    objs = [o for o in objs if ((o.kp[ix][0] + o.kp[ix][1]) + o.kp[ix][2]) + o.kp[ix][3] > -4.0]
    for o in objs:
        kp = o.kp[ix]
        lk, rk = 5000.0, 0.0
        for v in kp:
            if v != -1.0:
                if v < lk:
                    lk = v
                if v > rk:
                    rk = v
        vl, vr = o.vis[ix]
        for q in range(4):
            v = kp[q]
            if v != -1.0 and (v < vl - 5.0 or v > vr + 5.0 or v < lk + 3.0 or v > rk - 3.0):
                kp[q] = -1.0
    return objs


def image(rows, codes, cal, H, W):
    """one image -> (kept rows float32 [k,30] in sb_kitti_annotations' layout, status)"""
    rows = np.asarray(rows, np.float64).reshape(-1, IN)
    if H <= 0 or W <= 0:
        return np.zeros((0, OUT), np.float32), -1
    objs = []
    for i, (r, code) in enumerate(zip(rows, np.asarray(codes).tolist())):
        o = project(r, cal, H, W, code == 0)
        o.row = i
        objs.append(o)
    for ix in range(2):
        p = _fail(objs, ix)
        if p is not None:
            return np.zeros((0, OUT), np.float32), 1 + objs[p].row
        objs = occlusion_pass(objs, ix)
    out = []
    for o in objs:
        r = [float(v) for v in rows[o.row]]
        if r[TRUNC] < 0.98 and r[OCC] < 3.0 and o.box[0][3] - o.box[0][1] > 10.0 and o.car and \
                o.vis[0][1] - o.vis[0][0] > 3.0 and o.vis[1][1] - o.vis[1][0] > 3.0:
            out.append(o.box[0] + o.box[1] + o.merge + [r[W_], r[H_], r[L_], r[ALPHA]] + o.kp[0] + o.vis[0] +
                       o.kp[1] + o.vis[1] + [r[TRUNC], r[OCC]])
    return np.array(out, np.float64).reshape(-1, OUT).astype(np.float32), 0


def split(rows, codes, obj_off, calib, image_hw):
    """the packed split (kitti_data.Split.arrays()) -> (out float32 [n,30], n_kept int32, status int32), laid out as
    sb_kitti_annotations writes them"""
    rows = np.asarray(rows, np.float64).reshape(-1, IN)
    off = np.asarray(obj_off, np.int64)
    ni = len(off) - 1
    out = np.zeros((len(rows), OUT), np.float32)
    n_kept, status = np.zeros(ni, np.int32), np.zeros(ni, np.int32)
    for i in range(ni):
        a, b = int(off[i]), int(off[i + 1])
        kept, s = image(rows[a:b], np.asarray(codes)[a:b], np.asarray(calib)[i], int(image_hw[i][0]),
                        int(image_hw[i][1]))
        out[a:a + len(kept)] = kept
        n_kept[i], status[i] = len(kept), s
    return out, n_kept, status
