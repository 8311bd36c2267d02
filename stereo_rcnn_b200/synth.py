"""Seeded synthetic inputs (no dataset / checkpoint is reachable offline).

Shared by bench.py, the tests and tests/golden/make_golden.py so that every leg
sees byte-identical inputs.  Shapes follow BASELINE.md section 2 / SURVEY 8(d):
network-scale pair 1x3x600x1987 (a 1242x375 KITTI frame resized by 1.6), and the
config-5 pose sampler for dense_align RoIs.
"""
import zlib
from collections import OrderedDict

import numpy as np

# demo/calib.txt of the reference (KITTI 000xxx): P2 and P3, 3x4
DEMO_P2 = np.array([[721.5377, 0.0, 609.5593, 44.85728],
                    [0.0, 721.5377, 172.854, 0.2163791],
                    [0.0, 0.0, 1.0, 0.002745884]], np.float64)
DEMO_P3 = np.array([[721.5377, 0.0, 609.5593, -339.5242],
                    [0.0, 721.5377, 172.854, 2.199936],
                    [0.0, 0.0, 1.0, 0.002729905]], np.float64)


def _bicubic_up(base, H, W):
    import torch
    t = torch.from_numpy(base)[None]
    return torch.nn.functional.interpolate(t, size=(H, W), mode="bicubic", align_corners=True)[0].numpy()


def synth_pair(H, W, seed, shift=12):
    """smooth seeded network-scale pair (3,H,W) fp32; right = left shifted `shift` px"""
    rs = np.random.RandomState(seed)
    base = rs.randn(3, H // 4 + 2, W // 4 + 2).astype(np.float32)
    left = (_bicubic_up(base, H, W) * 40.0).astype(np.float32)
    right = np.empty_like(left)
    right[:, :, :-shift] = left[:, :, shift:]
    right[:, :, -shift:] = left[:, :, -1:]
    return left, right


def gen_rois(D, seed, p2=DEMO_P2, width=1242, height=375):
    """seeded 3D boxes projected with P2 -> box_left [D,4], keypoints [D,5], poses [D,7]"""
    r = np.random.RandomState(seed)
    out = []
    while len(out) < D:
        z = r.uniform(6, 60); x = r.uniform(-0.45 * z, 0.45 * z); y = 1.65
        w, h, l = r.normal([1.6, 1.5, 3.9], 0.1); th = r.uniform(-np.pi, np.pi)
        c, s = np.cos(th), np.sin(th)
        xs = np.array([-w / 2, -w / 2, w / 2, w / 2] * 2); ys = np.array([0, 0, 0, 0, -h, -h, -h, -h])
        zs = np.array([-l / 2, l / 2, l / 2, -l / 2] * 2)
        X = c * xs + s * zs + x; Y = ys + y; Z = -s * xs + c * zs + z
        if Z.min() < 1:
            continue
        u = p2[0, 0] * X / Z + p2[0, 2]; v = p2[1, 1] * Y / Z + p2[1, 2]
        x1, x2 = np.clip([u.min(), u.max()], 0, width - 1)
        y1, y2 = np.clip([v.min(), v.max()], 0, height - 1)
        if x2 - x1 < 10 or y2 - y1 < 10:
            continue
        out.append(([x1, y1, x2, y2], [(x1 + x2) / 2, 1, 0.9, x1, x2], [x, y, z, w, h, l, th]))
    f = np.float32
    return (np.array([o[0] for o in out], f), np.array([o[1] for o in out], f),
            np.array([o[2] for o in out], f))


LAYERS = [3, 4, 23, 3]
PLANES = [64, 128, 256, 512]


# --------------------------------------------------------------------------
# state dict layout
# --------------------------------------------------------------------------
def param_shapes(n_classes=2):
    """ordered {key: shape} of every tensor the forward reads (reference key names)"""
    s = OrderedDict()

    def conv(k, co, ci, kh, kw, bias):
        s[k + ".weight"] = (co, ci, kh, kw)
        if bias:
            s[k + ".bias"] = (co,)

    def bn(k, c):
        for n in ("weight", "bias", "running_mean", "running_var"):
            s[k + "." + n] = (c,)

    conv("RCNN_layer0.0", 64, 3, 7, 7, False)
    bn("RCNN_layer0.1", 64)
    inpl = 64
    for li, (nb, pl) in enumerate(zip(LAYERS, PLANES)):
        for b in range(nb):
            p = "RCNN_layer%d.0.%d" % (li + 1, b)
            conv(p + ".conv1", pl, inpl, 1, 1, False); bn(p + ".bn1", pl)
            conv(p + ".conv2", pl, pl, 3, 3, False); bn(p + ".bn2", pl)
            conv(p + ".conv3", pl * 4, pl, 1, 1, False); bn(p + ".bn3", pl * 4)
            if b == 0:
                conv(p + ".downsample.0", pl * 4, inpl, 1, 1, False); bn(p + ".downsample.1", pl * 4)
            inpl = pl * 4
    conv("RCNN_toplayer", 256, 2048, 1, 1, True)
    for i in (1, 2, 3):
        conv("RCNN_smooth%d" % i, 256, 256, 3, 3, True)
    conv("RCNN_latlayer1", 256, 1024, 1, 1, True)
    conv("RCNN_latlayer2", 256, 512, 1, 1, True)
    conv("RCNN_latlayer3", 256, 256, 1, 1, True)
    conv("RCNN_rpn.RPN_Conv", 512, 256, 3, 3, True)
    conv("RCNN_rpn.RPN_cls_score", 6, 1024, 1, 1, True)
    conv("RCNN_rpn.RPN_bbox_pred_left_right", 18, 1024, 1, 1, True)
    conv("RCNN_top.0", 2048, 512, 7, 7, True)
    conv("RCNN_top.3", 2048, 2048, 1, 1, True)
    for i in range(0, 12, 2):
        conv("RCNN_kpts.%d" % i, 256, 256, 3, 3, True)
    s["RCNN_kpts.12.weight"] = (256, 256, 2, 2)      # ConvTranspose2d: (Cin, Cout, kh, kw)
    s["RCNN_kpts.12.bias"] = (256,)
    s["RCNN_cls_score.weight"] = (n_classes, 2048); s["RCNN_cls_score.bias"] = (n_classes,)
    s["RCNN_bbox_pred.weight"] = (6 * n_classes, 2048); s["RCNN_bbox_pred.bias"] = (6 * n_classes,)
    s["RCNN_dim_orien_pred.weight"] = (5 * n_classes, 2048); s["RCNN_dim_orien_pred.bias"] = (5 * n_classes,)
    conv("kpts_class", 6, 256, 1, 1, True)
    return s


def make_state_dict(seed=3, n_classes=2, head_gain=1.0):
    """Deterministic synthetic weights, one private RNG stream per key.

    "Variance-preserving" variant of the reference's random init (SURVEY 7,
    hard part "random-init weights saturate the RPN"): He-normal conv weights,
    non-trivial frozen-BN statistics, and a small ``bn3.weight`` so the residual
    trunk neither explodes nor collapses; head weights scaled so that RPN scores
    and box deltas are spread out (non-degenerate NMS / top-k work).
    """
    import torch
    sd = OrderedDict()
    for k, shp in param_shapes(n_classes).items():
        g = torch.Generator().manual_seed((seed * 1000003 + zlib.crc32(k.encode())) % (2 ** 31))
        leaf = k.rsplit(".", 1)[1]
        is_bn = ".bn" in k or "downsample.1" in k or k.startswith("RCNN_layer0.1")
        if is_bn:
            n = shp[0]
            if leaf == "weight":
                lo, hi = (0.15, 0.35) if ".bn3." in k else (0.8, 1.2)
                t = torch.rand(n, generator=g) * (hi - lo) + lo
            elif leaf == "bias":
                t = torch.randn(n, generator=g) * 0.05
            elif leaf == "running_mean":
                t = torch.randn(n, generator=g) * 0.1
            else:
                t = torch.rand(n, generator=g) * 0.4 + 0.8
        elif leaf == "bias":
            t = torch.randn(shp, generator=g) * 0.02
        else:
            fan_in = int(np.prod(shp[1:]))
            if k.startswith("RCNN_kpts.12"):
                fan_in = shp[0]
            std = (2.0 / fan_in) ** 0.5
            if k.startswith(("RCNN_cls_score", "RCNN_bbox_pred", "RCNN_dim_orien_pred",
                             "RCNN_rpn.RPN_cls_score", "RCNN_rpn.RPN_bbox_pred", "kpts_class")):
                std = head_gain * (1.0 / fan_in) ** 0.5
            if k.startswith("RCNN_rpn.RPN_bbox_pred"):
                std *= 0.25
            # fixed gains (calibrated once on a 200x333 input so that every stage's
            # activations have rms ~1; see DESIGN.md "synthetic weights")
            for pre, gain in _GAINS:
                if k.startswith(pre):
                    std *= gain
            t = torch.randn(shp, generator=g) * std
        sd[k] = t.float().contiguous()
    return sd


_GAINS = (("RCNN_layer0.0", 1.0 / 64), ("RCNN_toplayer", 0.0625), ("RCNN_latlayer1", 0.075),
          ("RCNN_latlayer2", 0.22), ("RCNN_latlayer3", 0.32), ("RCNN_smooth", 0.5),
          ("RCNN_rpn.RPN_cls_score", 2.0), ("kpts_class", 0.1))




def make_reference_init_state_dict(seed=3, n_classes=2):
    """The reference's OWN random initialisation, restated with seeded per-key RNG streams: ResNet convs
    N(0, sqrt(2 / (kh*kw*Cout))) and BatchNorm weight 1 / bias 0 / mean 0 / var 1 (lib/model/stereo_rcnn/resnet.py:123-129);
    FPN / RPN / predictor layers N(0, 0.01) (bbox_pred, dim_orien_pred 0.001; kpts_class 0.1) with zero bias, RCNN_top and
    RCNN_kpts N(0, 0.02) with zero bias (stereo_rcnn.py:47-85).  Un-normalised: activations grow to ~1e6 by C4, far
    outside fp16 -- the tf32 precision mode is the one that runs such weights (BASELINE.md 2, SURVEY 8d)."""
    import torch
    sd = OrderedDict()
    for k, shp in param_shapes(n_classes).items():
        g = torch.Generator().manual_seed((seed * 1000003 + zlib.crc32(k.encode()) + 77) % (2 ** 31))
        leaf = k.rsplit(".", 1)[1]
        is_bn = ".bn" in k or "downsample.1" in k or k.startswith("RCNN_layer0.1")
        if is_bn:
            t = torch.ones(shp) if leaf in ("weight", "running_var") else torch.zeros(shp)
        elif leaf == "bias":
            t = torch.zeros(shp)
        elif k.startswith("RCNN_layer"):
            t = torch.randn(shp, generator=g) * (2.0 / (shp[2] * shp[3] * shp[0])) ** 0.5
        else:
            std = 0.01
            if k.startswith(("RCNN_bbox_pred", "RCNN_dim_orien_pred")):
                std = 0.001
            elif k.startswith("kpts_class"):
                std = 0.1
            elif k.startswith(("RCNN_top", "RCNN_kpts")):
                std = 0.02
            t = torch.randn(shp, generator=g) * std
        sd[k] = t.float().contiguous()
    return sd


def synth_train_gt(B, K, H, W, seed, n_boxes=None, disparity=6.0):
    """ground truth of a training batch in the layout of roibatchLoader.py:199-240: gt_left / gt_right / gt_merge
    [B,K,5] (x1, y1, x2, y2, class; zero rows pad to K = MAX_NUM_GT_BOXES), gt_dim_orien [B,K,5], gt_kpts [B,K,6]
    (four perspective keypoints, one visible, -1 otherwise; left / right border), all fp32"""
    rng = np.random.RandomState(seed)
    n_boxes = n_boxes or [min(K, 3 + 2 * b) for b in range(B)]
    gl = np.zeros((B, K, 5), np.float32)
    for b in range(B):
        for j in range(n_boxes[b]):
            w = rng.uniform(0.08 * W, 0.35 * W)
            h = rng.uniform(0.1 * H, 0.4 * H)
            x1 = rng.uniform(disparity + 2, W - w - 1)
            y1 = rng.uniform(0, H - h - 1)
            gl[b, j] = [x1, y1, x1 + w, y1 + h, 1]
    gr = gl.copy()
    gr[:, :, 0] -= disparity
    gr[:, :, 2] -= disparity
    gr[gl[:, :, 4] == 0] = 0
    gm = gl.copy()
    gm[:, :, 0] = np.minimum(gl[:, :, 0], gr[:, :, 0])
    gm[:, :, 2] = np.maximum(gl[:, :, 2], gr[:, :, 2])
    dim = rng.uniform(-1, 4, (B, K, 5)).astype(np.float32)
    kp = np.zeros((B, K, 6), np.float32)
    for b in range(B):
        for j in range(K):
            x1, x2 = gl[b, j, 0], gl[b, j, 2]
            kp[b, j, :4] = -1
            kp[b, j, rng.randint(4)] = rng.uniform(x1, x2)
            kp[b, j, 4] = rng.uniform(x1, x1 + 0.3 * (x2 - x1))
            kp[b, j, 5] = rng.uniform(x2 - 0.3 * (x2 - x1), x2)
    return gl, gr.astype(np.float32), gm.astype(np.float32), dim, kp, np.asarray(n_boxes, np.int64)


def synth_train_rois(gt_left, R, H, W, seed, near_gt=0.34, jitter=6.0, disparity=6.0):
    """proposals of a training step: a fraction `near_gt` jittered copies of ground-truth boxes (foreground
    candidates), the rest uniform boxes -> rois_left, rois_right [B,R,5] (batch index first)"""
    rng = np.random.RandomState(seed)
    B = gt_left.shape[0]
    out = np.zeros((B, R, 5), np.float32)
    for b in range(B):
        n = int((gt_left[b, :, 4] > 0).sum())
        for r in range(R):
            if n > 0 and rng.uniform() < near_gt:
                out[b, r, 1:] = gt_left[b, rng.randint(n), :4] + rng.uniform(-jitter, jitter, 4)
            else:
                w = rng.uniform(0.04 * W, 0.4 * W)
                h = rng.uniform(0.06 * H, 0.5 * H)
                x1 = rng.uniform(disparity, W - w - 1)
                y1 = rng.uniform(0, H - h - 1)
                out[b, r, 1:] = [x1, y1, x1 + w, y1 + h]
        out[b, :, 0] = b
    right = out.copy()
    right[:, :, 1] -= disparity
    right[:, :, 3] -= disparity
    return out, right


def kitti_split(n_images, seed=0, n_cars=4, n_dets=30):
    """A seeded synthetic KITTI split as text: per image about n_cars Cars, a Van, a Pedestrian and two DontCare
    label lines, and about n_dets result lines -- jittered copies of the labelled objects (orientations across +-pi
    included) and detections away from them -> [(label_text, result_text)]"""
    rs = np.random.RandomState(seed)

    def obj(kind):
        z = rs.uniform(5.0, 60.0)
        x = rs.uniform(-15.0, 15.0)
        h, w, l = {"Car": (1.5, 1.6, 3.9), "Van": (2.2, 1.9, 5.0), "Pedestrian": (1.7, 0.6, 0.8)}[kind]
        h, w, l = h * rs.uniform(0.9, 1.1), w * rs.uniform(0.9, 1.1), l * rs.uniform(0.9, 1.1)
        u = 621.0 + 720.0 * x / z
        bh = 720.0 * h / z
        bw = 720.0 * max(w, l) / z
        y = 1.65 + rs.uniform(-0.2, 0.2)
        v2 = 175.0 + 720.0 * y / z
        return [float(rs.choice([0.0, 0.1, 0.15, 0.3, 0.6])), int(rs.choice([0, 1, 2, 3])), rs.uniform(-np.pi, np.pi),
                u - bw / 2, v2 - bh, u + bw / 2, v2, h, w, l, x, y, z, rs.uniform(-np.pi, np.pi)]

    def line(kind, r, score=None):
        s = "%s %.2f %d %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f %.2f" % tuple([kind] + list(r))
        return s + (" %.4f\n" % score if score is not None else "\n")

    split = []
    for _ in range(n_images):
        kinds = ["Car"] * max(0, n_cars + rs.randint(-1, 2)) + ["Van", "Pedestrian"]
        gts = [(k, obj(k)) for k in kinds]
        labels = [line(k, r) for k, r in gts]
        for _d in range(2):
            x1, y1 = rs.uniform(0, 1100), rs.uniform(100, 300)
            labels.append("DontCare -1 -1 -10 %.2f %.2f %.2f %.2f -1 -1 -1 -1000 -1000 -1000 -10\n"
                          % (x1, y1, x1 + rs.uniform(10, 120), y1 + rs.uniform(10, 60)))
        dets = []
        while len(dets) < n_dets + rs.randint(-3, 4):
            if rs.rand() < 0.6:
                k, r = gts[rs.randint(len(gts))]
                r = list(r)
                j = rs.uniform(0.0, 0.15)
                bw, bh = r[5] - r[3], r[6] - r[4]
                r[3:7] = [r[3] + rs.randn() * j * bw, r[4] + rs.randn() * j * bh, r[5] + rs.randn() * j * bw,
                          r[6] + rs.randn() * j * bh]
                r[10] += rs.randn() * j * r[9]
                r[12] += rs.randn() * j * r[9]
                r[13] = (r[13] + rs.randn() * 0.3 + np.pi) % (2 * np.pi) - np.pi
                r[2] = (r[2] + rs.randn() * 0.3 + np.pi) % (2 * np.pi) - np.pi
                k = "Car" if rs.rand() < 0.9 else k
            else:
                k, r = "Car", obj("Car")
            dets.append(line(k, r, rs.uniform(0.05, 1.0)))
        split.append(("".join(labels), "".join(dets)))
    return split


def png_bytes(rgb):
    """a uint8 [H,W,3] array as an 8-bit RGB PNG file (zlib, no filter)"""
    import struct
    a = np.ascontiguousarray(rgb, np.uint8)
    h, w = a.shape[:2]

    def chunk(tag, data):
        return struct.pack(">I", len(data)) + tag + data + struct.pack(">I", zlib.crc32(tag + data) & 0xFFFFFFFF)
    raw = b"".join(b"\x00" + a[r].tobytes() for r in range(h))
    return (b"\x89PNG\r\n\x1a\n" + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0)) +
            chunk(b"IDAT", zlib.compress(raw, 1)) + chunk(b"IEND", b""))


def kitti_folder(root, n_images, seed=0, sizes=((375, 1242), (370, 1224)), frames=None):
    """A seeded synthetic KITTI training folder: root/training/label_2 (kitti_split's label texts), calib (KITTI-like
    P0-P3 around the demo calibration) and image_2 / image_3.  The images are PNG headers only (enough for
    kitti_data, which reads the size) unless frames(k) -> (left, right) uint8 [H,W,3] gives the pixels; image k has
    size sizes[k % len(sizes)].  -> the image ids"""
    import os
    rs = np.random.RandomState(seed + 1)
    d = os.path.join(root, "training")
    for sub in ("label_2", "calib", "image_2", "image_3"):
        os.makedirs(os.path.join(d, sub), exist_ok=True)
    ids = []
    for k, (labels, _dets) in enumerate(kitti_split(n_images, seed)):
        i = "%06d" % k
        ids.append(i)
        f = DEMO_P2[0, 0] + rs.uniform(-15, 15)
        cx, cy = DEMO_P2[0, 2] + rs.uniform(-8, 8), DEMO_P2[1, 2] + rs.uniform(-8, 8)
        rows = []
        for name, t in (("P0", (0.0, 0.0, 0.0)), ("P1", (-f * 0.54, 0.0, 0.0)),
                        ("P2", (DEMO_P2[0, 3] + rs.uniform(-1, 1), DEMO_P2[1, 3], DEMO_P2[2, 3])),
                        ("P3", (DEMO_P3[0, 3] + rs.uniform(-3, 3), DEMO_P3[1, 3], DEMO_P3[2, 3]))):
            rows.append("%s: %s" % (name, " ".join("%.12e" % v for v in (f, 0.0, cx, t[0], 0.0, f, cy, t[1], 0.0, 0.0,
                                                                        1.0, t[2]))))
        rows += ["R0_rect: " + " ".join(["1.0", "0.0", "0.0", "0.0", "1.0", "0.0", "0.0", "0.0", "1.0"]),
                 "Tr_velo_to_cam: " + " ".join(["0.0"] * 12), "Tr_imu_to_velo: " + " ".join(["0.0"] * 12)]
        h, w = sizes[k % len(sizes)]
        # objects in view only, as in KITTI's labels (one whose box starts past the depth line is refused)
        labels = "".join(l + "\n" for l in labels.splitlines() if l.startswith("DontCare") or
                         (float(l.split()[4]) > 0.0 and float(l.split()[6]) < w - 1))
        with open(os.path.join(d, "label_2", i + ".txt"), "w") as fh:
            fh.write(labels)
        with open(os.path.join(d, "calib", i + ".txt"), "w") as fh:
            fh.write("\n".join(rows) + "\n\n")
        if frames is not None:
            pair = frames(k)
            assert pair[0].shape[:2] == (h, w)
        for j, sub in enumerate(("image_2", "image_3")):
            with open(os.path.join(d, sub, i + ".png"), "wb") as fh:
                if frames is not None:
                    fh.write(png_bytes(pair[j]))
                else:
                    fh.write(png_bytes(np.zeros((1, 1, 3), np.uint8))[:16] + w.to_bytes(4, "big") +
                             h.to_bytes(4, "big") + b"\x08\x02\x00\x00\x00")
    return ids
