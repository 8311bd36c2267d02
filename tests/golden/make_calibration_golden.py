"""Mint tests/golden/calibration.npz from the REFERENCE's own calibration reader (run in the build container only).

    python tests/golden/make_calibration_golden.py

kitti_utils.read_obj_calibration (kitti_utils.py:97-159) is imported from where it lies through oracle/ref_shim.py
(nothing copied) and run on three calibration files: the reference's demo/calib.txt and two synthetic KITTI-format
files with other focal lengths, principal points and baselines.  The texts are stored with P0-P3 and t_cam2_cam0[0]
as the reference returns them; tests/test_evaluate_args.py parses the stored texts and compares bit for bit.
"""
import os
import sys
import tempfile
import types

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "..", ".."))

from oracle import ref_shim  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def kitti_text(f, cx, cy, t0, t1, t2, t3):
    """a calib/*.txt in KITTI's layout; t_i = (P_i[0,3], P_i[1,3], P_i[2,3])"""
    def p(t):
        return [f, 0.0, cx, t[0], 0.0, f, cy, t[1], 0.0, 0.0, 1.0, t[2]]
    rows = [("P0", p(t0)), ("P1", p(t1)), ("P2", p(t2)), ("P3", p(t3)),
            ("R0_rect", [9.998817e-01, 1.511453e-02, -2.841595e-03, -1.511724e-02, 9.998853e-01, -9.338510e-04,
                         2.827154e-03, 9.766976e-04, 9.999955e-01]),
            ("Tr_velo_to_cam", [7.027555e-03, -9.999753e-01, 2.599616e-05, -7.137748e-03, -2.254837e-03,
                                -1.184917e-04, -9.999975e-01, -7.482656e-02, 9.999728e-01, 7.027479e-03,
                                -2.255075e-03, -3.336324e-01]),
            ("Tr_imu_to_velo", [9.999976e-01, 7.553071e-04, -2.035826e-03, -8.086759e-01, -7.854027e-04,
                                9.998898e-01, -1.482298e-02, 3.195559e-01, 2.024406e-03, 1.482454e-02,
                                9.998881e-01, -7.997231e-01])]
    return "".join("%s: %s\n" % (k, " ".join("%.12e" % v for v in vals)) for k, vals in rows) + "\n"


def main():
    ref_shim.load()
    try:
        import cv2  # noqa: F401
    except ImportError:                                   # kitti_utils imports cv2; the reader does not use it
        sys.modules["cv2"] = types.ModuleType("cv2")
    ku = ref_shim._exec_module("model.utils._kitti_utils_real", os.path.join(ref_shim.LIB, "model/utils/kitti_utils.py"))
    with open(os.path.join(ref_shim.REF, "demo", "calib.txt")) as fh:
        texts = [fh.read()]
    texts.append(kitti_text(7.070493e+02, 6.040814e+02, 1.805066e+02, (0.0, 0.0, 0.0), (-3.797842e+02, 0.0, 0.0),
                            (4.575831e+01, -3.454157e-01, 4.981016e-03), (-3.341081e+02, 2.330660e+00, 3.201153e-03)))
    texts.append(kitti_text(7.188560e+02, 6.071928e+02, 1.852157e+02, (1.234567e-01, 0.0, -0.0), (-3.861448e+02, 0.0, 0.0),
                            (4.538225e+01, -1.130887e-01, 3.779761e-03), (-3.372877e+02, 2.369057e+00, 4.915215e-03)))
    out = {k: [] for k in ("p0", "p1", "p2", "p3", "t_cam2_cam0_x")}
    with tempfile.TemporaryDirectory() as d:
        for i, text in enumerate(texts):
            path = os.path.join(d, "%06d.txt" % i)
            with open(path, "w") as fh:
                fh.write(text)
            c = ku.read_obj_calibration(path)
            for k in ("p0", "p1", "p2", "p3"):
                out[k].append(np.asarray(getattr(c, k), np.float64))
            out["t_cam2_cam0_x"].append(np.float64(c.t_cam2_cam0[0]))
    np.savez_compressed(os.path.join(HERE, "calibration.npz"), texts=np.array(texts),
                        **{k: np.array(v, np.float64) for k, v in out.items()})
    print("wrote calibration.npz:", len(texts), "calibrations")


if __name__ == "__main__":
    main()
