"""CPU: the case builders of the KITTI evaluation's edge tests, each checked to reach the boundary it names, with the
oracle (oracle/kitti_eval.py) and numpy only.  test_gpu_kitti_eval_edges.py runs every builder through sb_kitti_eval.

* the threshold scan's 1024-image chunks: splits of 1023 to 3769 images whose TP scores interleave across chunks,
  with TPs on both sides of every chunk edge, or none at the edges, or empty first and last images;
* the rank kernel's 256-score blocks: more than 512 TPs with two-decimal scores, one score for all, detections at a
  threshold's exact value, scores at and below the no-match value -1e7;
* the threshold lanes of pass 2: splits reaching 0, 1, 31, 32, 33, 40 and 41 thresholds, and images of more than 32
  detections whose top-scored detections sit in assigned-bit words 1 and 2;
* the 8 KB staging of an image: (63 gt, 16 det) at exactly 8192 B, (64, 16) at 8320 B, 31 / 32 / 33 / 64 / 65
  detections on both sides of the limit, runs of global-path images first, in the middle and last;
* the pair search: empty images at the start, at the end and at the 1024 edge, and a split with no pairs but gt rows;
* overlap geometry against scipy's polygon areas: zero extents, rotations by multiples of pi/2, thin and far
  rectangles, collinear and touching edges.

Images are light (one to three Cars, a few detections), laid out in slots: slot k of an image is apart from every other
slot in 2D, BEV and 3D, so a detection overlaps the ground truth of its own slot only.
"""
import math

import numpy as np
import pytest

from oracle import kitti_eval as O
from test_kitti_eval import DONTCARE_ROW, _d, bev_row, image, row, scipy_area

CHUNK, RANK_BLOCK, STAGE_BYTES, LANES = 1024, 256, 8192, 32
CHUNK_SIZES = (1023, 1024, 1025, 2048, 2049, 3769)
THRESHOLD_COUNTS = (0, 1, 31, 32, 33, 40, 41)
RANK_KINDS = ("two_decimals", "one_score", "at_threshold", "no_match")
FOUR_BARS = (0.0, 0.3, 0.7, 1.0)
ABOVE_NO_MATCH = float(np.nextafter(O.NO_MATCH, 0.0))


# ------------------------------------------------------------------------------------------------ slots ----
def car(k, occ=0, trunc=0.0, alpha=0.0):
    """a Car label (easy unless occ / trunc say otherwise) in slot k"""
    return row((110.0 * k, 100.0, 110.0 * k + 100.0, 160.0), x=-100.0 + 5.0 * k, z=30.0, occ=occ, trunc=trunc,
               alpha=alpha)


def dontcare(k):
    """a DontCare label over slot k's 2D box (negative dimensions, as in KITTI's label files)"""
    return _d(DONTCARE_ROW, x1=110.0 * k, y1=90.0, x2=110.0 * k + 120.0, y2=170.0)


def det(kind, k, score, alpha=0.0):
    """a detection of slot k: "hit" copies the label (IoU 1 everywhere); "near2d" is shifted in the image only (2D IoU
    0.6), "wide2d" further (2D IoU 0.4); "nearbev" is moved along x only (BEV and 3D IoU 0.6); "lifted" and "high" are
    moved up only (3D IoU 0.43 and 0.2); "far" and "distant" are shifted in the image and in x (IoU 0.4 and 0.2 in
    every metric)"""
    r = list(car(k))
    shift = {"near2d": (25.0, 0.0), "nearbev": (0.0, 0.975), "far": (300.0 / 7.0, 3.9 * 3.0 / 7.0),
             "distant": (200.0 / 3.0, 2.6), "wide2d": (300.0 / 7.0, 0.0)}.get(kind, (0.0, 0.0))
    r[O.X1], r[O.X2], r[O.X] = r[O.X1] + shift[0], r[O.X2] + shift[0], r[O.X] + shift[1]
    r[O.Y] -= {"lifted": 0.6, "high": 1.0}.get(kind, 0.0)
    r[O.SCORE], r[O.ALPHA] = score, alpha
    return r


def stage_bytes(ng, nd):
    """bytes stage_image needs to hold an image in shared memory: the overlap matrix and 32 lanes' assigned bits"""
    return ng * nd * 8 + (nd + 31) // 32 * 32 * 4


def max_staged(nd):
    """the largest gt count whose image with nd detections is still staged"""
    return (STAGE_BYTES - (nd + 31) // 32 * 128) // (nd * 8)


def offsets(images):
    ng = np.array([len(gc) for _g, gc, _d, _dc in images], np.int64)
    nd = np.array([len(dc) for _g, _gc, _dt, dc in images], np.int64)
    return [np.concatenate([[0], np.cumsum(v)]) for v in (ng, nd, ng * nd)]


def per_image_tp(images, metric=0, bar=0.7, d=0):
    """pass 1 of one configuration, image by image: the TP scores of each image, in gt order"""
    out = []
    for g, gc, dt, dc in images:
        g, dt = np.asarray(g, np.float64).reshape(-1, 16).tolist(), np.asarray(dt, np.float64).reshape(-1, 16).tolist()
        gc, dc = [int(c) for c in gc], [int(c) for c in dc]
        ov = O.overlaps(g, gc, dt)[metric].tolist()
        out.append(O.stats(O.above(ov, len(g), bar), O.gt_flags(g, gc, d), O.det_flags(dt, dc, d), gc,
                           [r[O.SCORE] for r in dt], [r[O.ALPHA] for r in g], [r[O.ALPHA] for r in dt], False)[4])
    return out


def n_gt_of(images, d=0):
    return sum(sum(1 for f in O.gt_flags(np.asarray(g).reshape(-1, 16).tolist(), [int(c) for c in gc], d) if f == 0)
               for g, gc, _dt, _dc in images)


def misplaced_compaction(tps):
    """the TP scores as the scan would compact them if every chunk started at slot 0 (its carry dropped), the slots
    no chunk reaches left at 0"""
    out = [0.0] * sum(len(t) for t in tps)
    for c0 in range(0, len(tps), CHUNK):
        flat = [s for t in tps[c0:c0 + CHUNK] for s in t]
        out[:len(flat)] = flat
    return out


def config_thresholds(images, metric=0, bar=0.7, d=0):
    tps = per_image_tp(images, metric, bar, d)
    return O.thresholds([s for t in tps for s in t], n_gt_of(images, d)), tps


# ------------------------------------------------------------------------------------------------ builders ----
def light(k, rs, score=None):
    """a light image: one or two easy Cars, each hit by a detection, and now and then a false positive"""
    n_car = 1 + (k % 3 == 0)
    gts = [(0, car(s, alpha=0.1 * (k % 7))) for s in range(n_car)]
    dets = [(0, det("hit", s, rs.uniform() if score is None else score, alpha=0.3)) for s in range(n_car)]
    if k % 5 == 1:
        dets.append((0, det("hit", 3, rs.uniform())))
    return image(gts, dets)


def chunk_split(n, quiet_edges=False, empty_ends=False):
    """n images whose TP scores are a random permutation, so every 1024-image chunk holds scores from the whole range.
    Image k: one or two Cars (occluded when k % 4 == 2), each hit exactly, or near (IoU 0.6) when k % 11 == 5, or missed
    when k % 7 == 3; a false positive when k % 5 == 1.  The last and first image of each chunk carry easy TPs, unless
    quiet_edges, which turns the two images on each side of every chunk edge into misses; empty_ends leaves the first
    and the last three images without rows."""
    rs = np.random.RandomState(1000 + n)
    perm = rs.permutation(3 * n)
    score = lambda k, s: (perm[3 * k + s] + 0.5) / (3 * n)
    imgs = []
    for k in range(n):
        if empty_ends and (k < 3 or k >= n - 3):
            imgs.append(image())
            continue
        edge = k >= 1 and (k + 1) % CHUNK < 2
        quiet = quiet_edges and k >= 2 and (k + 2) % CHUNK < 4
        n_car = 1 + (k % 3 == 0)
        occ = 1 if k % 4 == 2 and not edge else 0
        gts = [(0, car(s, occ=occ, alpha=0.1 * (k % 7))) for s in range(n_car)]
        dets = []
        for s in range(n_car):
            if quiet or (k % 7 == 3 and not edge):
                dets.append((0, det("hit", 4 + s, score(k, s))))
            else:
                dets.append((0, det("near2d" if k % 11 == 5 and not edge else "hit", s, score(k, s), alpha=0.3)))
        if k % 5 == 1:
            dets.append((0, det("hit", 3, score(k, 2))))
        imgs.append(image(gts, dets))
    return imgs


def rank_split(kind, n=600):
    """n images of one easy Car each, hit exactly (600 TPs: three rank CTAs, three 256-score chunks), a false positive
    in every fourth image.  two_decimals: scores rounded to 0.01 (ties across every chunk); one_score: every score
    0.5; at_threshold: false positives added at the exact value of thresholds 0, 1, 17 and the last, and one ulp below
    them; no_match: some Cars' only detections score -1e7 (the no-match value) or below, one scores one ulp above it"""
    rs = np.random.RandomState(50 + RANK_KINDS.index(kind))
    u = rs.uniform(0.0, 1.0, 2 * n)
    s = {"two_decimals": np.round(u, 2), "one_score": np.full(2 * n, 0.5)}.get(kind, np.round(u, 6))
    imgs = []
    for k in range(n):
        dets = [(0, det("hit", 0, float(s[k]), alpha=0.2))]
        if k % 4 == 0:
            dets.append((0, det("hit", 1, float(s[n + k]))))
        imgs.append(image([(0, car(0))], dets))
    if kind == "no_match":
        low = {3: O.NO_MATCH, 260: O.NO_MATCH * 1.5, 300: -1e300, 520: ABOVE_NO_MATCH}
        for k, v in low.items():
            g, gc, dt, dc = imgs[k]
            dt = dt.copy()
            dt[0, O.SCORE] = v
            imgs[k] = (g, gc, dt, dc)
        # a Car with a detection at -1e7 and one just above it in the same image; a false positive at -1e7
        imgs[400] = image([(0, car(0)), (0, car(1))], [(0, det("hit", 0, O.NO_MATCH)), (0, det("hit", 1, ABOVE_NO_MATCH)),
                                                      (0, det("hit", 2, O.NO_MATCH))])
    if kind == "at_threshold":
        thr, _ = config_thresholds(imgs)
        at = [thr[0], thr[1], thr[17], thr[-1]]
        for i, v in enumerate(at):
            for j, w in enumerate((v, float(np.nextafter(v, -1.0)))):
                k = 37 + 131 * i + j
                g, gc, dt, dc = imgs[k]
                extra = np.array([det("hit", 5 + j, w)])
                imgs[k] = (g, gc, np.concatenate([dt, extra]), np.concatenate([dc, [0]]).astype(np.int32))
    return imgs


def threshold_split(k, one_image=False):
    """k easy Cars hit exactly, each with its own score, so every configuration takes each TP score as a threshold
    (k <= 41); spread over images of one to three Cars, or all in one image (33 x 33: the global path).  Around them:
    a Van hit by a detection, a DontCare row, false positives below every TP score.  k = 0: the Cars' detections miss"""
    scores = [0.5 + 0.4 * (i + 0.5) / max(k, 1) for i in range(max(k, 1))]
    rs = np.random.RandomState(7 + k)
    rs.shuffle(scores)
    if k == 0:
        return [image([(0, car(0)), (0, car(1))], [(0, det("hit", 2, 0.8)), (0, det("hit", 3, 0.4))]),
                image([(0, car(0))], [(0, det("distant", 0, 0.9))]), image([], [(0, det("hit", 0, 0.3))])]
    sizes = [k] if one_image else []
    while sum(sizes) < k:
        sizes.append(min(1 + len(sizes) % 3, k - sum(sizes)))
    imgs, i = [], 0
    for m, n in enumerate(sizes):
        gts = [(0, car(s, alpha=0.05 * s)) for s in range(n)]
        dets = [(0, det("hit", s, scores[i + s], alpha=0.1)) for s in range(n)]
        i += n
        if m % 2 == 0:
            gts.append((1, car(n)))
            dets.append((0, det("hit", n, 0.95)))
        if m % 3 == 1:
            gts.append((2, dontcare(n + 1)))
            dets.append((0, det("hit", n + 2, 0.1)))
        imgs.append(image(gts, dets))
    return imgs


def lane_image(ng, nd, n_hit, first_hit, seed):
    """ng easy Cars; detections 0 .. first_hit - 1 and those after the hits are false positives in free slots with
    scores below 0.3; detections first_hit .. first_hit + n_hit - 1 hit Cars 0 .. n_hit - 1 with scores from 0.5 up"""
    rs = np.random.RandomState(seed)
    gts = [(0, car(s)) for s in range(ng)]
    dets = []
    for j in range(nd):
        if first_hit <= j < first_hit + n_hit:
            dets.append((0, det("hit", j - first_hit, 0.5 + 0.5 * rs.uniform(), alpha=0.2)))
        else:
            dets.append((0, det("hit", ng + j, 0.3 * rs.uniform())))
    return image(gts, dets)


def lane_split():
    """an image staged in shared memory (15 gt, 64 det) and one on the global path (40 gt, 65 det) whose hits are
    detections 32 and later (assigned-bit words 1 and 2) and hold the top scores, among light images: more than 32
    thresholds, so lanes 0 .. nt - 33 run a second threshold after a first that assigned those detections"""
    rs = np.random.RandomState(31)
    return ([light(k, rs, score=0.2 + 0.1 * rs.uniform()) for k in range(3)] + [lane_image(15, 64, 15, 32, 1)] +
            [light(k, rs, score=0.2 + 0.1 * rs.uniform()) for k in range(3, 6)] + [lane_image(40, 65, 33, 32, 2)])


def dense_image(ng, nd, seed):
    """ng labels (Cars of every difficulty, a Van every 9th, a DontCare every 13th) and nd detections: detection j
    targets slot (5 j + 1) % ng as a hit, near in 2D, near in BEV, lifted, or a false positive in a free slot"""
    rs = np.random.RandomState(seed)
    gts = []
    for s in range(ng):
        gts.append((1, car(s)) if s % 9 == 4 else (2, dontcare(s)) if s % 13 == 7 else (0, car(s, occ=s % 3)))
    dets = []
    for j in range(nd):
        kind = ("hit", "near2d", "nearbev", "lifted", "miss")[j % 5]
        t = (5 * j + 1) % ng
        sc = round(rs.uniform(), 3)
        dets.append((0, det("hit", ng + j, sc) if kind == "miss" else det(kind, t, sc, alpha=rs.uniform(-3, 3))))
    return image(gts, dets)


STAGE_SHAPES = [(63, 16), (64, 16)] + [(max_staged(nd) + e, nd) for nd in (31, 32, 33, 64, 65) for e in (0, 1)]


def stage_split():
    """every staging-edge shape of STAGE_SHAPES, each after a light image"""
    rs = np.random.RandomState(12)
    imgs = []
    for i, (ng, nd) in enumerate(STAGE_SHAPES):
        imgs += [light(i, rs), dense_image(ng, nd, 100 + i)]
    return imgs


GLOBAL_SHAPES = [(64, 16), (40, 65), (16, 64)]


def global_run_split():
    """three adjacent global-path images first, three in the middle and three last, light images between"""
    rs = np.random.RandomState(13)
    run = lambda base: [dense_image(ng, nd, base + i) for i, (ng, nd) in enumerate(GLOBAL_SHAPES)]
    return run(200) + [light(k, rs) for k in range(6)] + run(210) + [light(k, rs) for k in range(6, 12)] + run(220)


def pair_split(n=1040):
    """light images with empty ones at the start (4), around the 1024 edge (images 1020 .. 1027: empty, gt only and
    detections only) and at the end (4): runs of equal pair offsets for the overlap kernel's binary search"""
    rs = np.random.RandomState(14)
    gt_only = image([(0, car(0)), (0, car(1, occ=1))], [])
    det_only = image([], [(0, det("hit", 0, 0.7)), (0, det("hit", 1, 0.2))])
    imgs = []
    for k in range(n):
        if k < 4 or k >= n - 4:
            imgs.append(image())
        elif 1020 <= k < 1028:
            imgs.append((image(), gt_only, det_only)[k % 3])
        else:
            imgs.append(light(k, rs))
    return imgs


def no_pair_split():
    """gt rows and detection rows, never in the same image: no pairs, every gt missed, every detection false"""
    return [image([(0, car(0)), (1, car(1))], []), image([], [(0, det("hit", 0, 0.9))]), image(),
            image([(0, car(0)), (2, dontcare(1))], []), image([], [(0, det("hit", 0, 0.4)), (0, det("hit", 1, 0.6))])]


def table_split():
    """images whose configurations all differ: every kind of det() between the bars 0.7, 0.5 and 0.3 in one metric and
    not in another, on Cars of every difficulty"""
    rs = np.random.RandomState(15)
    kinds = ("hit", "near2d", "nearbev", "lifted", "far", "distant", "wide2d", "high", "hit")
    imgs = []
    for k in range(60):
        gts = [(0, car(s, occ=(k + s) % 3, trunc=0.2 * ((k + s) % 2))) for s in range(2)]
        dets = [(0, det(kinds[(k + s) % len(kinds)], s, round(rs.uniform(), 3), alpha=rs.uniform(-1, 1))) for s in range(2)]
        if k % 4 == 0:
            dets.append((0, det("hit", 3, round(rs.uniform(), 3))))
        imgs.append(image(gts, dets))
    return imgs


def val_split(n=3769, seed=2017):
    """a light split the size of KITTI val: synth.kitti_split's objects with one Car a image on average and about
    three detections, scores printed with four decimals (ties), through the product's parser"""
    from stereo_rcnn_b200 import kitti_eval as K
    from stereo_rcnn_b200 import synth
    ev = K.KittiEval("cpu")
    for g, d in synth.kitti_split(n, seed=seed, n_cars=1, n_dets=3):
        ev.add(g, d)
    return [(g, gc, d, dc) for gc, g, dc, d in ev.images]


# ------------------------------------------------------------------------------------------- BEV geometry ----
def rect(x, z, l, w, c, s):
    r = [0.0] * 16
    r[O.X], r[O.Z], r[O.L], r[O.W], r[O.COS], r[O.SIN] = x, z, l, w, c, s
    return r


def geometry_pairs():
    """(name, det, gt) BEV rows"""
    base = bev_row(0.0, 0.0, 4.0, 2.0, 0.0)
    out = [("zero_length_det", bev_row(0.0, 0.0, 0.0, 2.0, 0.3), base),
           ("zero_width_gt", base, bev_row(0.5, 0.0, 3.0, 0.0, 0.0)),
           ("both_zero_length", bev_row(0.0, 0.0, 0.0, 2.0, 0.0), bev_row(0.0, 0.0, 0.0, 2.0, 0.0)),
           ("zero_both_extents", bev_row(0.0, 0.0, 0.0, 0.0, 0.0), base)]
    for k in range(-4, 5):
        out.append(("ry_%d_half_pi" % k, bev_row(0.3, 0.1, 4.0, 2.0, k * math.pi / 2), base))
    for k, (c, s) in enumerate(((0.0, 1.0), (-1.0, 0.0), (0.0, -1.0), (1.0, 0.0))):
        out.append(("exact_quarter_turn_%d" % k, rect(0.3, 0.1, 4.0, 2.0, c, s), base))
    out += [("thin_cross", bev_row(0.0, 0.0, 6.0, 1e-4, 0.4), base),
            ("thin_both", bev_row(0.0, 0.0, 6.0, 1e-4, 0.0), bev_row(1.0, 0.0, 6.0, 1e-4, 0.0)),
            ("far_z", bev_row(3.0, 1e4 + 0.7, 4.0, 2.0, 0.25), bev_row(3.5, 1e4, 3.9, 1.6, -0.1)),
            ("far_xz", bev_row(1e4 + 0.2, 1e4 - 0.3, 4.0, 2.0, 1.2), bev_row(1e4, 1e4, 4.2, 1.7, 1.0)),
            ("collinear_edges", rect(0.0, 0.0, 4.0, 2.0, 1.0, 0.0), rect(2.0, 0.0, 4.0, 2.0, 1.0, 0.0)),
            ("nested_three_shared_edges", rect(-1.0, 0.0, 2.0, 2.0, 1.0, 0.0), base),
            ("touching_edge", rect(4.0, 0.0, 4.0, 2.0, 1.0, 0.0), base),
            ("touching_edge_offset", rect(4.0, 1.0, 4.0, 2.0, 1.0, 0.0), base),
            ("touching_corner_diamond", bev_row(2.0 + math.sqrt(2.0), 0.0, 2.0, 2.0, math.pi / 4), base),
            ("identical_rotated", bev_row(5.0, 7.0, 4.0, 2.0, 0.7), bev_row(5.0, 7.0, 4.0, 2.0, 0.7))]
    return out


ZERO_AREA = ("zero_length_det", "zero_width_gt", "both_zero_length", "zero_both_extents", "touching_edge",
             "touching_edge_offset", "touching_corner_diamond")


def full_row(b, box=(0.0, 0.0, 10.0, 60.0), y=1.6, h=1.5):
    r = list(b)
    r[O.X1], r[O.Y1], r[O.X2], r[O.Y2] = box
    r[O.Y], r[O.H] = y, h
    return r


def geometry_images():
    """one image per BEV pair, the gt once as a Car and once as a DontCare (intersection / area(det)), plus 2D boxes
    of zero width or height, 3D boxes of zero height, and bottoms at y = +-0"""
    imgs = []
    for k, (_n, d, g) in enumerate(geometry_pairs()):
        box = (10.0, 0.0, 60.0, 60.0)
        imgs.append(image([(0, full_row(g, box)), (2, full_row(g, box))],
                          [(0, _d(full_row(d, (12.0, 0.0, 62.0, 55.0)), score=0.1 + 0.02 * k))]))
    base = bev_row(0.0, 0.0, 4.0, 2.0, 0.0)
    g = full_row(base, (10.0, 10.0, 60.0, 70.0))
    flat = [full_row(base, (10.0, 10.0, 10.0, 70.0)), full_row(base, (10.0, 40.0, 60.0, 40.0)),
            full_row(base, (10.0, 10.0, 60.0, 70.0), h=0.0), full_row(base, (10.0, 10.0, 60.0, 70.0), y=0.0, h=0.0),
            full_row(base, (10.0, 10.0, 60.0, 70.0), y=-0.0, h=0.0), full_row(base, (60.0, 10.0, 90.0, 70.0))]
    imgs.append(image([(0, g), (2, g), (0, flat[2]), (0, flat[3])], [(0, _d(r, score=0.5)) for r in flat] + [(0, _d(g, score=0.6))]))
    return imgs


# ------------------------------------------------------------------------------------------------ tests ----
@pytest.mark.parametrize("n", CHUNK_SIZES)
def test_chunk_split_crosses_every_chunk_edge_with_interleaved_scores(n):
    imgs = chunk_split(n)
    assert len(imgs) == n
    thr, tps = config_thresholds(imgs)
    counts = np.array([len(t) for t in tps])
    edges = list(range(CHUNK, n, CHUNK))
    assert (n > CHUNK) == bool(edges)
    for e in edges + ([n] if n % CHUNK == 0 else []):
        assert counts[e - 1] > 0 and counts[e - 1024:e].sum() > 100
        if e < n:
            assert counts[e] > 0 and counts[e:].sum() > 0
    chunks = [[s for t in tps[c:c + CHUNK] for s in t] for c in range(0, n, CHUNK)]
    for a, b in zip(chunks, chunks[1:]):             # interleaved: each chunk's scores reach into the next one's range
        assert max(a) > min(b) and min(a) < max(b)
    assert len(thr) > LANES
    for ch in chunks:                                # every full chunk owns thresholds
        assert len(ch) < 100 or set(ch) & set(thr)
    if edges:                                        # a chunk written at the wrong offset changes the thresholds
        assert O.thresholds(misplaced_compaction(tps), n_gt_of(imgs)) != thr


def test_chunk_split_variants():
    imgs = chunk_split(2060, quiet_edges=True)
    counts = np.array([len(t) for t in per_image_tp(imgs)])
    for e in (CHUNK, 2 * CHUNK):
        assert (counts[e - 2:e + 2] == 0).all() and counts[e - 1024:e - 2].sum() > 0 and counts[e + 2:].sum() > 0
        assert all(len(imgs[k][2]) > 0 for k in range(e - 2, e + 2))       # the quiet images still have pairs
    imgs = chunk_split(2049, empty_ends=True)
    for k in (0, 1, 2, 2046, 2047, 2048):
        assert len(imgs[k][1]) == 0 and len(imgs[k][3]) == 0
    counts = np.array([len(t) for t in per_image_tp(imgs)])
    assert counts[3:6].sum() > 0 and counts[CHUNK - 1] > 0 and counts[CHUNK] > 0 and counts[2040:2046].sum() > 0


@pytest.mark.parametrize("kind", RANK_KINDS)
def test_rank_split_spans_several_blocks(kind):
    imgs = rank_split(kind)
    thr, tps = config_thresholds(imgs)
    compact = [s for t in tps for s in t]
    assert len(compact) > 2 * RANK_BLOCK
    first = {}
    across = set()
    for i, v in enumerate(compact):
        if v in first and first[v] // RANK_BLOCK != i // RANK_BLOCK:
            across.add(v)
        first.setdefault(v, i)
    if kind in ("two_decimals", "one_score"):
        assert len(across & set(thr)) >= (1 if kind == "one_score" else 10)   # tied thresholds straddle the blocks
    if kind == "one_score":
        assert thr == [0.5] * O.N_T
    if kind == "at_threshold":
        fp_scores = {float(r[O.SCORE]) for g, gc, dt, dc in imgs for r in dt[1:]}
        at = [v for v in thr if v in fp_scores]
        below = [v for v in thr if float(np.nextafter(v, -1.0)) in fp_scores]
        assert len(set(at)) >= 4 and len(set(below)) >= 4 and max(thr) in at and min(thr) in at
        assert config_thresholds(imgs)[0] == thr
    if kind == "no_match":
        assert all(s > O.NO_MATCH for s in compact) and ABOVE_NO_MATCH in compact and min(thr) == ABOVE_NO_MATCH
        for k in (3, 260, 300):
            assert tps[k] == [] and imgs[k][2][0, O.SCORE] <= O.NO_MATCH
        assert tps[400] == [ABOVE_NO_MATCH]


@pytest.mark.parametrize("k", THRESHOLD_COUNTS)
def test_threshold_split_reaches_its_count(k):
    r = O.evaluate(threshold_split(k))
    assert (r["n_thresholds"] == k).all() and (r["n_gt"] == max(k, 3 if k == 0 else k)).all()
    if k == 33:
        imgs = threshold_split(33, one_image=True)
        ng, nd = len(imgs[0][1]), len(imgs[0][3])
        assert stage_bytes(ng, nd) > STAGE_BYTES and nd > LANES
        assert (O.evaluate(imgs)["n_thresholds"] == 33).all()


def test_lane_split_assigns_high_words_at_a_lanes_first_threshold():
    imgs = lane_split()
    r = O.evaluate(imgs)
    nt = int(r["n_thresholds"].min())
    assert nt > LANES
    staged = {False: 0, True: 0}
    for g, gc, dt, dc in imgs:
        nd = len(dc)
        if nd <= LANES:
            continue
        staged[stage_bytes(len(gc), nd) <= STAGE_BYTES] += 1
        for c in range(len(r["n_thresholds"])):
            first = r["thresholds"][c, :nt - LANES]     # first thresholds of the lanes that run two
            hi = dt[LANES:, O.SCORE]
            assert (hi[:, None] >= first[None, :]).any()
    assert staged == {False: 1, True: 1}


def test_stage_shapes_straddle_the_limit():
    assert stage_bytes(63, 16) == STAGE_BYTES and stage_bytes(64, 16) == 8320
    for nd in (31, 32, 33, 64, 65):
        ng = max_staged(nd)
        assert stage_bytes(ng, nd) <= STAGE_BYTES < stage_bytes(ng + 1, nd)
    imgs = stage_split()
    shapes = [(len(gc), len(dc)) for _g, gc, _dt, dc in imgs[1::2]]
    assert shapes == STAGE_SHAPES
    r = O.evaluate(imgs)
    last = r["n_thresholds"] - 1
    assert (last >= 0).all() and (r["fp"][np.arange(len(last)), last] > 0).all()
    imgs = global_run_split()
    glob = [stage_bytes(len(gc), len(dc)) > STAGE_BYTES for _g, gc, _dt, dc in imgs]
    n = len(imgs)
    assert all(glob[:3]) and all(glob[9:12]) and all(glob[n - 3:]) and sum(glob) == 9


def test_pair_split_has_runs_of_equal_offsets():
    imgs = pair_split()
    _go, _do, po = offsets(imgs)
    assert len(imgs) > CHUNK
    assert (po[:5] == 0).all() and (po[-5:] == po[-1]).all()
    assert len(set(po[1020:1029].tolist())) == 1 and po[1028] > 0 and po[-1] > po[1028]
    go, do, po = offsets(no_pair_split())
    assert po[-1] == 0 and go[-1] > 0 and do[-1] > 0
    r = O.evaluate(no_pair_split())
    assert (r["n_thresholds"] == 0).all() and (r["n_gt"] > 0).all()


def test_table_split_configurations_differ():
    for bars in ((0.7, 0.5, 0.3), FOUR_BARS):
        r = O.evaluate(table_split(), bars)
        nb = len(bars)
        blocks = [tuple(r["ap"][(m * nb + b) * 3:(m * nb + b) * 3 + 3, :2].ravel()) for m in range(3) for b in range(nb)
                  if 0.0 < bars[b] < 1.0]
        assert len(set(blocks)) == len(blocks), bars


def test_bev_geometry_against_scipy():
    for name, d, g in geometry_pairs():
        got = O.bev_intersection(d, g)
        assert math.isfinite(got) and math.isfinite(O.overlap_bev(d, g)) and math.isfinite(O.overlap_bev(d, g, True))
        if name in ZERO_AREA:
            assert got == 0.0 and O.overlap_bev(d, g) == 0.0 and O.overlap_bev(d, g, True) == 0.0, name
            continue
        ref = scipy_area(d, g)
        # the shoelace sum takes products of absolute coordinates: far from the origin it rounds at their scale
        span = max(abs(d[O.X]), abs(d[O.Z]), abs(g[O.X]), abs(g[O.Z])) + 10.0
        tol = 1e-9 * ref + 1e-12 + 16 * np.finfo(np.float64).eps * span * span
        assert ref > 0 and abs(got - ref) <= tol, (name, got, ref)
        assert abs(O.bev_intersection(g, d) - ref) <= tol, name


def test_zero_extents_give_zero_overlap():
    """the zero-denominator rule: l or w = 0 in BEV, h = 0 in 3D, zero width or height in 2D, on both criteria"""
    b = full_row(bev_row(0.0, 0.0, 4.0, 2.0, 0.0), (10.0, 10.0, 60.0, 70.0))
    z = lambda **kw: _d(b, **kw)
    for d, g in ((z(l=0.0), b), (b, z(w=0.0)), (z(l=0.0), z(l=0.0)), (z(w=0.0), z(w=0.0))):
        assert O.overlap_bev(d, g) == 0.0 and O.overlap_bev(d, g, True) == 0.0 and O.overlap_3d(d, g) == 0.0
    for d, g in ((z(h=0.0), b), (b, z(h=0.0)), (z(h=0.0), z(h=0.0)), (z(h=0.0, y=0.0), z(h=0.0, y=-0.0))):
        assert O.overlap_3d(d, g) == 0.0 and O.overlap_3d(d, g, True) == 0.0 and O.overlap_bev(d, g) == 1.0
    for d in (z(x2=10.0), z(y2=10.0), z(x1=60.0), z(y1=70.0)):
        assert O.overlap_2d(d, b) == 0.0 and O.overlap_2d(b, d) == 0.0 and O.overlap_2d(d, b, True) == 0.0
    assert O.overlap_2d(b, b) == 1.0
    ov = np.concatenate([O.overlaps(g, gc, dt).ravel() for g, gc, dt, _dc in geometry_images()])
    assert np.isfinite(ov).all() and (ov == 0).any() and (ov > 0).any()
