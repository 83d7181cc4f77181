"""Generate tests/golden/eval_geometry.npz: the REFERENCE's KITTI overlaps at their geometric edges.

    NUMBA_ENABLE_CUDASIM=1 python tests/golden/make_golden_eval_geometry.py

Runs mmdet/core/post_processing/rotate_nms_gpu.py:rotate_iou_gpu_eval (numba.cuda code, in numba's CUDA simulator)
and mmdet/core/evaluation/kitti_eval.py:image_box_overlap / d3_box_overlap (numba-jitted CPU code) on constructed
pairs, one pair per call, and stores per pair:

  bev_*   rotated BEV pairs (x, y, dx, dy, yaw) as (box, query): the reference's value under criteria -1, 0, 1, 2, the
          number of points its quadrilateral_intersection collects, and whether the reference is defined there.  Its
          point buffer is a 16-float local array, 8 points: a pair that collects more writes past it (the simulator
          raises IndexError), so its value is undefined and stored as NaN.  The count comes from a restatement of the
          reference's corner, inside and segment tests in float32 below, cross-checked here against the simulator:
          it raises exactly when the count exceeds 8.
  bb_*    2-D image boxes (x0, y0, x1, y1) as (detection, GT): image_box_overlap under the four criteria.
  d3_*    camera boxes (x, y, z, l, h, w, ry) as (detection, GT): d3_box_overlap under the four criteria.  Where the
          reference divides by zero (numba raises ZeroDivisionError) the value is undefined and stored as NaN.
  e2e_*   a split of one frame per family plus GT frames evaluated against themselves at yaw 0.3 and at yaw 0, the
          official text of the reference's get_official_eval_result on the frames where it is defined and on each
          self-evaluation alone.

Every pair carries its family name, so a failing comparison names its case.
"""
import importlib.util
import math
import os
import sys

import numpy as np
import numpy.ma  # noqa: F401  (before make_golden's np.bool shim)
import numba  # noqa: F401
try:
    import scipy.sparse  # noqa: F401
except Exception:
    pass

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import import_reference_mmdet  # noqa: E402

F = np.float32
CRITERIA = (-1, 0, 1, 2)
PI = math.pi


def _ulp_up(v):
    return float(np.nextafter(F(v), F(np.inf)))


def bev_pairs():
    """(family, box, query) of the rotated BEV overlap."""
    out = []

    def add(fam, b, q):
        out.append((fam, [float(v) for v in b], [float(v) for v in q]))

    for yaw in (0.0, 0.3, PI / 2, PI, -PI / 2, 1e3):
        add("identical", (0, 0, 4, 2, yaw), (0, 0, 4, 2, yaw))
        add("identical_at_5_5", (5, 5, 4, 2, yaw), (5, 5, 4, 2, yaw))
    for yaw in (0.0, 0.3, PI / 2, 1e3):
        add("flipped_at_origin", (0, 0, 4, 2, yaw), (0, 0, 4, 2, yaw + PI))
        add("flipped_at_5_5", (5, 5, 4, 2, yaw), (5, 5, 4, 2, yaw + PI))
    for yaw in (0.0, 0.3):
        add("near_yaw_1e-7", (0, 0, 4, 2, yaw), (0, 0, 4, 2, yaw + 1e-7))
        add("near_centre_1ulp", (1, 1, 4, 2, yaw), (_ulp_up(1), 1, 4, 2, yaw))
        add("near_extent_1ulp", (1, 1, 4, 2, yaw), (1, 1, _ulp_up(4), 2, yaw))
    for yaw in (0.0, 0.3):
        c, s = math.cos(yaw), math.sin(yaw)

        def at(u, v):        # a point of the box frame rotated as rbbox_to_corners rotates (clockwise by yaw)
            return c * u + s * v, -s * u + c * v
        add("shared_edge", (*at(0, 0), 2, 2, yaw), (*at(2, 0), 2, 2, yaw))
        add("collinear_edges", (*at(0, 0), 4, 2, yaw), (*at(2, 0), 4, 2, yaw))
        add("collinear_one_edge", (*at(0, 0), 4, 2, yaw), (*at(1, 0.5), 2, 1, yaw))
        add("corner_contact", (*at(0, 0), 2, 2, yaw), (*at(2, 2), 2, 2, yaw))
        add("nested_same_centre", (*at(0, 0), 4, 2, yaw), (*at(0, 0), 2, 1, yaw))
        add("nested_off_centre", (*at(0, 0), 4, 2, yaw), (*at(0.5, 0.2), 1, 0.5, yaw))
        add("nested_other_yaw", (*at(0, 0), 6, 6, yaw), (*at(0.5, 0.5), 1, 2, yaw + 0.7))
        add("square_45_octagon", (0, 0, 2, 2, yaw), (0, 0, 2, 2, yaw + PI / 4))
        add("square_90", (0, 0, 2, 2, yaw), (0, 0, 2, 2, yaw + PI / 2))
        add("cross", (0, 0, 4, 1, yaw), (0, 0, 4, 1, yaw + PI / 2))
        add("cross_off_centre", (0.5, 0.2, 4, 1, yaw), (0, 0, 4, 1, yaw + PI / 2))
    for z in (0.0, 1e-6, 1e-30):
        add("zero_or_tiny_both", (0, 0, z, z, 0), (0, 0, 2, 2, 0))
        add("zero_or_tiny_one", (0, 0, z, 2, 0.3), (0, 0, 2, 2, 0))
        add("zero_or_tiny_one", (0.5, 0, 2, z, 0), (0, 0, 2, 2, 0.3))
    add("zero_or_tiny_both", (0, 0, 0, 0, 0), (0, 0, 0, 0, 0))
    add("zero_or_tiny_both", (5, 5, 0, 0, 0), (0, 0, 2, 2, 0))
    for x, y in ((70.0, 0.0), (70.4, 39.9), (35.0, -40.0), (1e4, 1e4), (-1e4, 1e4)):
        add("far_identical", (x, y, 3.9, 1.6, 0.3), (x, y, 3.9, 1.6, 0.3))
        add("far_shifted", (x, y, 3.9, 1.6, 0.3), (x + 0.5, y + 0.25, 3.9, 1.6, 0.4))
        add("far_shifted", (x, y, 3.9, 1.6, 0.0), (x + 1.0, y, 3.9, 1.6, 0.0))
    nan, inf = math.nan, math.inf
    # no infinite yaw: math.cos raises on it in the simulator, where the device's cos gives NaN
    for col, v in ((0, nan), (1, nan), (2, nan), (3, nan), (4, nan), (0, inf), (1, -inf), (2, inf), (3, -inf)):
        b = [0, 0, 4, 2, 0.3]
        b[col] = v
        add("nonfinite_%d" % col, b, (0.5, 0.2, 3.9, 1.8, 0.1))
        add("nonfinite_%d" % col, (0.5, 0.2, 3.9, 1.8, 0.1), b)
    return out


def image_pairs():
    """(family, detection bbox, GT bbox) of the 2-D overlap."""
    out = []
    base = [50.0, 0.0, 100.0, 2.0]

    def add(fam, b, q):
        out.append((fam, [float(v) for v in b], [float(v) for v in q]))

    add("contained", (10, 10, 20, 20), (0, 0, 40, 40))
    add("contained", (0, 0, 40, 40), (10, 10, 20, 20))
    add("contained", (0, 0, 40, 40), (0, 0, 40, 40))
    add("inverted", (20, 0, 10, 10), (0, 0, 40, 40))
    add("inverted", (0, 20, 10, 10), (0, 0, 40, 40))
    add("inverted", (20, 20, 10, 10), (0, 0, 40, 40))
    add("inverted", (0, 0, 40, 40), (20, 20, 10, 10))
    add("zero_area", (10, 10, 10, 20), (0, 0, 40, 40))
    add("zero_area", (10, 10, 20, 10), (0, 0, 40, 40))
    add("zero_area", (10, 10, 10, 10), (10, 10, 10, 10))
    add("touching", (0, 0, 10, 10), (10, 0, 20, 10))
    add("touching", (0, 0, 10, 10), (0, 10, 10, 20))
    add("touching", (0, 0, 10, 10), (10, 10, 20, 20))
    for col in range(4):
        for v in (math.nan, math.inf, -math.inf):
            b = list(base)
            b[col] = v
            add("nonfinite_dt_%d" % col, b, base)
            add("nonfinite_gt_%d" % col, base, b)
    add("nonfinite_gt_12", base, (50, math.nan, math.nan, 2))
    add("nonfinite_dt_12", (50, math.nan, math.nan, 2), base)
    return out


def cam_pairs():
    """(family, detection, GT) camera boxes (x, y, z, l, h, w, ry) of the 3-D overlap.  The footprints are chosen so
    that the reference's BEV intersection is positive (yaw 0, or rotated boxes off each other's centre: not the
    rotated identical pairs whose intersection it makes 0), so that its height computation decides the value; only
    zero_bev, flipped_at_origin, huge_cross, huge_overlap and the non-finite BEV columns (0, 2, 3, 5, 6) are about
    the footprint itself."""
    out = []
    gt = [0.0, 1.0, 10.0, 4.0, 1.5, 2.0, 0.0]          # y spans [y - h, y] = [-0.5, 1]
    dt = [0.5, 1.0, 10.3, 4.0, 1.5, 2.0, 0.0]          # the same heights, the footprint shifted

    def add(fam, b, q):
        out.append((fam, [float(v) for v in b], [float(v) for v in q]))

    def tall(y, h, b=dt):
        return b[:1] + [y] + b[2:4] + [h] + b[5:]

    add("overlapping", dt, gt)
    add("overlapping", (0.3, 1, 10.2, 4, 1.5, 2, 0.25), (0, 1, 10, 4, 1.5, 2, 0.1))
    add("contained", (0, 0.8, 10, 2, 0.5, 1, 0), gt)
    add("contained", gt, (0, 0.8, 10, 2, 0.5, 1, 0))
    add("contained", gt, gt)
    add("heights_touch", tall(2, 1), gt)                # [1, 2] against [-0.5, 1]
    add("heights_touch", tall(-0.5, 1), gt)             # [-1.5, -0.5] against [-0.5, 1]
    add("heights_touch", tall(1, 1.5), tall(-0.5, 1, gt))
    add("heights_apart", tall(3, 1), gt)
    add("zero_height", tall(1, 0), gt)
    add("zero_height", dt, tall(1, 0, gt))
    add("zero_height", tall(0.5, 0), gt)                # a zero height inside the other interval
    add("inverted_height", tall(1, -1), gt)
    add("inverted_height", dt, tall(0, -1, gt))
    add("zero_bev", (0, 1, 10, 0, 1.5, 0, 0), (0, 1, 10, 2, 1.5, 2, 0))
    add("flipped_at_origin", (0, 1, 0, 4, 1.5, 2, 0.3), (0, 1, 0, 4, 1.5, 2, 0.3 + PI))
    add("huge_cross", (0, 1, 10, 3e38, 1.5, 2, 0), (0, 1, 10, 2, 1.5, 3e38, 0))   # BEV intersection NaN
    add("huge_overlap", (0, 1, 10, 3e38, 1.5, 3e38, 0), (1, 1, 11, 3e38, 1.5, 3e38, 0))   # BEV intersection inf
    for col in range(7):
        for v in (math.nan, math.inf, -math.inf) if col < 6 else (math.nan,):
            b = list(dt)
            b[col] = v
            add("nonfinite_dt_%d" % col, b, gt)
            b = list(gt)
            b[col] = v
            add("nonfinite_gt_%d" % col, dt, b)
    return out


# ------------------------------------------------------------------ restated point count
def _corners32(box):
    cx, cy, dx, dy, ang = (F(v) for v in box)
    c, s = F(math.cos(ang)), F(math.sin(ang))
    hx, hy = -dx / F(2), -dy / F(2)
    xs, ys = [hx, hx, -hx, -hx], [hy, -hy, -hy, hy]
    return [(F(c * x + s * y + cx), F(-s * x + c * y + cy)) for x, y in zip(xs, ys)]


def _inside32(px, py, q):
    ab0, ab1 = q[1][0] - q[0][0], q[1][1] - q[0][1]
    ad0, ad1 = q[3][0] - q[0][0], q[3][1] - q[0][1]
    ap0, ap1 = px - q[0][0], py - q[0][1]
    abab, abap = ab0 * ab0 + ab1 * ab1, ab0 * ap0 + ab1 * ap1
    adad, adap = ad0 * ad0 + ad1 * ad1, ad0 * ap0 + ad1 * ap1
    return bool(abab >= abap and abap >= 0 and adad >= adap and adap >= 0)


def _crosses32(p1, p2, i, j):
    a, b, c, d = p1[i], p1[(i + 1) % 4], p2[j], p2[(j + 1) % 4]
    acd = (d[1] - a[1]) * (c[0] - a[0]) > (c[1] - a[1]) * (d[0] - a[0])
    bcd = (d[1] - b[1]) * (c[0] - b[0]) > (c[1] - b[1]) * (d[0] - b[0])
    abc = (c[1] - a[1]) * (b[0] - a[0]) > (b[1] - a[1]) * (c[0] - a[0])
    abd = (d[1] - a[1]) * (b[0] - a[0]) > (b[1] - a[1]) * (d[0] - a[0])
    return bool(acd != bcd and abc != abd)


def collected_points(box, query):
    """How many points quadrilateral_intersection (rotate_nms_gpu.py:317-337) collects for inter(query, box)."""
    with np.errstate(all="ignore"):
        p1, p2 = _corners32(query), _corners32(box)
        n = sum(_inside32(*p1[i], p2) + _inside32(*p2[i], p1) for i in range(4))
        return n + sum(_crosses32(p1, p2, i, j) for i in range(4) for j in range(4))


# ------------------------------------------------------------------ the end-to-end split
def _anno(cam, bbox, score=None):
    n = len(bbox)
    cam, bbox = np.asarray(cam, np.float64).reshape(n, 7), np.asarray(bbox, np.float64).reshape(n, 4)
    a = dict(name=np.array(["Car"] * n, "<U8"), truncated=np.zeros(n), occluded=np.zeros(n, np.int64), alpha=np.zeros(n),
             bbox=bbox, dimensions=cam[:, 3:6], location=cam[:, :3], rotation_y=cam[:, 6])
    if score is not None:
        a["score"] = np.full(n, score)
    return a


def dontcare_frame():
    """(gt, dt) of a frame that puts NaN and +-inf into every bbox column of DontCare rows and of the detections
    tested against them (image_box_overlap(dt, dontcare, 0) > min overlap, kitti_eval.py:259-270).  A car GT with a
    detection of score 0.5 on it, then 24 DontCare boxes 100 x 60 pixels, each with a detection of score 0.9 on the
    same box: in the first 12 the DontCare box carries the non-finite value, in the last 12 the detection does.  Each
    detection the DontCare test does not take is a false positive above the true positive's score, so the test's
    outcome shows in the AP.  The camera boxes are apart, so only the bbox metric's DontCare test joins them."""
    variants = [(c, v) for c in range(4) for v in (math.nan, math.inf, -math.inf)]
    boxes = [[250.0 + 150 * i, 100.0, 350.0 + 150 * i, 160.0] for i in range(2 * len(variants))]
    dc_bb, dt_bb = [list(b) for b in boxes], [list(b) for b in boxes]
    for i, (c, v) in enumerate(variants):
        dc_bb[i][c] = v
        dt_bb[len(variants) + i][c] = v

    def cams(n, z0):
        return [[-10.0 + 4 * i, 1.6, z0, 3.9, 1.5, 1.6, 0.0] for i in range(n)]
    car = [[0.0, 1.6, 20.0, 3.9, 1.5, 1.6, 0.0]]
    gt = _anno(car + cams(len(boxes), 40.0), [[50.0, 100.0, 150.0, 160.0]] + dc_bb)
    gt["name"][1:] = "DontCare"
    dt = _anno(car + cams(len(boxes), 60.0), [[50.0, 100.0, 150.0, 160.0]] + dt_bb, 0.9)
    dt["score"][0] = 0.5
    return gt, dt


def e2e_frames(bev, img, cam):
    """One frame per family, its pairs as (detection, GT) objects, the DontCare frame (dontcare_frame), plus 50 frames of four cars evaluated against
    themselves at yaw 0.3 and 50 at yaw 0 (the reference splits a split into 50 parts, so a split has 50 frames or
    more).  BEV pairs become camera boxes (x, 1.6, y, dx, 1.5, dy, yaw) with image boxes 60 pixels tall; 2-D pairs,
    stretched 30 times in y so that they pass the height limits, keep one camera box; 3-D pairs get equal image
    boxes.  Returns (name, gt, dt) triples."""
    frames = []
    for fams, boxes, queries, kind in ((bev[0], bev[1], bev[2], "bev"), (img[0], img[1], img[2], "bb"),
                                       (cam[0], cam[1], cam[2], "d3")):
        fams = np.asarray(fams)
        for fam in dict.fromkeys(fams.tolist()):
            sel = np.flatnonzero(fams == fam)
            b, q = np.asarray(boxes, np.float64)[sel], np.asarray(queries, np.float64)[sel]
            n = len(sel)
            tall = np.tile([100.0, 100.0, 200.0, 160.0], (n, 1))
            if kind == "bev":
                dc, gc = (np.stack([v[:, 0], np.full(n, 1.6), v[:, 1], v[:, 2], np.full(n, 1.5), v[:, 3], v[:, 4]], 1)
                          for v in (b, q))
                db = gb = tall
            elif kind == "bb":
                dc = gc = np.tile([2.0, 1.6, 20.0, 3.9, 1.5, 1.6, 0.3], (n, 1))
                db, gb = b * [1, 30, 1, 30], q * [1, 30, 1, 30]
            else:
                dc, gc = b, q
                db = gb = tall
            frames.append(("%s:%s" % (kind, fam), _anno(gc, gb), _anno(dc, db, 0.9)))
    frames.append(("dontcare",) + dontcare_frame())
    for name, yaw in (("self_yaw_0.3", 0.3), ("self_yaw_0", 0.0)):
        cams = [[x, 1.6, z, 3.9, 1.5, 1.6, yaw] for x, z in ((-6.0, 12.0), (0.0, 20.0), (5.0, 30.0), (9.0, 15.0))]
        bbs = [[100.0 + 150 * i, 100.0, 200.0 + 150 * i, 160.0] for i in range(4)]
        frames += [(name, _anno(cams, bbs), _anno(cams, bbs, 0.9))] * 50
    return frames


def store_frames(out, frames):
    """Each distinct frame once; e2e_repeat says how many times it follows itself in the split."""
    uniq, rep = [], []
    for f in frames:
        if uniq and f is uniq[-1]:
            rep[-1] += 1
        else:
            uniq.append(f); rep.append(1)
    out["e2e_names"], out["e2e_repeat"] = np.array([f[0] for f in uniq]), np.array(rep)
    for i, (_, g, d) in enumerate(uniq):
        for k, v in g.items():
            out["e2e_gt%d_%s" % (i, k)] = v
        for k, v in d.items():
            out["e2e_dt%d_%s" % (i, k)] = v


def main():
    assert os.environ.get("NUMBA_ENABLE_CUDASIM") == "1", "run with NUMBA_ENABLE_CUDASIM=1 (no GPU here)"
    import_reference_mmdet()
    for k in list(sys.modules):
        if k.startswith("mmdet.core.post_processing"):
            del sys.modules[k]
    spec = importlib.util.spec_from_file_location(
        "mmdet.core.post_processing.rotate_nms_gpu", "/root/reference/mmdet/core/post_processing/rotate_nms_gpu.py")
    m = importlib.util.module_from_spec(spec); sys.modules[spec.name] = m; spec.loader.exec_module(m)
    spec = importlib.util.spec_from_file_location("ref_kitti_eval", "/root/reference/mmdet/core/evaluation/kitti_eval.py")
    ke = importlib.util.module_from_spec(spec); spec.loader.exec_module(ke)
    import warnings
    warnings.simplefilter("ignore")
    np.seterr(all="ignore")
    out = {}

    bev = bev_pairs()
    P = len(bev)
    box, query = (np.array([p[k] for p in bev], np.float32) for k in (1, 2))
    ref = np.full((P, 4), np.nan, np.float32)
    npts = np.array([collected_points(b, q) for b, q in zip(box, query)], np.int32)
    for p in range(P):
        for ci, c in enumerate(CRITERIA):
            try:
                ref[p, ci] = m.rotate_iou_gpu_eval(box[p:p + 1], query[p:p + 1], c)[0, 0]
                raised = False
            except IndexError:
                raised = True
            assert raised == (npts[p] > 8), (bev[p][0], npts[p], raised)
    out.update(bev_family=np.array([p[0] for p in bev]), bev_box=box, bev_query=query, bev_ref=ref,
               bev_npts=npts, bev_defined=npts <= 8)

    img = image_pairs()
    b4, q4 = (np.array([p[k] for p in img], np.float64) for k in (1, 2))
    ref = np.full((len(img), 4), np.nan)
    for p in range(len(img)):
        for ci, c in enumerate(CRITERIA):
            ref[p, ci] = ke.image_box_overlap(b4[p:p + 1], q4[p:p + 1], c)[0, 0]
    out.update(bb_family=np.array([p[0] for p in img]), bb_box=b4, bb_query=q4, bb_ref=ref)

    cam = cam_pairs()
    b7, q7 = (np.array([p[k] for p in cam], np.float64) for k in (1, 2))
    ref = np.full((len(cam), 4), np.nan, np.float32)
    defined = np.ones((len(cam), 4), bool)
    cnt = np.array([collected_points(b[[0, 2, 3, 5, 6]], q[[0, 2, 3, 5, 6]]) for b, q in zip(b7, q7)], np.int32)
    for p in range(len(cam)):
        for ci, c in enumerate(CRITERIA):
            if cnt[p] > 8:
                defined[p, ci] = False
                continue
            try:
                ref[p, ci] = ke.d3_box_overlap(b7[p:p + 1], q7[p:p + 1], c)[0, 0]
            except ZeroDivisionError:
                defined[p, ci] = False
    out.update(d3_family=np.array([p[0] for p in cam]), d3_box=b7, d3_query=q7, d3_ref=ref, d3_defined=defined,
               d3_npts=cnt)

    frames = e2e_frames((out["bev_family"], out["bev_box"], out["bev_query"]),
                        (out["bb_family"], out["bb_box"], out["bb_query"]),
                        (out["d3_family"], out["d3_box"], out["d3_query"]))
    store_frames(out, frames)
    # the official text where the reference is defined: every frame whose pairs it evaluates without overflow or a
    # division by zero; and the two self-evaluations alone
    def defined(g, d):
        cam = [np.concatenate([a["location"], a["dimensions"], a["rotation_y"][:, None]], 1) for a in (d, g)]
        if any(collected_points(x[[0, 2, 3, 5, 6]], y[[0, 2, 3, 5, 6]]) > 8 for x in cam[0] for y in cam[1]):
            return False
        try:
            ke.d3_box_overlap(cam[0], cam[1], -1)
        except ZeroDivisionError:
            return False
        return True
    keep = np.array([not f[0].startswith("self") and defined(f[1], f[2]) for f in frames])
    assert keep.sum() >= 50, keep.sum()
    out["e2e_defined"] = np.array([k for k, f, g in zip(keep, frames, [None] + frames[:-1]) if f is not g])
    names = np.array([f[0] for f in frames])
    for key, sel in (("e2e_text", keep), ("e2e_text_self_yaw_0.3", names == "self_yaw_0.3"),
                     ("e2e_text_self_yaw_0", names == "self_yaw_0")):
        gts = [f[1] for f, s in zip(frames, sel) if s]
        dts = [f[2] for f, s in zip(frames, sel) if s]
        out[key] = np.array(ke.get_official_eval_result(gts, dts, [0]))
    text = str(out["e2e_text"])
    np.savez_compressed(os.path.join(HERE, "eval_geometry.npz"), **out)
    print(text)
    print("bev pairs %d (%d undefined), 2-D pairs %d, 3-D pairs %d (%d undefined entries)"
          % (P, int((npts > 8).sum()), len(img), len(cam), int((~out["d3_defined"]).sum())))


if __name__ == "__main__":
    main()
