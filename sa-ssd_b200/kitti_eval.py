"""KITTI official-style evaluation (SURVEY.md §8 row f4): bbox / BEV / 3-D AP (R11) and AOS.

Mirrors the reference's evaluator so that `tools/test.py`-style code can swap the import:

* `get_official_eval_result(gt_annos, dt_annos, current_classes, difficultys)` -> the same printed table
  (mmdet/core/evaluation/kitti_eval.py:791-851); `official_eval` additionally returns the AP arrays;
* `get_coco_eval_result(gt_annos, dt_annos, current_classes)` -> the COCO-style table, AP averaged over ten IoU
  thresholds per class (kitti_eval.py:853-930); `coco_eval` additionally returns the AP arrays;
* `rotate_iou_gpu_eval(boxes, query_boxes, criterion)` <- mmdet/core/post_processing/rotate_nms_gpu.py:592-627.

What runs where: with no ``overlap_fn`` (the product path) everything after flattening the annotations runs on the
device (csrc/kitti_match.cu, `_eval_device`): the ignore flags, the rotated overlaps (`sassd_rotate_overlap_eval`,
one launch per criterion for every (set, frame)), the 2-D and 3-D overlaps, both matching passes, the 41 score
thresholds and the per-threshold sums over frames, for every detection set, class, difficulty, metric and
min-overlap row at once; only the precision / recall ratios, their envelope and the AP sums run in numpy on the
downloaded sums.  With an injected ``overlap_fn`` the host path runs: vectorised float64 numpy overlaps, per-frame
`clean_gt` / `clean_dt` and the host C++ matcher `sassd_kitti_match` (numba-jitted CPU loops in the reference).
Both paths give the same arrays bit for bit.  Annotations are dicts of numpy arrays as produced by
`results.kitti_bbox2results` / the reference's `get_label_annos` (camera-frame boxes, dimensions l, h, w), or an
AnnoBlock: the same rows as flat columns on the device, built from dicts or parsed from a directory of KITTI files on
the device (`read_block`, csrc/kitti_parse.cu).

``eval_many(..., ranges=[e0, e1, ...])`` adds every table per bin [e_i, e_i+1) of ground distance from the camera (more
difficulty entries of the same evaluation), and ``match_table`` / ``eval_many(..., match=True)`` the evaluator's own
per-object assignment with the 3-D true positives' ATE / ASE / AOE (``tp_errors``).  ``eval_many(...,
bootstrap=idx)`` adds every table over bootstrap replicates of the frames (``bootstrap_indices``), each replicate bit for
bit the evaluation of its resampled lists, with ``percentile_interval`` / ``paired_summary`` to summarise them.  The
replicates may also be a ``ReplicateLists`` of lists of any length: ``bootstrap_groups`` draws whole raw drives
(a drive-level bootstrap, from the devkit's frame mapping), and ``per_drive_report`` evaluates each drive's own frames.

    python -m sassd_b200.kitti_eval --data-root DIR [--split val] --results DIR [DIR ...] [--classes Car ...]
                                    [--r40] [--coco] [--json FILE] [--ranges EDGE ...] [--matches FILE.npz]
                                    [--bootstrap R [--bootstrap-seed S] [--bootstrap-by frame|drive]]
                                    [--mapping DIR [--per-drive]]

evaluates directories of result files against a split's labels (`main`, `eval_dirs`).
"""
import argparse
import ctypes
import json
import os
import sys
import time

import numpy as np

from . import lib as _lib

CLASS_NAMES = ['car', 'pedestrian', 'cyclist', 'van', 'person_sitting', 'car', 'tractor', 'trailer']
CLASS_TO_NAME = {0: 'Car', 1: 'Pedestrian', 2: 'Cyclist', 3: 'Van', 4: 'Person_sitting', 5: 'car', 6: 'tractor',
                 7: 'trailer'}
MIN_HEIGHT, MAX_OCCLUSION, MAX_TRUNCATION = (40, 25, 25), (0, 1, 2), (0.15, 0.3, 0.5)
# [metric (bbox, bev, 3d), class]: the two official overlap sets (kitti_eval.py:792-797)
OVERLAP_0_7 = np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.7, 0.7, 0.7]] * 3)
OVERLAP_0_5 = np.array([[0.7, 0.5, 0.5, 0.7, 0.5, 0.5, 0.5, 0.5], [0.5, 0.25, 0.25, 0.5, 0.25, 0.5, 0.5, 0.5],
                        [0.5, 0.25, 0.25, 0.5, 0.25, 0.5, 0.5, 0.5]])
# class -> (start, stop, num) of the COCO-style overlaps, the same for the three metrics (kitti_eval.py:869-879)
COCO_RANGE = {0: (0.5, 0.95, 10), 1: (0.25, 0.7, 10), 2: (0.25, 0.7, 10), 3: (0.5, 0.95, 10), 4: (0.25, 0.7, 10),
              5: (0.5, 0.95, 10), 6: (0.5, 0.95, 10), 7: (0.5, 0.95, 10)}
TABLES = (11, 40, "coco")       # official AP at 11 / 40 recall positions, COCO-style AP


def _p(a):
    return ctypes.c_void_p(a.ctypes.data) if a is not None else None


def _offsets(counts, dtype=np.int32):
    return np.concatenate([[0], np.cumsum(counts)]).astype(dtype)


# ------------------------------------------------------------------ overlaps
def _rotated_overlaps_device(boxes, box_off, query, query_off, out_off, criterion):
    """All frames in one kernel launch (float32, [sum nb*nq] flat)."""
    import torch
    from . import ops
    ops.require_cuda()
    dev = torch.device("cuda")
    total = int(out_off[-1])
    out = torch.zeros((max(total, 1),), dtype=torch.float32, device=dev)
    if total:
        t = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (boxes, box_off, query, query_off, out_off)]
        pairs = np.diff(box_off).astype(np.int64) * np.diff(query_off).astype(np.int64)
        ops._call("sassd_rotate_overlap_eval", None, ops._ptr(t[0]), ops._ptr(t[1]), ops._ptr(t[2]), ops._ptr(t[3]),
                  ops._ptr(t[4]), len(box_off) - 1, int(criterion), int(pairs.max()), ops._ptr(out), ops._stream())
    return out[:total].cpu().numpy()


def _rotated_overlaps(boxes_list, query_list, criterion, overlap_fn=None):
    """Per-frame [nb, nq] float32 overlap matrices.  `overlap_fn(boxes, query, criterion)` replaces the CUDA kernel
    (the tests inject the CPU oracle there)."""
    if overlap_fn is not None:
        return [np.asarray(overlap_fn(b.astype(np.float32), q.astype(np.float32), criterion), np.float32)
                .reshape(b.shape[0], q.shape[0]) for b, q in zip(boxes_list, query_list)]
    nb = [b.shape[0] for b in boxes_list]
    nq = [q.shape[0] for q in query_list]
    box_off, query_off = _offsets(nb), _offsets(nq)
    out_off = _offsets(np.asarray(nb, np.int64) * np.asarray(nq, np.int64), np.int64)
    boxes = np.concatenate(boxes_list, 0).astype(np.float32).reshape(-1, 5)
    query = np.concatenate(query_list, 0).astype(np.float32).reshape(-1, 5)
    flat = _rotated_overlaps_device(boxes, box_off, query, query_off, out_off, criterion)
    return [flat[out_off[f]:out_off[f + 1]].reshape(nb[f], nq[f]) for f in range(len(nb))]


def rotate_iou_gpu_eval(boxes, query_boxes, criterion=-1, device_id=0):
    """Reference signature (rotate_nms_gpu.py:592): [N,5] x [K,5] (x, y, dx, dy, angle) -> [N,K] float32 (the
    reference casts to the dtype of its float32 working copy, so float64 inputs come back as float32 too)."""
    boxes, query_boxes = np.asarray(boxes), np.asarray(query_boxes)
    if boxes.shape[0] == 0 or query_boxes.shape[0] == 0:
        return np.zeros((boxes.shape[0], query_boxes.shape[0]), np.float32)
    return _rotated_overlaps([boxes], [query_boxes], criterion)[0]


def _min(a, b):
    """The reference's min(a, b) (numba's and Python's): b if b < a else a, so a NaN counts only as the first argument."""
    return np.where(b < a, b, a)


def _max(a, b):
    """The reference's max(a, b): b if b > a else a."""
    return np.where(b > a, b, a)


def image_box_overlap(boxes, query_boxes, criterion=-1):
    """Axis-aligned 2-D overlap, kitti_eval.py:95-122, vectorised (same expressions per element, min / max in the
    reference's argument order, which decides what a NaN coordinate gives)."""
    b, q = boxes[:, None, :], query_boxes[None, :, :]
    iw = _min(b[..., 2], q[..., 2]) - _max(b[..., 0], q[..., 0])
    ih = _min(b[..., 3], q[..., 3]) - _max(b[..., 1], q[..., 1])
    area_b = (b[..., 2] - b[..., 0]) * (b[..., 3] - b[..., 1])
    area_q = (q[..., 2] - q[..., 0]) * (q[..., 3] - q[..., 1])
    if criterion == -1:
        ua = area_b + area_q - iw * ih
    elif criterion == 0:
        ua = np.broadcast_to(area_b, iw.shape)      # the other box's area, NaN or not, takes no part
    elif criterion == 1:
        ua = np.broadcast_to(area_q, iw.shape)
    else:
        ua = np.ones_like(iw)
    hit = (iw > 0) & (ih > 0)
    out = np.zeros(iw.shape, dtype=boxes.dtype)
    out[hit] = (iw * ih)[hit] / ua[hit]
    return out


def _d3_from_bev(boxes, qboxes, rinc, criterion=-1):
    """Height overlap on top of the BEV intersection area, camera frame (kitti_eval.py:130-154)."""
    # rinc stays float32 (rotate_iou_gpu_eval returns its float32 working copy's dtype) and the quotient is stored
    # back into it, i.e. rounded to float32, exactly as d3_box_overlap_kernel does
    rinc = np.asarray(rinc, np.float32)
    iw = (_min(boxes[:, None, 1], qboxes[None, :, 1])
          - _max(boxes[:, None, 1] - boxes[:, None, 4], qboxes[None, :, 1] - qboxes[None, :, 4]))
    a1 = (boxes[:, 3] * boxes[:, 4] * boxes[:, 5])[:, None]
    a2 = (qboxes[:, 3] * qboxes[:, 4] * qboxes[:, 5])[None, :]
    inc = iw * rinc
    if criterion == -1:
        ua = a1 + a2 - inc
    elif criterion == 0:
        ua = np.broadcast_to(a1, inc.shape)         # the other box's volume, NaN or not, takes no part
    elif criterion == 1:
        ua = np.broadcast_to(a2, inc.shape)
    else:
        ua = np.ones_like(inc)
    # a pair whose BEV intersection is not > 0 (0 or NaN) keeps it; one whose heights do not overlap gets 0
    out = np.where(rinc > 0, np.float32(0), rinc)
    hit = (rinc > 0) & (iw > 0)
    out[hit] = (inc[hit] / ua[hit]).astype(np.float32)
    return out


def calculate_overlaps(gt_annos, dt_annos, metric, overlap_fn=None):
    """overlaps[f][detection, ground truth] as float64 (what calculate_iou_partly(dt, gt, metric) returns)."""
    return calculate_overlaps_many(gt_annos, [dt_annos], metric, overlap_fn)[0]


def calculate_overlaps_many(gt_annos, dt_sets, metric, overlap_fn=None):
    """calculate_overlaps of each detection set in ``dt_sets`` against the same GT: the rotated overlaps of every
    (set, frame) pair in one kernel launch."""
    if metric == 0:
        gts = [np.asarray(g["bbox"], np.float64).reshape(-1, 4) for g in gt_annos]
        return [[image_box_overlap(np.asarray(d["bbox"], np.float64).reshape(-1, 4), g) for g, d in zip(gts, dts)]
                for dts in dt_sets]

    def cam(a):
        return np.concatenate([np.asarray(a["location"], np.float64).reshape(-1, 3),
                               np.asarray(a["dimensions"], np.float64).reshape(-1, 3),
                               np.asarray(a["rotation_y"], np.float64).reshape(-1, 1)], 1)
    gts = [cam(g) for g in gt_annos]
    dts = [cam(d) for dt_annos in dt_sets for d in dt_annos]
    bev = [0, 2, 3, 5, 6]
    ov = _rotated_overlaps([d[:, bev] for d in dts], [g[:, bev] for g in gts] * len(dt_sets), -1 if metric == 1 else 2,
                           overlap_fn)
    if metric == 1:
        ov = [o.astype(np.float64) for o in ov]
    else:
        ov = [_d3_from_bev(d, g, r).astype(np.float64) for d, g, r in zip(dts, gts * len(dt_sets), ov)]
    n = len(gt_annos)
    return [ov[k * n:(k + 1) * n] for k in range(len(dt_sets))]


# ------------------------------------------------------------------ matching
def clean_data(gt_anno, dt_anno, current_class, difficulty, rng=None):
    """Ignore flags of one frame (kitti_eval.py:39-92): 0 evaluate, 1 ignore, -1 other class."""
    return clean_gt(gt_anno, current_class, difficulty, rng) + (clean_dt(dt_anno, current_class, difficulty, rng),)


def ground_range(anno):
    """Each row's ground distance from the camera: sqrt(x * x + z * z) of its camera-frame location, fp64."""
    loc = np.asarray(anno["location"], np.float64).reshape(-1, 3)
    return np.sqrt(loc[:, 0] * loc[:, 0] + loc[:, 2] * loc[:, 2])


def _in_bin(anno, rng):
    """Rows whose ground range lies in the bin ``rng`` = (lo, hi), lo <= range < hi; a NaN range lies in no bin."""
    r = ground_range(anno)
    return (rng[0] <= r) & (r < rng[1])


def clean_gt(gt_anno, current_class, difficulty, rng=None):
    """clean_data's GT side: (valid GT count, GT ignore flags, DontCare boxes).  ``rng`` = (lo, hi): a GT of the class
    outside that range bin is ignored (1), as one harder than the difficulty is."""
    cls = CLASS_NAMES[current_class].lower()
    names = np.char.lower(np.asarray(gt_anno["name"], dtype=str)) if len(gt_anno["name"]) else np.zeros((0,), str)
    bbox = np.asarray(gt_anno["bbox"], np.float64).reshape(-1, 4)
    valid = np.where(names == cls, 1, -1)
    if cls == "pedestrian":
        valid = np.where(names == "person_sitting", 0, valid)
    elif cls == "car":
        valid = np.where(names == "van", 0, valid)
    ignore = ((np.asarray(gt_anno["occluded"]) > MAX_OCCLUSION[difficulty])
              | (np.asarray(gt_anno["truncated"]) > MAX_TRUNCATION[difficulty])
              | ((bbox[:, 3] - bbox[:, 1]) <= MIN_HEIGHT[difficulty]))
    if rng is not None:
        ignore = ignore | ~_in_bin(gt_anno, rng)
    ign_gt = np.where((valid == 1) & ~ignore, 0, np.where((valid == 0) | (ignore & (valid == 1)), 1, -1)).astype(np.int32)
    dc = bbox[np.asarray(gt_anno["name"], dtype=str) == "DontCare"] if len(names) else np.zeros((0, 4))
    return int((ign_gt == 0).sum()), ign_gt, dc


def clean_dt(dt_anno, current_class, difficulty, rng=None):
    """clean_data's detection side: the detections' ignore flags.  ``rng`` = (lo, hi): a detection of the class
    outside that range bin is ignored (1), as a low one is."""
    cls = CLASS_NAMES[current_class].lower()
    dnames = np.char.lower(np.asarray(dt_anno["name"], dtype=str)) if len(dt_anno["name"]) else np.zeros((0,), str)
    dbox = np.asarray(dt_anno["bbox"], np.float64).reshape(-1, 4)
    height = np.abs(dbox[:, 3] - dbox[:, 1])
    own = 0 if rng is None else np.where(_in_bin(dt_anno, rng), 0, 1)
    return np.where(height < MIN_HEIGHT[difficulty], 1, np.where(dnames == cls, own, -1)).astype(np.int32)


def get_thresholds(scores, num_gt, num_sample_pts=41):
    """Score thresholds at the 41 sampled recall positions (kitti_eval.py:17-36)."""
    scores = np.sort(np.asarray(scores, np.float64))[::-1]
    current_recall, thresholds = 0.0, []
    for i, score in enumerate(scores):
        l_recall = (i + 1) / num_gt
        r_recall = (i + 2) / num_gt if i < len(scores) - 1 else l_recall
        if (r_recall - current_recall) < (current_recall - l_recall) and i < len(scores) - 1:
            continue
        thresholds.append(score)
        current_recall += 1 / (num_sample_pts - 1.0)
    return np.asarray(thresholds, np.float64)


def _cat(xs, shape, dt):
    return np.ascontiguousarray(np.concatenate(xs, 0), dtype=dt) if len(xs) else np.zeros(shape, dt)


class _GtSide:
    """The GT half of sassd_kitti_match's flat arrays for one (class, difficulty): clean_gt of every frame, flattened.
    Every detection set evaluated against the same GT shares it."""

    def __init__(self, gt_annos, current_class, difficulty, rng=None):
        prep = [clean_gt(g, current_class, difficulty, rng) for g in gt_annos]
        self.nframes = len(gt_annos)
        self.total_valid = sum(p[0] for p in prep)
        self.ng = [len(p[1]) for p in prep]
        self.gt_off = _offsets(self.ng)
        self.dc_off = _offsets([p[2].shape[0] for p in prep])
        self.gt_alpha = _cat([np.asarray(g["alpha"], np.float64).reshape(-1) for g in gt_annos], (0,), np.float64)
        self.dc_bbox = _cat([p[2].reshape(-1, 4) for p in prep], (0, 4), np.float64)
        self.ign_gt = _cat([p[1] for p in prep], (0,), np.int32)


class _Packed:
    """Per-(class, difficulty) flat arrays for sassd_kitti_match: a _GtSide and one detection set's half."""

    def __init__(self, gt, dt_annos, overlaps, current_class, difficulty, rng=None):
        ign_dt = [clean_dt(d, current_class, difficulty, rng) for d in dt_annos]
        self.gt = gt
        self.nframes, self.total_valid = gt.nframes, gt.total_valid
        nd = [len(i) for i in ign_dt]
        self.dt_off = _offsets(nd)
        self.ov_off = _offsets(np.asarray(gt.ng, np.int64) * np.asarray(nd, np.int64), np.int64)
        self.overlaps = _cat([np.asarray(o, np.float64).reshape(-1) for o in overlaps], (0,), np.float64)
        self.dt_alpha = _cat([np.asarray(d["alpha"], np.float64).reshape(-1) for d in dt_annos], (0,), np.float64)
        self.dt_score = _cat([np.asarray(d["score"], np.float64).reshape(-1) for d in dt_annos], (0,), np.float64)
        self.dt_bbox = _cat([np.asarray(d["bbox"], np.float64).reshape(-1, 4) for d in dt_annos], (0, 4), np.float64)
        self.ign_dt = _cat(ign_dt, (0,), np.int32)

    def match(self, metric, min_overlap, thresholds=None, compute_aos=False):
        L = _lib.load()
        nth = 0 if thresholds is None else len(thresholds)
        pr = np.zeros((max(nth, 1), 4), np.float64)
        g = self.gt
        tp_scores = np.zeros((max(len(g.gt_alpha), 1),), np.float64)
        ntp = np.zeros((1,), np.int64)
        th = np.ascontiguousarray(thresholds, np.float64) if nth else None
        _lib.check(L.sassd_kitti_match(self.nframes, _p(self.overlaps), _p(self.ov_off), _p(g.gt_off), _p(self.dt_off),
                                       _p(g.dc_off), _p(g.gt_alpha), _p(self.dt_alpha), _p(self.dt_score),
                                       _p(self.dt_bbox), _p(g.dc_bbox), _p(g.ign_gt), _p(self.ign_dt), int(metric),
                                       float(min_overlap), int(bool(compute_aos)), nth, _p(th), _p(pr), _p(tp_scores),
                                       _p(ntp)), "sassd_kitti_match")
        return pr[:nth], tp_scores[:int(ntp[0])]

    def assign(self, metric, min_overlap):
        """The match table's columns of this (class, difficulty) at one metric (sassd_kitti_assign): per GT row the
        matched detection's row or -1 and their overlap, per detection row its lib.KITTI_DT_* state."""
        g = self.gt
        gt_det = np.zeros((len(g.ign_gt),), np.int32)
        gt_ov = np.zeros((len(g.ign_gt),), np.float64)
        state = np.zeros((len(self.ign_dt),), np.int8)
        _lib.check(_lib.load().sassd_kitti_assign(self.nframes, _p(self.overlaps), _p(self.ov_off), _p(g.gt_off),
                                                  _p(self.dt_off), _p(g.dc_off), _p(self.dt_score), _p(self.dt_bbox),
                                                  _p(g.dc_bbox), _p(g.ign_gt), _p(self.ign_dt), int(metric),
                                                  float(min_overlap), _p(gt_det), _p(gt_ov), _p(state)),
                   "sassd_kitti_assign")
        return gt_det, gt_ov, state


def eval_class(gt_annos, dt_annos, current_classes, difficultys, metric, min_overlaps, compute_aos=False,
               overlap_fn=None):
    """precision / recall / orientation [class, difficulty, min_overlap, 41] (eval_class_v3, kitti_eval.py:549-657).
    min_overlaps: [num_minoverlap, metric, class]."""
    return eval_class_many(gt_annos, [dt_annos], current_classes, difficultys, metric, min_overlaps, [compute_aos],
                           overlap_fn)[0]


def eval_class_many(gt_annos, dt_sets, current_classes, difficultys, metric, min_overlaps, compute_aos, overlap_fn=None,
                    gt_sides=None, bins=None):
    """eval_class for each detection set of ``dt_sets`` against the same GT (``compute_aos``: one flag per set): one
    overlap pass for all sets (calculate_overlaps_many) and one GT side per class and difficulty entry (``gt_sides``:
    {(class, difficulty, bin): _GtSide}, built here when not given).  ``bins``: a range bin (lo, hi) or None per entry
    of ``difficultys`` (clean_gt / clean_dt's ``rng``); None: no bins."""
    assert all(len(gt_annos) == len(d) for d in dt_sets)
    bins = [None] * len(difficultys) if bins is None else list(bins)
    overlaps = calculate_overlaps_many(gt_annos, dt_sets, metric, overlap_fn)
    shape = (len(current_classes), len(difficultys), len(min_overlaps), 41)
    out = [dict(recall=np.zeros(shape), precision=np.zeros(shape), orientation=np.zeros(shape)) for _ in dt_sets]
    for m, cls in enumerate(current_classes):
        for l, (diff, rng) in enumerate(zip(difficultys, bins)):
            gt = _GtSide(gt_annos, cls, diff, rng) if gt_sides is None else gt_sides[cls, diff, rng]
            for dt_annos, ov, aos_s, res in zip(dt_sets, overlaps, compute_aos, out):
                packed = _Packed(gt, dt_annos, ov, cls, diff, rng)
                recall, precision, aos = res["recall"], res["precision"], res["orientation"]
                for k, min_overlap in enumerate(min_overlaps[:, metric, m]):
                    _, tp_scores = packed.match(metric, min_overlap)
                    thresholds = get_thresholds(tp_scores, packed.total_valid)
                    pr, _ = packed.match(metric, min_overlap, thresholds, aos_s)
                    n = len(thresholds)
                    with np.errstate(divide="ignore", invalid="ignore"):
                        recall[m, l, k, :n] = pr[:, 0] / (pr[:, 0] + pr[:, 2])
                        precision[m, l, k, :n] = pr[:, 0] / (pr[:, 0] + pr[:, 1])
                        if aos_s:
                            aos[m, l, k, :n] = pr[:, 3] / (pr[:, 0] + pr[:, 1])
                    for i in range(n):      # monotone envelope over the sampled points (:645-651)
                        precision[m, l, k, i] = np.max(precision[m, l, k, i:])
                        recall[m, l, k, i] = np.max(recall[m, l, k, i:])
                        if aos_s:
                            aos[m, l, k, i] = np.max(aos[m, l, k, i:])
    return out


# ------------------------------------------------------------------ device path
_NAME_IDS = {n: i for i, n in enumerate(dict.fromkeys(CLASS_NAMES))}     # one id per distinct lower-cased class name
_IGNORED_NAME = {"car": "van", "pedestrian": "person_sitting"}           # counted as ignored, not missed (clean_data)


_ID_NAMES = list(_NAME_IDS)


def _flat_names(annos):
    """(name ids, DontCare flags) of every row of ``annos``, frames concatenated; names are mapped once per distinct
    name."""
    names = [np.asarray(a["name"], dtype=str).reshape(-1) for a in annos]
    names = np.concatenate(names) if names else np.zeros((0,), str)
    if not len(names):
        return np.zeros((0,), np.int32), np.zeros((0,), np.int32)
    uniq, inv = np.unique(names, return_inverse=True)
    ids = np.array([_NAME_IDS.get(str(u).lower(), -1) for u in uniq], np.int32)
    return ids[inv.reshape(-1)], (uniq == "DontCare").astype(np.int32)[inv.reshape(-1)]


def _flat(annos, key, width):
    return _cat([np.asarray(a[key], np.float64).reshape(-1, width) for a in annos], (0, width), np.float64)


def _flat_cam(annos):
    return np.concatenate([_flat(annos, "location", 3), _flat(annos, "dimensions", 3), _flat(annos, "rotation_y", 1)], 1)


def _cuda_device():
    import torch
    from . import ops
    ops.require_cuda()
    return torch.device("cuda", torch.cuda.current_device())


class AnnoBlock:
    """The annotations of a list of frames as the flat columns the device evaluator reads: ``off`` [frames + 1] int64
    row offsets (host), and torch tensors on one device, a row per object: ``name_id`` int32 (the index of the
    lower-cased name among the class names, -1 for any other name), ``dontcare`` int32 (name == "DontCare"),
    ``truncated``, ``occluded``, ``alpha`` and ``score`` float64, ``bbox`` [rows, 4] float64 and ``cam`` [rows, 7]
    float64 (location, dimensions l, h, w, rotation_y).  ``trunc_dtype`` is the dtype the truncation values came in:
    numpy compares a float32 column with the Python-float limit in float32, so the evaluator rounds the limit into it.

    Built from annotation dicts (``from_annos``) or parsed from a directory of KITTI files on the device
    (``read_block``)."""
    COLUMNS = ("name_id", "dontcare", "truncated", "occluded", "alpha", "bbox", "cam", "score")

    def __init__(self, off, columns, trunc_dtype=np.float64):
        self.off = np.asarray(off, np.int64)
        for name in self.COLUMNS:
            setattr(self, name, columns[name])
        self.trunc_dtype = np.dtype(trunc_dtype)

    def __len__(self):
        return len(self.off) - 1

    @property
    def counts(self):
        return np.diff(self.off)

    @classmethod
    def from_annos(cls, annos, device=None):
        """The block of a list of annotation dicts (``device``: default the current CUDA device).  A dict without
        ``score`` (ground truth) gets zeros."""
        import torch
        device = _cuda_device() if device is None else torch.device(device)
        names, dc = _flat_names(annos)
        truncs = [np.asarray(a["truncated"]).reshape(-1) for a in annos]
        trunc = np.concatenate(truncs) if truncs else np.zeros((0,))
        scores = [np.asarray(a["score"], np.float64).reshape(-1) if "score" in a else np.zeros((len(a["name"]),))
                  for a in annos]
        cols = dict(name_id=names, dontcare=dc, truncated=trunc.astype(np.float64),
                    occluded=_flat(annos, "occluded", 1).reshape(-1), alpha=_flat(annos, "alpha", 1).reshape(-1),
                    bbox=_flat(annos, "bbox", 4), cam=_flat_cam(annos), score=_cat(scores, (0,), np.float64))
        cols = {k: torch.from_numpy(np.ascontiguousarray(v)).to(device) for k, v in cols.items()}
        return cls(_offsets([len(a["name"]) for a in annos], np.int64), cols,
                   trunc.dtype if trunc.dtype.kind == "f" else np.float64)

    def to(self, device):
        return AnnoBlock(self.off, {k: getattr(self, k).to(device) for k in self.COLUMNS}, self.trunc_dtype)

    def to_annos(self):
        """Per-frame annotation dicts for the host path: the columns, ``truncated`` in ``trunc_dtype``, and a name per
        row that the evaluator treats as the original (the class's lower-cased name, "DontCare", or "" for any other
        name)."""
        c = {k: getattr(self, k).cpu().numpy() for k in self.COLUMNS}
        names = np.array([""] + _ID_NAMES + ["DontCare"])[np.where(c["dontcare"] != 0, len(_ID_NAMES) + 1,
                                                                    c["name_id"] + 1)]
        out = []
        for f in range(len(self)):
            r = slice(self.off[f], self.off[f + 1])
            out.append(dict(name=names[r], truncated=c["truncated"][r].astype(self.trunc_dtype),
                            occluded=c["occluded"][r], alpha=c["alpha"][r], bbox=c["bbox"][r],
                            location=c["cam"][r, :3], dimensions=c["cam"][r, 3:6], rotation_y=c["cam"][r, 6],
                            score=c["score"][r]))
        return out


def _as_block(annos):
    return annos if isinstance(annos, AnnoBlock) else AnnoBlock.from_annos(annos)


def _as_annos(annos):
    return annos.to_annos() if isinstance(annos, AnnoBlock) else annos


def read_block(directory, ids, device=None, workers=8, times=None):
    """``directory/%06d.txt`` of every id (KITTI label or result files, a 16th field the score) -> an AnnoBlock, what
    ``AnnoBlock.from_annos(kitti_data.read_labels(directory, ids))`` gives, bit for bit.  The files are read on a
    thread pool into one pinned buffer, copied to the device once and parsed there (csrc/kitti_parse.cu); a file
    outside the device's grammar is read by kitti_data.read_label instead, and so raises what it raises.  A missing
    file raises FileNotFoundError naming it.  ``times``: a dict whose "read" and "parse" entries accumulate the seconds
    spent reading the files and parsing them (the device synchronised)."""
    from concurrent.futures import ThreadPoolExecutor

    import torch
    from . import lib, ops
    from .kitti_data import read_label
    t0 = time.perf_counter()
    paths = [os.path.join(directory, "%06d.txt" % i) for i in ids]

    def load(path):
        with open(path, "rb") as fh:
            return fh.read()
    with ThreadPoolExecutor(max_workers=max(1, int(workers))) as ex:
        data = list(ex.map(load, paths))
    device = _cuda_device() if device is None else torch.device(device)
    file_off = _offsets([len(d) for d in data], np.int64)
    host = torch.empty((max(int(file_off[-1]), 1),), dtype=torch.uint8, pin_memory=True)
    host.numpy()[:file_off[-1]] = np.frombuffer(b"".join(data), np.uint8)
    t1 = time.perf_counter()
    buf = host.to(device, non_blocking=True)
    d_file_off = torch.from_numpy(file_off).to(device)
    n_lines, flags = ops.kitti_scan_labels(buf, d_file_off)
    n_lines, flags = torch.stack([n_lines, flags]).cpu().numpy() if len(ids) else np.zeros((2, 0), np.int32)
    deferred = np.flatnonzero(flags & lib.KITTI_PARSE_DEFER)
    slow = AnnoBlock.from_annos([read_label(paths[f]) for f in deferred], "cpu")
    counts = n_lines.astype(np.int64)
    counts[deferred] = slow.counts
    row_off = _offsets(counts)
    nrows = int(row_off[-1])
    names = "".join(_ID_NAMES).encode()
    name_off = _offsets([len(n) for n in _ID_NAMES])
    cols = ops.kitti_parse_labels(buf, d_file_off, torch.from_numpy(flags).to(device), torch.from_numpy(row_off).to(device),
                                  nrows, torch.frombuffer(bytearray(names), dtype=torch.uint8).to(device),
                                  torch.from_numpy(name_off).to(device))
    cols = dict(zip(AnnoBlock.COLUMNS, cols))
    if len(deferred):
        rows = np.concatenate([np.arange(row_off[f], row_off[f + 1]) for f in deferred])
        idx = torch.from_numpy(rows).to(device)
        for k in AnnoBlock.COLUMNS:
            cols[k][idx] = getattr(slow, k).to(device)
    block = AnnoBlock(row_off.astype(np.int64), cols)
    if times is not None:
        torch.cuda.synchronize(device)
        t2 = time.perf_counter()
        times["read"] = times.get("read", 0.0) + t1 - t0
        times["parse"] = times.get("parse", 0.0) + t2 - t1
    return block


def _eval_device(gt_annos, dt_sets, classes, difficultys, min_overlaps, aos_flags):
    """eval_class_many's precision / recall / orientation arrays for the three metrics, [metric][set] ->
    dict of [class, difficulty, min_overlap, 41], with the flags, overlaps, matching, thresholds and per-threshold sums
    on the device (csrc/kitti_match.cu); bit for bit what the host path computes.  The GT and each detection set are
    AnnoBlocks (lists of annotation dicts are flattened into one first)."""
    return _eval_device_full(gt_annos, dt_sets, classes, difficultys, min_overlaps, aos_flags)[0]


def _eval_device_full(gt_annos, dt_sets, classes, difficultys, min_overlaps, aos_flags, bins=None, assign=None,
                      ap=True):
    """_eval_device with a range bin (lo, hi) or None per difficulty entry (``bins``), and with ``assign`` = (row,
    ndiff) also the match table of the first ndiff entries at min-overlap row ``row`` (match_table's dicts, one per
    set), from the flags and overlaps already on the device.  ``ap`` False skips the AP matching (the arrays are then
    None).  Returns (arrays, tables)."""
    st = _device_setup(gt_annos, dt_sets, classes, difficultys, min_overlaps, aos_flags, bins, assign is not None)
    return _device_arrays(st, assign, ap)


def _device_setup(gt_annos, dt_sets, classes, difficultys, min_overlaps, aos_flags, bins=None, ranged_out=False,
                  aos_table=False):
    """What every device evaluation of these sets starts from, built once: the blocks on the device, the flags, the
    rotated and metric overlaps, the AOS cos table (when a set computes AOS, or ``aos_table``) and the matching
    descriptor.  ``ranged_out``: also each row's ground range.  Returns a namespace."""
    import types

    import torch
    from . import ops
    dev = _cuda_device()
    gt = _as_block(gt_annos).to(dev)
    dts = [_as_block(d).to(dev) for d in dt_sets]
    K, F, C, Dn, M = len(dts), len(gt), len(classes), len(difficultys), min_overlaps.shape[0]
    assert all(len(d) == F for d in dts)
    ng = gt.counts
    nd = np.concatenate([d.counts for d in dts]) if dts else np.zeros((0,), np.int64)
    npairs = nd * np.tile(ng, K)
    gt_off, dt_off, ov_off = _offsets(ng), _offsets(nd), _offsets(npairs, np.int64)
    total = int(ov_off[-1])
    dt_name = torch.cat([d.name_id for d in dts])
    dt_bbox, dt_cam = torch.cat([d.bbox for d in dts]), torch.cat([d.cam for d in dts])
    # numpy compares a float32 column with the Python-float limit in float32: round the limit into the column's dtype
    limits = np.array([[MAX_OCCLUSION[d], float(gt.trunc_dtype.type(MAX_TRUNCATION[d])), MIN_HEIGHT[d]]
                       for d in difficultys], np.float64)
    cls_ids = np.array([[_NAME_IDS[CLASS_NAMES[c].lower()], _NAME_IDS.get(_IGNORED_NAME.get(CLASS_NAMES[c].lower()), -1)]
                        for c in classes], np.int32)

    def up(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(dev)

    t = dict(gt_off=up(gt_off), dt_off=up(dt_off), ov_off=up(ov_off), gt_dc=gt.dontcare, gt_bbox=gt.bbox,
             dt_bbox=dt_bbox, dt_score=torch.cat([d.score for d in dts]), gt_cam=gt.cam, dt_cam=dt_cam,
             min_overlaps=up(np.asarray(min_overlaps, np.float64)), compute_aos=up(np.asarray(aos_flags, np.int32)))
    ranged = bins is not None and any(b is not None for b in bins)
    gt_range = dt_range = None
    if ranged or ranged_out:
        # an entry without a bin has a lower edge of -inf: no range test
        ranges = up(np.array([(-np.inf, np.inf) if b is None else b for b in bins], np.float64)) if ranged else None
        ign_gt, ign_dt, n_valid, gt_range, dt_range = ops.kitti_eval_flags_ranged(
            gt.name_id, gt.occluded, gt.truncated, t["gt_bbox"], gt.cam, dt_name, t["dt_bbox"], dt_cam, up(cls_ids),
            up(limits), ranges)
    else:
        ign_gt, ign_dt, n_valid = ops.kitti_eval_flags(gt.name_id, gt.occluded, gt.truncated, t["gt_bbox"], dt_name,
                                                       t["dt_bbox"], up(cls_ids), up(limits))
    # the rotated overlaps of every (set, frame) block: BEV IoU and the intersection area the 3-D overlap builds on
    bev = [0, 2, 3, 5, 6]
    dt_bev, gt_bev = dt_cam[:, bev].float().contiguous(), gt.cam[:, bev].float().repeat(K, 1)
    q_off = up(_offsets(np.tile(ng, K)))
    rot = []
    for criterion in (-1, 2):
        out = torch.zeros((max(total, 1),), dtype=torch.float32, device=dev)
        if total:
            ops._call("sassd_rotate_overlap_eval", None, ops._ptr(dt_bev), ops._ptr(t["dt_off"]), ops._ptr(gt_bev),
                      ops._ptr(q_off), ops._ptr(t["ov_off"]), K * F, criterion, int(npairs.max()), ops._ptr(out),
                      ops._stream())
        rot.append(out)
    ov = ops.kitti_eval_overlaps(K, F, t["gt_off"], t["dt_off"], t["ov_off"], t["gt_cam"], t["dt_cam"], t["gt_bbox"],
                                 t["dt_bbox"], rot[0], rot[1], total, int(npairs.max()) if len(npairs) else 0)
    aos_tab = None
    if (any(aos_flags) or aos_table) and total:
        table = np.zeros((total,), np.float64)
        gt_alpha = gt.alpha.cpu().numpy()
        dt_alpha = torch.cat([d.alpha for d in dts]).cpu().numpy()
        _lib.check(_lib.load().sassd_kitti_aos_table(K, F, _p(gt_off), _p(dt_off), _p(ov_off), _p(gt_alpha),
                                                     _p(dt_alpha), _p(table)), "sassd_kitti_aos_table")
        aos_tab = up(table)
    # each job's score region: the next power of two of its (class, difficulty)'s valid GT count
    nv = n_valid.cpu().numpy().astype(np.int64)
    region = np.broadcast_to((1 << np.ceil(np.log2(np.maximum(nv, 1))).astype(np.int64))[None, :, :, None, None],
                             (K, C, Dn, 3, M)).reshape(-1)
    score_off = up(_offsets(region, np.int64))
    desc = _lib.KittiEvalDesc(nsets=K, nframes=F, nclass=C, ndiff=Dn, nover=M, max_nd=int(nd.max()) if len(nd) else 0,
                              max_ng=int(ng.max()) if len(ng) else 0)
    keep = dict(t, ign_gt=ign_gt, ign_dt=ign_dt, n_valid=n_valid, score_off=score_off, ov_bbox=ov[0], ov_bev=ov[1],
                ov_3d=ov[2], aos_table=aos_tab)
    for name, _ in desc._fields_[7:]:
        setattr(desc, name, keep[name].data_ptr() if keep[name] is not None else None)
    return types.SimpleNamespace(gt=gt, dts=dts, K=K, F=F, C=C, Dn=Dn, M=M, ng=ng, nd=nd, region=region, desc=desc,
                                 keep=keep, dt_cam=dt_cam, gt_range=gt_range, dt_range=dt_range, aos_flags=aos_flags,
                                 up=up)


def _device_arrays(st, assign, ap):
    """_eval_device_full's arrays and match tables from a _device_setup."""
    from . import ops
    K, C, Dn, M, gt, dts = st.K, st.C, st.Dn, st.M, st.gt, st.dts
    tables = None
    if assign is not None:
        row, nd_t = assign
        gt_det, gt_ov, dt_state, tp_err = (x.cpu().numpy() for x in ops.kitti_eval_assign(st.desc, row, nd_t, gt.cam,
                                                                                            st.dt_cam))
        gt_flag, dt_flag = st.keep["ign_gt"][:, :nd_t].cpu().numpy(), st.keep["ign_dt"][:, :nd_t].cpu().numpy()
        gt_range, dt_range = st.gt_range.cpu().numpy(), st.dt_range.cpu().numpy()
        rows = _offsets([int(d.off[-1]) for d in dts], np.int64)
        tables = []
        for k in range(K):
            r = slice(rows[k], rows[k + 1])
            tables.append(dict(gt_off=gt.off.copy(), dt_off=dts[k].off.copy(), gt_range=gt_range, dt_range=dt_range[r],
                               gt_flag=gt_flag, dt_flag=np.ascontiguousarray(dt_flag[..., r]), gt_det=gt_det[k],
                               gt_overlap=gt_ov[k], dt_state=np.ascontiguousarray(dt_state[..., r]),
                               tp_errors=tp_err[k]))
    if not ap:
        return None, tables
    _, n_thresh, pr = ops.kitti_eval_match(st.desc, len(st.region), int(st.region.sum()))
    n_thresh = n_thresh.cpu().numpy().reshape(K, C, Dn, 3, M)
    pr = pr.cpu().numpy().reshape(K, C, Dn, 3, M, 41, 4)
    return _pr_arrays(pr, n_thresh, np.asarray(st.aos_flags, bool)), tables


def _pr_arrays(pr, n_thresh, aos_flags):
    """precision, recall and AOS of the sampled thresholds and their monotone envelope, as eval_class_many computes
    them, from the per-threshold sums pr [..., K, C, Dn, 3, M, 41, 4] and threshold counts n_thresh [..., K, C, Dn, 3,
    M]; ``aos_flags`` [..., K] bool.  Returns [metric][set] -> dict of [..., C, Dn, M, 41]."""
    past = np.arange(41) >= n_thresh[..., None]
    with np.errstate(divide="ignore", invalid="ignore"):
        recall = pr[..., 0] / (pr[..., 0] + pr[..., 2])
        precision = pr[..., 0] / (pr[..., 0] + pr[..., 1])
        aos = pr[..., 3] / (pr[..., 0] + pr[..., 1])
    K = pr.shape[-7]
    out = []
    for m in range(3):
        per_set = []
        for k in range(K):
            res = {}
            for key, a in (("recall", recall), ("precision", precision), ("orientation", aos)):
                v = np.where(past[..., k, :, :, m, :, :], 0.0, a[..., k, :, :, m, :, :])
                if key == "orientation":
                    on = aos_flags[..., k] & (m == 0)
                    v = np.where(np.reshape(on, np.shape(on) + (1,) * 4), v, 0.0)
                res[key] = np.ascontiguousarray(np.maximum.accumulate(v[..., ::-1], axis=-1)[..., ::-1])
            per_set.append(res)
        out.append(per_set)
    return out


def get_mAP(prec):
    """11-point interpolated AP over the 41 samples (get_mAP_v2, kitti_eval.py:683-688)."""
    return sum(prec[..., i] for i in range(0, prec.shape[-1], 4)) / 11 * 100


def get_mAP_R40(prec):
    """AP at 40 recall positions over the same 41 samples: recall 1/40 ... 1, recall 0 dropped (the KITTI benchmark's
    AP since 2019, which the reference's readme quotes)."""
    return sum(prec[..., i] for i in range(1, prec.shape[-1])) / 40 * 100


def official_eval(gt_annos, dt_annos, current_classes, difficultys=(0, 1, 2), overlap_fn=None, recall_positions=11):
    """-> (text, dict(bbox, bev, d3, aos) of AP arrays [class, difficulty, min_overlap]).  ``recall_positions``: 11
    (get_mAP, the reference's table) or 40 (get_mAP_R40; the text's headings then read AP_R40)."""
    if recall_positions not in (11, 40):
        raise ValueError("recall_positions must be 11 or 40, not %r" % (recall_positions,))
    return official_eval_many(gt_annos, [dt_annos], current_classes, (recall_positions,), overlap_fn,
                              difficultys)[0][recall_positions]


def official_eval_many(gt_annos, dt_sets, classes, recall_positions=(11, 40), overlap_fn=None, difficultys=(0, 1, 2)):
    """official_eval of K detection sets (each a list of per-frame annotation dicts, e.g. one per checkpoint) against
    the same GT, at each of ``recall_positions`` (11 and / or 40).  Returns one dict per set, {recall positions:
    official_eval's (text, ap)}.  One evaluation (eval_many) serves every set and both recall positions."""
    positions = tuple(recall_positions)
    if not positions or any(r not in (11, 40) for r in positions):
        raise ValueError("recall_positions must be 11 or 40, not %r" % (recall_positions,))
    return eval_many(gt_annos, dt_sets, classes, positions, overlap_fn, difficultys)


def coco_min_overlaps(classes):
    """[10, metric, class]: the host's np.linspace(start, stop, 10) of each class's COCO range, for all three metrics
    (do_coco_style_eval, kitti_eval.py:713-717, with the integer ``num`` NumPy requires)."""
    out = np.zeros((10, 3, len(classes)))
    for j, c in enumerate(classes):
        start, stop, num = COCO_RANGE[c]
        out[:, :, j] = np.linspace(start, stop, int(num))[:, None]
    return out


def _class_ids(classes):
    current = classes if isinstance(classes, (list, tuple)) else [classes]
    name_to_class = {v: k for k, v in CLASS_TO_NAME.items()}
    return [name_to_class[c] if isinstance(c, str) else c for c in current]


def _aos_flag(dt_annos):
    """compute_aos as the reference decides it (kitti_eval.py:818-823): from the first frame with detections."""
    if isinstance(dt_annos, AnnoBlock):
        return bool(dt_annos.off[-1] > 0 and float(dt_annos.alpha[0]) != -10)
    for anno in dt_annos:
        if anno['alpha'].shape[0] != 0:
            return bool(anno['alpha'][0] != -10)
    return False


def check_ranges(ranges):
    """The range bin edges e0 < e1 < ... as a tuple of floats: at least two, non-negative and strictly increasing (the
    last may be inf); anything else is a ValueError."""
    try:
        edges = np.asarray(ranges, np.float64).reshape(-1)
    except (TypeError, ValueError):
        raise ValueError("ranges must be numbers, not %r" % (ranges,)) from None
    with np.errstate(invalid="ignore"):
        bad = len(edges) < 2 or not np.all(edges >= 0) or not np.all(np.diff(edges) > 0)
    if bad:
        raise ValueError("ranges must be two or more non-negative, strictly increasing edges, not %r" % (ranges,))
    return tuple(float(e) for e in edges)


def range_bins(edges):
    """The half-open bins [e_i, e_i+1) of the edges."""
    return list(zip(edges[:-1], edges[1:]))


def eval_many(gt_annos, dt_sets, classes, tables=(11,), overlap_fn=None, difficultys=(0, 1, 2), ranges=None,
              match=False, bootstrap=None):
    """Every table of ``tables`` (11 and 40: the official tables at 11 / 40 recall positions; "coco": the COCO-style
    table) for each of the K detection sets of ``dt_sets`` against the same GT.  Returns one dict per set, {table:
    (text, ap)}.  The official and COCO overlap rows form one list of min overlaps, so the overlaps, the GT side and
    the matching run once for all of them; R11 and R40 read the same precision samples.  The GT and each set are a
    list of annotation dicts or an AnnoBlock.

    ``ranges``: bin edges (check_ranges); each set's dict then also holds ``"ranges"``: [(lo, hi, {table: (text,
    ap)}), ...], the tables over the objects whose ground range (ground_range) lies in [lo, hi), each text naming its
    range.  The bins are more difficulty entries of the same evaluation: a GT or detection of the class outside a bin is
    ignored there (clean_gt / clean_dt).  ``match``: each set's dict also holds ``"matches"``, its match_table.

    ``bootstrap``: an int array [R, F] of frame indices (bootstrap_indices), replicate r the list of frames idx[r, 0],
    idx[r, 1], ... (duplicates included), or a ReplicateLists of lists of any length (bootstrap_groups: drive-level
    replicates; or each drive's own frames, for per-drive AP).  Each set's dict then also holds ``"bootstrap"``:
    {table: ap} with a leading R axis on every array, replicate r's AP bit for bit what this evaluation gives on the
    resampled GT and detection lists (compute_aos decided per replicate; ``aos`` is NaN in a replicate without it, None
    when no replicate has it); with ``ranges`` also ``"bootstrap_ranges"``, laid out like ``"ranges"``.  Every set uses
    the same lists, so the replicates are paired (paired_summary)."""
    tables = tuple(tables)
    if not tables or any(t not in TABLES for t in tables):
        raise ValueError("tables must be among %r, not %r" % (TABLES, tables))
    return _evaluate(gt_annos, dt_sets, classes, tables, overlap_fn, difficultys, ranges, match, bootstrap)


def match_table(gt_annos, dt_sets, classes, difficultys=(0, 1, 2), overlap_fn=None):
    """compute_statistics_jit's whole-range assignment (kitti_eval.py:164-283, compute_fp=True at a threshold below
    every score, each class's first official min overlap) of each detection set, for every class, difficulty and metric
    (bbox, BEV, 3-D).  One dict per set of numpy arrays, with G GT rows and D_k detection rows (frames concatenated):

    * ``gt_off`` / ``dt_off`` [frames + 1]: each frame's first row;
    * ``gt_range`` [G] / ``dt_range`` [D_k]: each row's ground range;
    * ``gt_flag`` [C, Dn, G] / ``dt_flag`` [C, Dn, D_k]: clean_data's flags;
    * ``gt_det`` [C, Dn, 3, G]: the matched detection row or -1; ``gt_overlap`` [C, Dn, 3, G] their overlap (0 when
      unmatched);
    * ``dt_state`` [C, Dn, 3, D_k]: lib.KITTI_DT_TP, _FP, _DONTCARE (in a DontCare area, bbox metric only), _IGNORED
      (assigned to an ignored GT or through an ignored detection) or _NOT_COUNTED (flag -1 or 1);
    * ``tp_errors`` [C, Dn, G, 3]: the 3-D metric's true positives' ATE, ASE, AOE (tp_errors) on their GT rows, NaN
      elsewhere.

    On the device this is one kernel over the flags and overlaps of the evaluation (csrc/kitti_match.cu); with
    ``overlap_fn`` the host matcher records the same assignment."""
    return [r["matches"] for r in _evaluate(gt_annos, dt_sets, classes, (), overlap_fn, difficultys, None, True)]


def tp_errors(gt_cam, dt_cam):
    """[n, 3] (ATE, ASE, AOE) of camera rows (x, y, z, l, h, w, ry) of GTs against their detections': ATE the BEV
    centre distance in camera x-z, ASE 1 - vi / (vg + vd - vi) with vi = min(l) * min(h) * min(w), AOE |ry_d - ry_g|
    wrapped to [0, pi].  fp64, in the device kernel's operation order."""
    g, q = np.asarray(gt_cam, np.float64).reshape(-1, 7), np.asarray(dt_cam, np.float64).reshape(-1, 7)
    dx, dz = q[:, 0] - g[:, 0], q[:, 2] - g[:, 2]
    vi = np.fmin(q[:, 3], g[:, 3]) * np.fmin(q[:, 4], g[:, 4]) * np.fmin(q[:, 5], g[:, 5])
    vg, vd = g[:, 3] * g[:, 4] * g[:, 5], q[:, 3] * q[:, 4] * q[:, 5]
    d = q[:, 6] - g[:, 6]
    aoe = np.fmin(np.abs(d - 2 * np.pi * np.floor((d + np.pi) / (2 * np.pi))), np.pi)
    return np.stack([np.sqrt(dx * dx + dz * dz), 1.0 - vi / (vg + vd - vi), aoe], 1)


def _table_host(gt_annos, dt_sets, classes, difficultys, row, overlap_fn, gt_sides):
    """match_table on the host path: the host matcher's recorded assignment per (class, difficulty, metric)."""
    ovs = [calculate_overlaps_many(gt_annos, dt_sets, m, overlap_fn) for m in range(3)]
    gt_cam = _flat_cam(gt_annos)
    gt_range = _cat([ground_range(g) for g in gt_annos], (0,), np.float64)
    C, Dn, G = len(classes), len(difficultys), len(gt_range)
    gt_flag = np.zeros((C, Dn, G), np.int8)
    out = []
    for k, dts in enumerate(dt_sets):
        dt_cam = _flat_cam(dts)
        D = dt_cam.shape[0]
        t = dict(gt_off=_offsets([len(g["name"]) for g in gt_annos], np.int64),
                 dt_off=_offsets([len(d["name"]) for d in dts], np.int64), gt_range=gt_range,
                 dt_range=_cat([ground_range(d) for d in dts], (0,), np.float64), gt_flag=gt_flag,
                 dt_flag=np.zeros((C, Dn, D), np.int8), gt_det=np.zeros((C, Dn, 3, G), np.int32),
                 gt_overlap=np.zeros((C, Dn, 3, G)), dt_state=np.zeros((C, Dn, 3, D), np.int8),
                 tp_errors=np.full((C, Dn, G, 3), np.nan))
        for ci, c in enumerate(classes):
            for di, d in enumerate(difficultys):
                side = gt_sides[c, d, None]
                gt_flag[ci, di] = side.ign_gt
                for m in range(3):
                    packed = _Packed(side, dts, ovs[m][k], c, d)
                    t["gt_det"][ci, di, m], t["gt_overlap"][ci, di, m], t["dt_state"][ci, di, m] = packed.assign(
                        m, row[m, ci])
                t["dt_flag"][ci, di] = packed.ign_dt
                j = t["gt_det"][ci, di, 2]
                tp = np.flatnonzero(j >= 0)
                tp = tp[t["dt_state"][ci, di, 2][j[tp]] == _lib.KITTI_DT_TP]
                t["tp_errors"][ci, di, tp] = tp_errors(gt_cam[tp], dt_cam[j[tp]])
        out.append(t)
    return out


def _evaluate(gt_annos, dt_sets, classes, tables, overlap_fn, difficultys, ranges, match, bootstrap=None):
    """eval_many's work: the AP tables of ``tables`` (none: no AP matching) over the whole range and each bin of
    ``ranges``, with ``match`` the match table, and with ``bootstrap`` the replicates' AP."""
    classes = _class_ids(classes)
    edges = None if ranges is None else check_ranges(ranges)
    lists = None if bootstrap is None else check_bootstrap(bootstrap, len(gt_annos))
    diffs = list(difficultys)
    bins = [None] + ([] if edges is None else range_bins(edges))
    entries = [(d, b) for b in bins for d in diffs]     # difficulty entries: the whole range, then bin by bin
    official = any(t in (11, 40) for t in tables)
    rows = ([np.stack([OVERLAP_0_7, OVERLAP_0_5], axis=0)[:, :, classes]] if official else [])
    if "coco" in tables:
        rows.append(coco_min_overlaps(classes))
    table_row = 0
    if match and not official:          # the match table is at each class's first official min overlap
        table_row = sum(r.shape[0] for r in rows)
        rows.append(OVERLAP_0_7[None][:, :, classes])
    min_overlaps = np.concatenate(rows, 0)
    n_off = 2 if official else 0
    aos_flags = [_aos_flag(d) for d in dt_sets]
    ent_diffs, ent_bins = [d for d, _ in entries], [b for _, b in entries]
    Dn = len(diffs)
    boot = None
    if overlap_fn is None:
        boot_aos = None
        if lists is not None:
            dt_sets = [_as_block(d) for d in dt_sets]
            boot_aos = _bootstrap_aos_flags(dt_sets, lists)
        st = _device_setup(gt_annos, dt_sets, classes, ent_diffs, min_overlaps, aos_flags, ent_bins, match,
                           boot_aos is not None and bool(boot_aos.any()))
        prec, matches = _device_arrays(st, (table_row, Dn) if match else None, bool(tables))
        if lists is not None:
            boot = _bootstrap_device(st, lists, boot_aos, tables, Dn, len(bins), n_off)
    else:
        gt_annos, dt_sets = _as_annos(gt_annos), [_as_annos(d) for d in dt_sets]
        gt_sides = {(c, d, b): _GtSide(gt_annos, c, d, b) for c in classes for d, b in entries}
        prec = [eval_class_many(gt_annos, dt_sets, classes, ent_diffs, metric, min_overlaps,
                                aos_flags if metric == 0 else [False] * len(dt_sets), overlap_fn, gt_sides, ent_bins)
                for metric in (0, 1, 2)] if tables else None
        matches = (_table_host(gt_annos, dt_sets, classes, diffs, min_overlaps[table_row], overlap_fn, gt_sides)
                   if match else None)
        if lists is not None:
            boot = _bootstrap_host(gt_annos, dt_sets, classes, tables, overlap_fn, difficultys, edges, lists)
    out = []
    for s, compute_aos in enumerate(aos_flags):
        res = {}
        if tables:
            r = [p[s] for p in prec]
            res = _ap_tables(r, 0, Dn, tables, classes, min_overlaps, n_off, compute_aos, None)
            if edges is not None:
                res["ranges"] = [(lo, hi, _ap_tables(r, (b + 1) * Dn, Dn, tables, classes, min_overlaps, n_off,
                                                     compute_aos, (lo, hi)))
                                 for b, (lo, hi) in enumerate(bins[1:])]
        if match:
            res["matches"] = matches[s]
        if boot is not None:
            res["bootstrap"] = boot[s][0]
            if edges is not None:
                res["bootstrap_ranges"] = [(lo, hi, boot[s][b + 1]) for b, (lo, hi) in enumerate(bins[1:])]
        out.append(res)
    return out


# ------------------------------------------------------------------ bootstrap
BOOTSTRAP_CHUNK = 64    # replicates per device pass: the device arrays of a pass grow with it, not with R


def bootstrap_indices(nframes, replicates, seed=0):
    """[replicates, nframes] int64 frame indices, row r the r-th draw of np.random.RandomState(seed).randint(0,
    nframes, nframes): a row does not depend on how many rows follow it."""
    rs = np.random.RandomState(seed)
    return np.stack([rs.randint(0, nframes, nframes) for _ in range(int(replicates))]).astype(np.int64)


class ReplicateLists:
    """R >= 1 bootstrap replicates, each a non-empty list of frame indices of any length (a drive-level replicate is
    the frames of its drawn drives): ``flat`` int64 the lists concatenated, ``off`` int64 [R + 1] replicate r's slice
    flat[off[r]:off[r + 1]].  Built from a sequence of 1-D integer arrays; an empty list, a non-integer index or no list
    at all is a ValueError.  eval_many refuses an index outside the split's frames."""

    def __init__(self, lists):
        rows = [np.asarray(l) for l in lists]
        if not rows:
            raise ValueError("bootstrap replicate lists: need at least one replicate")
        for r, row in enumerate(rows):
            if row.ndim != 1 or not len(row):
                raise ValueError("bootstrap replicate %d must be a non-empty 1-D list of frame indices, not shape %r"
                                 % (r, row.shape))
            if row.dtype.kind not in "iu":
                raise ValueError("bootstrap replicate %d: frame indices must be integers, not %s" % (r, row.dtype))
        self.flat = np.concatenate(rows).astype(np.int64)
        self.off = _offsets([len(row) for row in rows], np.int64)

    @classmethod
    def _from(cls, flat, off):
        out = cls.__new__(cls)
        out.flat, out.off = flat, off
        return out

    @classmethod
    def _of_array(cls, idx):
        """The rows of an [R, F] index array: replicate r at offset r * F."""
        return cls._from(np.ascontiguousarray(idx, np.int64).reshape(-1),
                         np.arange(idx.shape[0] + 1, dtype=np.int64) * idx.shape[1])

    def __len__(self):
        return len(self.off) - 1

    def __getitem__(self, r):
        return self.flat[self.off[r]:self.off[r + 1]]

    def __iter__(self):
        return (self[r] for r in range(len(self)))

    @property
    def lengths(self):
        return np.diff(self.off)

    def rows(self, r0, r1):
        """Replicates [r0, r1) as a ReplicateLists."""
        return ReplicateLists._from(self.flat[self.off[r0]:self.off[r1]], self.off[r0:r1 + 1] - self.off[r0])


def bootstrap_groups(groups, replicates, seed=0):
    """Drive-level (cluster) bootstrap replicates as ReplicateLists: ``groups`` holds one label per split frame (its
    raw drive).  The G distinct labels are sorted; replicate r draws G of them with the r-th
    np.random.RandomState(seed).randint(0, G, G) and lists each drawn group's frame positions in ascending order, group
    after group.  A row does not depend on how many rows follow it; with groups = np.arange(F) the rows are
    bootstrap_indices(F, replicates, seed)'s."""
    labels, inv = np.unique(np.asarray(groups), return_inverse=True)
    inv = inv.reshape(-1)
    G = len(labels)
    if G < 1:
        raise ValueError("bootstrap groups: need a label per frame, not an empty list")
    members = [np.flatnonzero(inv == g) for g in range(G)]
    rs = np.random.RandomState(seed)
    return ReplicateLists([np.concatenate([members[g] for g in rs.randint(0, G, G)]) for _ in range(int(replicates))])


def check_bootstrap(idx, nframes):
    """The bootstrap replicates as ReplicateLists.  An array must be an int [R >= 1, nframes] array; a ReplicateLists
    may hold lists of any length; every index must lie in [0, nframes).  Anything else is a ValueError."""
    if isinstance(idx, ReplicateLists):
        if nframes < 1 or idx.flat.min() < 0 or idx.flat.max() >= nframes:
            raise ValueError("bootstrap indices must lie in [0, %d)" % nframes)
        return idx
    a = np.asarray(idx)
    if a.dtype.kind not in "iu":
        raise ValueError("bootstrap indices must be integers, not %s" % a.dtype)
    if a.ndim != 2 or a.shape[0] < 1 or a.shape[1] != nframes or nframes < 1:
        raise ValueError("bootstrap indices must be [R >= 1, %d frames], not %r" % (nframes, a.shape))
    if a.min() < 0 or a.max() >= nframes:
        raise ValueError("bootstrap indices must lie in [0, %d)" % nframes)
    return ReplicateLists._of_array(a)


def percentile_interval(samples, lo=2.5, hi=97.5):
    """[2, ...]: np.percentile of the replicates (axis 0) at ``lo`` and ``hi`` percent."""
    return np.percentile(np.asarray(samples, np.float64), [lo, hi], axis=0)


def paired_summary(ap, ap0, lo=2.5, hi=97.5):
    """A set's replicate AP against the first set's, paired replicate by replicate: dict(interval=percentile_interval
    of ap - ap0, better=the fraction of replicates with ap - ap0 > 0)."""
    d = np.asarray(ap, np.float64) - np.asarray(ap0, np.float64)
    return dict(interval=percentile_interval(d, lo, hi), better=np.mean(d > 0, axis=0))


def _bootstrap_aos_flags(dt_blocks, lists):
    """[R, K] compute_aos of every replicate (ReplicateLists) and set, as _aos_flag decides it on the replicate's list:
    from its first frame with detections."""
    out = np.zeros((len(lists), len(dt_blocks)), bool)
    for k, d in enumerate(dt_blocks):
        has = d.counts > 0
        ok = np.zeros(len(d), bool)
        if has.any():
            ok[has] = d.alpha[d.off[:-1][has]].cpu().numpy() != -10
        hit = np.flatnonzero(has[lists.flat])               # list positions of frames with detections
        j = np.searchsorted(hit, lists.off[:-1])            # each replicate's first such position, if in its slice
        found = j < len(hit)
        found[found] = hit[j[found]] < lists.off[1:][found]
        out[found, k] = ok[lists.flat[hit[j[found]]]]
    return out


def _with_aos(ap, flags):
    """A bootstrap AP dict's aos: NaN in the replicates without compute_aos, None when no replicate has it."""
    if not flags.any():
        return dict(ap, aos=None)
    return dict(ap, aos=np.where(flags.reshape((-1,) + (1,) * (ap["aos"].ndim - 1)), ap["aos"], np.nan))


def _stack_aps(aps):
    """One AP dict with a leading replicate axis from per-replicate AP dicts (a None aos becomes NaN)."""
    out = {}
    for key in aps[0]:
        vals = [a[key] for a in aps]
        some = next((v for v in vals if v is not None), None)
        out[key] = None if some is None else np.stack([np.full_like(some, np.nan) if v is None else v for v in vals])
    return out


def _bootstrap_host(gt_annos, dt_sets, classes, tables, overlap_fn, difficultys, edges, lists):
    """The reference implementation: the host evaluation of each replicate's lists (ReplicateLists).  [set][whole
    range, bins...] -> {table: ap with a leading R axis}."""
    per = [[] for _ in dt_sets]
    for row in lists:
        ev = _evaluate([gt_annos[i] for i in row], [[d[i] for i in row] for d in dt_sets], classes, tables, overlap_fn,
                       difficultys, edges, False)
        for s, e in enumerate(ev):
            per[s].append([{t: e[t][1] for t in tables}] + [{t: r[t][1] for t in tables} for _, _, r in
                                                            e.get("ranges", [])])
    return [[{t: _stack_aps([rep[b][t] for rep in reps]) for t in tables} for b in range(len(reps[0]))]
            for reps in per]


def _bootstrap_device(st, lists, boot_aos, tables, Dn, nbins, n_off):
    """The replicates (ReplicateLists) on the device from the evaluation's set-up ``st``: each job's sorted
    true-positive scores and each (job, frame)'s step table once (sassd_kitti_boot_prepare), then per chunk of
    BOOTSTRAP_CHUNK replicates their thresholds and per-threshold sums (sassd_kitti_boot_eval) and eval_many's numpy
    tail on [R, ...] arrays.  Returns _bootstrap_host's layout."""
    from . import ops
    K, F, C, D, M = st.K, st.F, st.C, st.Dn, st.M
    njobs = len(st.region)
    desc = _lib.KittiEvalDesc.from_buffer_copy(st.desc)
    any_aos = st.up(boot_aos.any(0).astype(np.int32))
    desc.compute_aos = any_aos.data_ptr()
    # set k's block per job: one entry per detection row and one per frame
    per_set = np.array([int(d.off[-1]) + F for d in st.dts], np.int64)
    tab_off = st.up(_offsets(np.repeat(per_set, njobs // K), np.int64))
    prep = ops.kitti_boot_prepare(desc, njobs, int(st.region.sum()), tab_off)
    # each frame's valid GT count per (class, difficulty entry)
    valid = (st.keep["ign_gt"] == 0).cpu().numpy().reshape(C * D, -1).astype(np.int64)
    cs = np.concatenate([np.zeros((C * D, 1), np.int64), np.cumsum(valid, 1)], 1)
    nv = cs[:, st.gt.off[1:]] - cs[:, st.gt.off[:-1]]
    chunks = []
    for r0 in range(0, len(lists), BOOTSTRAP_CHUNK):
        part = lists.rows(r0, min(r0 + BOOTSTRAP_CHUNK, len(lists)))
        R = len(part)
        rep = np.repeat(np.arange(R), part.lengths)
        w = np.bincount(part.flat + F * rep, minlength=R * F).reshape(R, F)
        n_thresh, pr = ops.kitti_boot_eval(desc, njobs, st.up(part.flat.astype(np.int32)), st.up(part.off),
                                           st.up(w.astype(np.int32)), st.up((w @ nv.T).astype(np.float64)), prep,
                                           tab_off)
        prec = _pr_arrays(pr.cpu().numpy().reshape(R, K, C, D, 3, M, 41, 4),
                          n_thresh.cpu().numpy().reshape(R, K, C, D, 3, M), boot_aos[r0:r0 + R])
        chunks.append([[_ap_dicts([p[k] for p in prec], b * Dn, Dn, tables, n_off, True) for b in range(nbins)]
                       for k in range(K)])
    return [[{t: _with_aos({key: np.concatenate([c[k][b][t][key] for c in chunks]) for key in chunks[0][k][b][t]},
                           boot_aos[:, k]) for t in tables} for b in range(nbins)] for k in range(K)]


def _ap_tables(r, e0, Dn, tables, classes, min_overlaps, n_off, compute_aos, rng):
    """{table: (text, ap)} of difficulty entries [e0, e0 + Dn) of one set's precision arrays r[metric]."""
    res = {}
    for t, ap in _ap_dicts(r, e0, Dn, tables, n_off, compute_aos).items():
        text = (_coco_text(ap, classes, compute_aos, rng) if t == "coco" else
                _ap_text(ap, classes, min_overlaps[:n_off], compute_aos, "AP" if t == 11 else "AP_R40", rng))
        res[t] = (text, ap)
    return res


def _ap_dicts(r, e0, Dn, tables, n_off, compute_aos):
    """{table: ap} of difficulty entries [e0, e0 + Dn) of precision arrays r[metric] of [..., C, entries, M, 41] (any
    leading axes, e.g. bootstrap replicates)."""
    r0, r1, r2 = ({k: v[..., e0:e0 + Dn, :, :] for k, v in m.items()} for m in r)
    res = {}
    for rp in (t for t in tables if t in (11, 40)):
        get_mAP_n = get_mAP if rp == 11 else get_mAP_R40
        res[rp] = dict(bbox=get_mAP_n(r0["precision"][..., :n_off, :]),
                       aos=get_mAP_n(r0["orientation"][..., :n_off, :]) if compute_aos else None,
                       bev=get_mAP_n(r1["precision"][..., :n_off, :]), d3=get_mAP_n(r2["precision"][..., :n_off, :]))
    if "coco" in tables:
        # do_coco_style_eval (kitti_eval.py:711-729): the mean over the ten overlaps of get_mAP_v2
        c0 = n_off + 10
        res["coco"] = dict(bbox=get_mAP(r0["precision"][..., n_off:c0, :]).mean(-1),
                           aos=get_mAP(r0["orientation"][..., n_off:c0, :]).mean(-1) if compute_aos else None,
                           bev=get_mAP(r1["precision"][..., n_off:c0, :]).mean(-1),
                           d3=get_mAP(r2["precision"][..., n_off:c0, :]).mean(-1))
    return res


def coco_eval_many(gt_annos, dt_sets, classes, overlap_fn=None):
    """coco_eval of K detection sets against the same GT in one evaluation: one (text, ap) per set."""
    return [r["coco"] for r in eval_many(gt_annos, dt_sets, classes, ("coco",), overlap_fn)]


def coco_eval(gt_annos, dt_annos, classes, overlap_fn=None):
    """-> (text, dict(bbox, bev, d3, aos) of AP arrays [class, difficulty]): the reference's COCO-style KITTI AP, each
    value the mean over the class's ten IoU thresholds of the 11-point AP (``aos`` is None when the detections carry
    no alpha)."""
    return coco_eval_many(gt_annos, [dt_annos], classes, overlap_fn)[0]


def get_coco_eval_result(gt_annos, dt_annos, current_classes, overlap_fn=None):
    """Reference signature (kitti_eval.py:853): the printed COCO-style table."""
    return coco_eval(gt_annos, dt_annos, current_classes, overlap_fn)[0]


def _range_label(rng):
    """The heading suffix of a range bin's table ("" for the whole range)."""
    return "" if rng is None else " range [%g, %g) m" % rng


def _coco_text(ap, classes, compute_aos, rng=None):
    """get_coco_eval_result's table (kitti_eval.py:904-930); a range bin's names its range in each heading."""
    lines = []
    for j, cls in enumerate(classes):
        start, stop, num = COCO_RANGE[cls]
        lines.append("%s coco AP@%.2f:%.2f:%.2f%s:" % (CLASS_TO_NAME[cls], start, (stop - start) / (num - 1), stop,
                                                      _range_label(rng)))
        for key, label in (("bbox", "bbox AP"), ("bev", "bev  AP"), ("d3", "3d   AP")) + ((("aos", "aos  AP"),)
                                                                                           if compute_aos else ()):
            lines.append("%s:%.2f, %.2f, %.2f" % (label, ap[key][j, 0], ap[key][j, 1], ap[key][j, 2]))
    return "".join(l + "\n" for l in lines)


def _ap_text(ap, classes, min_overlaps, compute_aos, tag, rng=None):
    """The official table of official_eval's AP arrays; a range bin's names its range in each heading."""
    lines = []
    for j, cls in enumerate(classes):
        for i in range(min_overlaps.shape[0]):
            lines.append("%s %s@%.2f, %.2f, %.2f%s:" % ((CLASS_TO_NAME[cls], tag) + tuple(min_overlaps[i, :, j])
                                                       + (_range_label(rng),)))
            for key, label in (("bbox", "bbox AP"), ("bev", "bev  AP"), ("d3", "3d   AP")):
                lines.append("%s:%.2f, %.2f, %.2f" % (label, ap[key][j, 0, i], ap[key][j, 1, i], ap[key][j, 2, i]))
            if compute_aos:
                lines.append("aos  AP:%.2f, %.2f, %.2f" % (ap["aos"][j, 0, i], ap["aos"][j, 1, i], ap["aos"][j, 2, i]))
    return "".join(l + "\n" for l in lines)


def get_official_eval_result(gt_annos, dt_annos, current_classes, difficultys=[0, 1, 2], overlap_fn=None):
    """Reference signature (kitti_eval.py:791): the printed result table."""
    return official_eval(gt_annos, dt_annos, current_classes, difficultys, overlap_fn)[0]


# ------------------------------------------------------------------ result directories
def ap_lists(ap):
    """An AP dict as JSON-ready nested lists."""
    return {k: (None if v is None else np.asarray(v).tolist()) for k, v in ap.items()}


def tp_error_summary(table, classes, difficultys=(0, 1, 2), ranges=None):
    """Per class, at moderate difficulty: the 3-D metric's true-positive count and the means (numpy's) of their ATE,
    ASE and AOE (None without a true positive), over the whole range and, with ``ranges``, per bin of the GT's range.
    ``table``: one set's match_table.  A list of dicts (class, tp, ate, ase, aoe[, ranges: [dict(lo, hi, tp, ...)]])."""
    d = list(difficultys).index(1)
    out = []
    for ci, c in enumerate(_class_ids(classes)):
        j = table["gt_det"][ci, d, 2]
        tp = j >= 0
        tp[tp] = table["dt_state"][ci, d, 2][j[tp]] == _lib.KITTI_DT_TP
        err = table["tp_errors"][ci, d]

        def stats(mask):
            e = err[mask]
            return dict(tp=int(mask.sum()), **{k: (float(np.mean(e[:, i])) if len(e) else None)
                                                for i, k in enumerate(("ate", "ase", "aoe"))})
        entry = dict(cls=CLASS_TO_NAME[c], **stats(tp))
        if ranges is not None:
            r = table["gt_range"]
            entry["ranges"] = [dict(lo=lo, hi=_json_edge(hi), **stats(tp & (lo <= r) & (r < hi)))
                               for lo, hi in range_bins(check_ranges(ranges))]
        out.append(entry)
    return out


def _json_edge(e):
    """A bin edge for JSON: inf as None."""
    return None if np.isinf(e) else e


def _fmt_err(st):
    return "TP %d ATE %s ASE %s AOE %s" % ((st["tp"],) + tuple("-" if st[k] is None else "%.4f" % st[k]
                                                               for k in ("ate", "ase", "aoe")))


def range_report(entry, ev, class_names, log=print, tp_err=None):
    """Print a set's per-range tables (``ev``: eval_many's dict with ``ranges``, or without: nothing) after its
    whole-range ones and put their texts and AP lists into ``entry`` (text_ranges / ap_ranges and the _r40 / _coco
    variants evaluated), and ``tp_err`` (tp_error_summary) as ``tp_errors``.  Returns the summary fields: moderate 3D
    AP per class per bin, then the TP error means per class."""
    fields = []
    if "ranges" in ev:
        for suffix, t in (("", 11), ("_r40", 40), ("_coco", "coco")):
            if t not in ev:
                continue
            for _, _, res in ev["ranges"]:
                log(res[t][0], end="")
            entry["text_ranges" + suffix] = [res[t][0] for _, _, res in ev["ranges"]]
            entry["ap_ranges" + suffix] = [dict(lo=lo, hi=_json_edge(hi), ap=ap_lists(res[t][1]))
                                           for lo, hi, res in ev["ranges"]]
        for j, c in enumerate(class_names):
            for lo, hi, res in ev["ranges"]:
                fields.append("%s 3d mod [%g, %g) R11 %6.2f" % (c, lo, hi, res[11][1]["d3"][j, 1, 0]) +
                              (" R40 %6.2f" % res[40][1]["d3"][j, 1, 0] if 40 in res else "") +
                              (" COCO %6.2f" % res["coco"][1]["d3"][j, 1] if "coco" in res else ""))
    if tp_err is not None:
        entry["tp_errors"] = tp_err
        for st in tp_err:
            fields.append("%s %s" % (st["cls"], _fmt_err(st)))
            for b in st.get("ranges", []):
                fields.append("%s [%g, %g) %s" % (st["cls"], b["lo"], np.inf if b["hi"] is None else b["hi"],
                                                  _fmt_err(b)))
    return fields


def _interval_lists(ap):
    """percentile_interval of each of a bootstrap AP dict's arrays as JSON-ready lists ([2, ...]: low, high)."""
    return {k: (None if v is None else percentile_interval(v).tolist()) for k, v in ap.items()}


def _strict(a):
    """[R, C, 3] of an AP array: the class's strict (first) overlap row of an official table; COCO has no row axis."""
    return a[..., 0] if a.ndim == 4 else a


def _replicates_text(nrep, groups=None):
    """How the blocks name the replicates: "R replicates", or "R drive-level replicates of G drives" (``groups``: G
    for a drive-level bootstrap)."""
    return "%d replicates" % nrep if groups is None else "%d drive-level replicates of %d drives" % (nrep, groups)


def bootstrap_report(ev, class_names, log=print, groups=None):
    """Print a set's bootstrap block (``ev``: eval_many's dict with ``bootstrap``): per table and class the 95 %
    percentile interval of bbox / BEV / 3D / AOS AP for easy, moderate and hard at the class's strict overlap
    (``groups``: the drive count of a drive-level bootstrap, named in the headings).  Returns (the JSON entry {table:
    interval lists}, the summary fields: the moderate 3D interval per class and table)."""
    boot = ev["bootstrap"]
    nrep = len(boot[11]["d3"])
    for t, ap in boot.items():
        tag = "AP" if t == 11 else "AP_R40" if t == 40 else "coco AP"
        for j, c in enumerate(class_names):
            log("%s %s 95%% interval (%s):" % (c, tag, _replicates_text(nrep, groups)))
            for key, label in (("bbox", "bbox AP"), ("bev", "bev  AP"), ("d3", "3d   AP"), ("aos", "aos  AP")):
                if ap[key] is None:
                    continue
                iv = percentile_interval(_strict(ap[key])[:, j])
                log("%s:%s" % (label, ", ".join("[%.2f, %.2f]" % (iv[0, d], iv[1, d]) for d in range(3))))
    fields = []
    for j, c in enumerate(class_names):
        fields.append("%s 3d mod 95%% " % c + " ".join(
            "%s [%.2f, %.2f]" % ((("R11", "R40", "COCO")[TABLES.index(t)],) + tuple(percentile_interval(
                _strict(ap["d3"])[:, j, 1]))) for t, ap in boot.items()))
    return {str(t): _interval_lists(ap) for t, ap in boot.items()}, fields


def paired_report(labels, evs, class_names, log=print, groups=None):
    """Print each set's moderate 3D AP against the first set's, paired over the bootstrap replicates: per set and class
    and table the 95 % interval of the difference and the share of replicates in which the set is better (``groups``
    as bootstrap_report's).  Returns the JSON list."""
    out = []
    log("paired against %s (moderate 3D AP, %s):" % (labels[0], _replicates_text(len(evs[0]["bootstrap"][11]["d3"]),
                                                                                 groups)))
    for k in range(1, len(evs)):
        for t in evs[0]["bootstrap"]:
            name = ("R11", "R40", "COCO")[TABLES.index(t)]
            for j, c in enumerate(class_names):
                sm = paired_summary(_strict(evs[k]["bootstrap"][t]["d3"])[:, j, 1],
                                    _strict(evs[0]["bootstrap"][t]["d3"])[:, j, 1])
                log("%-24s %s %s dAP 95%% [%+.2f, %+.2f]  better in %.1f%% of replicates" % (
                    labels[k], c, name, sm["interval"][0], sm["interval"][1], 100 * sm["better"]))
                out.append(dict(set=str(labels[k]), against=str(labels[0]), table=str(t), cls=c,
                                interval=sm["interval"].tolist(), better=float(sm["better"])))
    return out


def add_bootstrap_args(p):
    """The --bootstrap / --bootstrap-seed options of the evaluation commands."""
    p.add_argument("--bootstrap", type=int, default=None, metavar="R",
                   help="also print 95%% intervals of the AP over R bootstrap replicates of the split's frames (and, "
                        "for several sets, each set's paired difference against the first)")
    p.add_argument("--bootstrap-seed", type=int, default=None, metavar="S",
                   help="the seed of the replicates' frame draws (default 0)")
    p.add_argument("--bootstrap-by", default=None, choices=("frame", "drive"),
                   help="resample the split's frames (default) or its raw drives, whole (needs --mapping)")
    p.add_argument("--mapping", default=None, metavar="DIR",
                   help="the KITTI object devkit's mapping/ directory (train_mapping.txt, train_rand.txt): each "
                        "training frame's raw drive, for --bootstrap-by drive and --per-drive")
    p.add_argument("--per-drive", action="store_true",
                   help="also print each drive's frame count and moderate 3D AP (needs --mapping)")


def check_bootstrap_args(p, args, unlabelled=None):
    """Refuse --bootstrap below 1, --bootstrap, --bootstrap-by, --mapping or --per-drive without labels
    (``unlabelled``: the option that has none), --bootstrap-seed or --bootstrap-by without --bootstrap,
    --bootstrap-by drive or --per-drive without --mapping, and --mapping without either of them."""
    if args.bootstrap is not None:
        if args.bootstrap < 1:
            p.error("--bootstrap must be at least 1")
        if unlabelled:
            p.error("--bootstrap needs a labelled split: %s has no labels" % unlabelled)
    elif args.bootstrap_seed is not None:
        p.error("--bootstrap-seed goes with --bootstrap")
    for flag, given in (("--bootstrap-by", args.bootstrap_by is not None), ("--mapping", args.mapping is not None),
                        ("--per-drive", args.per_drive)):
        if given and unlabelled:
            p.error("%s needs a labelled split: %s has no labels" % (flag, unlabelled))
    if args.bootstrap_by is not None and args.bootstrap is None:
        p.error("--bootstrap-by goes with --bootstrap")
    if args.bootstrap_by == "drive" and args.mapping is None:
        p.error("--bootstrap-by drive needs --mapping (the devkit's mapping/ directory)")
    if args.per_drive and args.mapping is None:
        p.error("--per-drive needs --mapping (the devkit's mapping/ directory)")
    if args.mapping is not None and args.bootstrap_by != "drive" and not args.per_drive:
        p.error("--mapping goes with --bootstrap-by drive or --per-drive")
    if args.bootstrap is not None and args.bootstrap_seed is None:
        args.bootstrap_seed = 0
    if args.bootstrap is not None and args.bootstrap_by is None:
        args.bootstrap_by = "frame"


def split_drives_of(args, ids):
    """Each frame of ``ids``'s raw drive from --mapping (kitti_data.read_drive_mapping, split_drives), or None
    without it."""
    if args.mapping is None:
        return None
    from .kitti_data import read_drive_mapping, split_drives
    return split_drives(read_drive_mapping(args.mapping), ids)


def bootstrap_kw(args, nframes, drives=None):
    """eval_many's bootstrap argument of the command's options (``drives``: split_drives_of's, for --bootstrap-by
    drive)."""
    if args.bootstrap is None:
        return {}
    if args.bootstrap_by == "drive":
        return dict(bootstrap=bootstrap_groups(drives, args.bootstrap, args.bootstrap_seed))
    return dict(bootstrap=bootstrap_indices(nframes, args.bootstrap, args.bootstrap_seed))


def bootstrap_groups_of(args, drives):
    """The drive count G of a drive-level bootstrap (what the blocks name), None otherwise."""
    if args.bootstrap is None or args.bootstrap_by != "drive":
        return None
    return len(np.unique(drives))


def pop_bootstrap(args, nframes, labels, entries, kw=None, drives=None):
    """The --json ``bootstrap`` entry, taken out of report_sets' entries: R, seed, F, per set its label and {table:
    intervals}, and the paired summaries against the first set (None without --bootstrap).  A drive-level bootstrap
    (``kw``: bootstrap_kw's, ``drives``: split_drives_of's) adds ``by``, the drive count ``groups`` and the replicate
    lists' lengths (min, median, max)."""
    if args.bootstrap is None:
        return None
    out = dict(replicates=args.bootstrap, seed=args.bootstrap_seed, frames=nframes,
               sets=[dict(label=str(l), intervals=e.pop("bootstrap")) for l, e in zip(labels, entries)],
               paired=entries[0].pop("bootstrap_paired", []))
    if args.bootstrap_by == "drive":
        n = kw["bootstrap"].lengths
        out.update(by="drive", groups=bootstrap_groups_of(args, drives),
                   lengths=dict(min=int(n.min()), median=float(np.median(n)), max=int(n.max())))
    return out


def per_drive_report(gt, dt_sets, labels, class_names, tables, drives, log=print):
    """Print one line per drive after the tables: its name, frame count and, for every set (columns, in ``labels``
    order), the moderate 3D AP per class of each table at the class's strict overlap.  One eval_many whose replicate r
    is drive r's frame list (drives sorted by name), so each line is that drive's own evaluation.  Returns the --json
    ``per_drive`` list: per drive its name, frame count and per set {table: AP dict}."""
    names, inv = np.unique(np.asarray(drives), return_inverse=True)
    lists = ReplicateLists([np.flatnonzero(inv.reshape(-1) == g) for g in range(len(names))])
    evs = eval_many(gt, dt_sets, class_names, tables, bootstrap=lists)
    tags = [("R11", "R40", "COCO")[TABLES.index(t)] for t in tables]
    log("per drive (moderate 3D AP, %d drives; columns: %s):" % (len(names), " | ".join(str(l) for l in labels)))
    out = []
    for g, name in enumerate(names):
        cols = []
        for ev in evs:
            d3 = [_strict(ev["bootstrap"][t]["d3"])[g] for t in tables]
            cols.append("  ".join("%s 3d mod %s" % (c, " ".join("%s %6.2f" % (tag, a[j, 1])
                                                              for tag, a in zip(tags, d3)))
                                  for j, c in enumerate(class_names)))
        log("%-32s %5d frames  %s" % (name, lists.lengths[g], " | ".join(cols)))
        out.append(dict(drive=str(name), frames=int(lists.lengths[g]),
                        sets=[dict(label=str(l), ap={str(t): ap_lists({k: None if v is None else v[g]
                                                                       for k, v in ev["bootstrap"][t].items()})
                                                     for t in tables}) for l, ev in zip(labels, evs)]))
    return out


def write_matches(path, labels, tables):
    """Write each set's match_table to an .npz: set k's arrays as ``set<k>_<name>``, ``labels`` [K] the sets' labels
    and the KITTI_DT_* state names ``states``."""
    out = dict(labels=np.array([str(l) for l in labels]),
               states=np.array(["not_counted", "tp", "fp", "dontcare", "ignored"]))
    for k, t in enumerate(tables):
        out.update({"set%d_%s" % (k, name): v for name, v in t.items()})
    np.savez_compressed(path, **out)


def report_sets(entries, labels, evs, class_names, noun, log=print, extra=None, ranges=None, groups=None):
    """Print each evaluated set's tables (``evs``: eval_many's dicts, with table 11) under ``== label ==``, then one
    summary line per set: moderate 3D AP per class at the class's strict overlap (R11, and R40 / COCO when evaluated).
    Each set's texts and AP lists go into its dict of ``entries`` (returned).  ``extra(k, entry)`` may add to set k's
    entry after its tables and returns more summary fields.  A set evaluated with ranges or a match table also prints
    its per-range tables, and its summary line gains range_report's fields (``ranges``: the bin edges).  ``groups``:
    the drive count of a drive-level bootstrap (bootstrap_report's)."""
    summary = []
    for k, (entry, label, ev) in enumerate(zip(entries, labels, evs)):
        log("== %s ==" % label)
        text, ap = ev[11]
        log(text, end="")
        entry.update(text=text, ap=ap_lists(ap))
        line = ["%-24s" % label]
        for j, c in enumerate(class_names):
            line.append("%s 3d mod R11 %6.2f" % (c, ap["d3"][j, 1, 0]) +
                        (" R40 %6.2f" % ev[40][1]["d3"][j, 1, 0] if 40 in ev else "") +
                        (" COCO %6.2f" % ev["coco"][1]["d3"][j, 1] if "coco" in ev else ""))
        if 40 in ev:
            log(ev[40][0], end="")
            entry.update(text_r40=ev[40][0], ap_r40=ap_lists(ev[40][1]))
        if "coco" in ev:
            log(ev["coco"][0], end="")
            entry.update(text_coco=ev["coco"][0], ap_coco=ap_lists(ev["coco"][1]))
        if "ranges" in ev or "matches" in ev:
            tp_err = tp_error_summary(ev["matches"], class_names, ranges=ranges) if "matches" in ev else None
            line += range_report(entry, ev, class_names, log, tp_err)
        if "bootstrap" in ev:
            entry["bootstrap"], fields = bootstrap_report(ev, class_names, log, groups)
            line += fields
        if extra is not None:
            line += extra(k, entry)
        summary.append("  ".join(line))
    log("summary: %d %s (moderate 3D AP)" % (len(labels), noun))
    for line in summary:
        log(line)
    if len(evs) > 1 and "bootstrap" in evs[0]:
        entries[0]["bootstrap_paired"] = paired_report(labels, evs, class_names, log, groups)
    return entries


def read_dirs(label_dir, result_dirs, ids, times=None):
    """The AnnoBlocks of the label files and of every result directory over the frames ``ids`` (read_block)."""
    return read_block(label_dir, ids, times=times), [read_block(d, ids, times=times) for d in result_dirs]


def eval_dirs(label_dir, result_dirs, ids, classes, tables=(11,), times=None, ranges=None, match=False,
              bootstrap=None):
    """Every table of ``tables`` for each directory of KITTI result files in ``result_dirs`` against the label files
    of ``label_dir``, over the frames ``ids``: the GT is read once, every directory is read and parsed on the device
    (read_block), and one eval_many evaluates them all (``ranges``, ``match``, ``bootstrap``: eval_many's).  Returns
    eval_many's list,
    one dict per directory.  ``times``: a dict whose "read", "parse" and "eval" entries accumulate seconds."""
    times = {} if times is None else times
    gt, dts = read_dirs(label_dir, result_dirs, ids, times)
    t0 = time.perf_counter()
    out = eval_many(gt, dts, classes, tables, ranges=ranges, match=match, bootstrap=bootstrap)
    times["eval"] = times.get("eval", 0.0) + time.perf_counter() - t0
    return out


def parse_args(argv=None):
    p = argparse.ArgumentParser(prog="python -m sassd_b200.kitti_eval", description=main.__doc__.split("\n\n")[0])
    p.add_argument("--data-root", required=True, help="KITTI root holding ImageSets/ and training/label_2/")
    p.add_argument("--split", default="val", help="the frames of ImageSets/<split>.txt (default val)")
    p.add_argument("--results", nargs="+", required=True, metavar="DIR",
                   help="directories of KITTI result files %%06d.txt (a 16th field the score)")
    p.add_argument("--classes", nargs="+", default=["Car"], metavar="CLASS",
                   help="classes to evaluate, among %s (default Car)" % ", ".join(CLASS_TO_NAME.values()))
    p.add_argument("--r40", action="store_true", help="also print the AP table at 40 recall positions")
    p.add_argument("--coco", action="store_true",
                   help="also print the COCO-style AP table (AP averaged over ten IoU thresholds per class)")
    p.add_argument("--json", default=None, help="write the AP arrays and times here")
    add_range_args(p)
    add_bootstrap_args(p)
    args = p.parse_args(argv)
    check_range_args(p, args)
    check_bootstrap_args(p, args)
    unknown = [c for c in args.classes if c not in CLASS_TO_NAME.values()]
    if unknown:
        p.error("--classes: unknown class %s (known: %s)" % (", ".join(unknown), ", ".join(CLASS_TO_NAME.values())))
    if not os.path.isfile(os.path.join(args.data_root, "ImageSets", args.split + ".txt")):
        p.error("--split %s: %s does not exist" % (args.split, os.path.join(args.data_root, "ImageSets",
                                                                              args.split + ".txt")))
    if not os.path.isdir(os.path.join(args.data_root, "training", "label_2")):
        p.error("--data-root %s has no training/label_2 directory" % args.data_root)
    missing = [d for d in args.results if not os.path.isdir(d)]
    if missing:
        p.error("--results: %s is not a directory" % missing[0])
    return args


def add_range_args(p):
    """The --ranges / --matches options of the evaluation commands."""
    p.add_argument("--ranges", nargs="+", type=float, default=None, metavar="EDGE",
                   help="also print the tables per range bin [e_i, e_i+1) of ground distance from the camera, in m "
                        "(e.g. 0 20 40 inf), and the true positives' mean ATE / ASE / AOE")
    p.add_argument("--matches", default=None, metavar="NPZ",
                   help="write each set's per-object match table (kitti_eval.match_table) to this .npz")


def check_range_args(p, args):
    if args.ranges is not None:
        try:
            args.ranges = list(check_ranges(args.ranges))
        except ValueError as e:
            p.error("--ranges: %s" % e)


def main(argv=None, log=print):
    """Evaluate directories of KITTI result files against a split's labels (SECOND's kitti-object-eval-python):

    python -m sassd_b200.kitti_eval --data-root DIR [--split val] --results DIR [DIR ...]
                                    [--classes Car Pedestrian Cyclist] [--r40] [--coco] [--json FILE]
                                    [--ranges EDGE EDGE [...]] [--matches FILE.npz]
                                    [--bootstrap R [--bootstrap-seed S] [--bootstrap-by frame|drive]]
                                    [--mapping DIR [--per-drive]]

    The labels are ``training/label_2/%06d.txt`` and the frames those of ``ImageSets/<split>.txt``; files a result
    directory holds beyond them are ignored.  Every file is read into pinned memory, copied to the device once and
    parsed there (read_block), and all directories are evaluated in one pass (eval_many) on the device.  Prints each
    directory's tables under ``== DIR ==``, one summary line per directory and the seconds spent reading, parsing and
    evaluating.  ``--ranges`` adds each directory's tables per range bin and, with ``--matches``, the true positives'
    TP errors to its summary line; ``--matches`` writes every directory's match table.  ``--bootstrap R`` adds each
    directory's 95 % AP intervals over R bootstrap replicates of the frames (bootstrap_indices, seed
    ``--bootstrap-seed``) and, for two or more directories, each one's paired difference against the first.
    ``--mapping DIR`` is the object devkit's ``mapping/`` directory; with it ``--bootstrap-by drive`` resamples whole
    raw drives (bootstrap_groups) and ``--per-drive`` prints each drive's frame count and moderate 3D AP, one column
    per directory (per_drive_report).  Returns the result dict that ``--json`` writes."""
    from .kitti_data import read_split
    args = parse_args(argv)
    ids = read_split(args.data_root, args.split)
    drives = split_drives_of(args, ids)
    tables = (11,) + ((40,) if args.r40 else ()) + (("coco",) if args.coco else ())
    times = {}
    match = args.ranges is not None or args.matches is not None
    gt, dts = read_dirs(os.path.join(args.data_root, "training", "label_2"), args.results, ids, times)
    kw = bootstrap_kw(args, len(ids), drives)
    t0 = time.perf_counter()
    evs = eval_many(gt, dts, args.classes, tables, ranges=args.ranges, match=match, **kw)
    times["eval"] = time.perf_counter() - t0
    entries = report_sets([dict(dir=d) for d in args.results], args.results, evs, args.classes, "directories", log,
                          ranges=args.ranges, groups=bootstrap_groups_of(args, drives))
    boot = pop_bootstrap(args, len(ids), args.results, entries, kw, drives)
    per_drive = (per_drive_report(gt, dts, args.results, args.classes, tables, drives, log) if args.per_drive
                 else None)
    if args.matches:
        write_matches(args.matches, args.results, [ev["matches"] for ev in evs])
    log("frames: %d, directories: %d, read %.3f s, parse %.3f s, evaluate %.3f s" % (
        len(ids), len(args.results), times["read"], times["parse"], times["eval"]))
    result = dict(split=args.split, frames=len(ids), classes=args.classes, results=entries, times_s=times)
    if boot is not None:
        result["bootstrap"] = boot
    if per_drive is not None:
        result["per_drive"] = per_drive
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(result, fh, indent=1)
    return result


if __name__ == "__main__":
    main(sys.argv[1:])
