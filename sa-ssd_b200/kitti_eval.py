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

    python -m sassd_b200.kitti_eval --data-root DIR [--split val] --results DIR [DIR ...] [--classes Car ...]
                                    [--r40] [--coco] [--json FILE]

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


def image_box_overlap(boxes, query_boxes, criterion=-1):
    """Axis-aligned 2-D overlap, kitti_eval.py:95-122, vectorised (same expressions per element)."""
    b, q = boxes[:, None, :], query_boxes[None, :, :]
    iw = np.minimum(b[..., 2], q[..., 2]) - np.maximum(b[..., 0], q[..., 0])
    ih = np.minimum(b[..., 3], q[..., 3]) - np.maximum(b[..., 1], q[..., 1])
    area_b = (b[..., 2] - b[..., 0]) * (b[..., 3] - b[..., 1])
    area_q = (q[..., 2] - q[..., 0]) * (q[..., 3] - q[..., 1])
    if criterion == -1:
        ua = area_b + area_q - iw * ih
    elif criterion == 0:
        ua = area_b + 0 * area_q
    elif criterion == 1:
        ua = area_q + 0 * area_b
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
    iw = (np.minimum(boxes[:, None, 1], qboxes[None, :, 1])
          - np.maximum(boxes[:, None, 1] - boxes[:, None, 4], qboxes[None, :, 1] - qboxes[None, :, 4]))
    a1 = (boxes[:, 3] * boxes[:, 4] * boxes[:, 5])[:, None]
    a2 = (qboxes[:, 3] * qboxes[:, 4] * qboxes[:, 5])[None, :]
    inc = iw * rinc
    if criterion == -1:
        ua = a1 + a2 - inc
    elif criterion == 0:
        ua = a1 + 0 * a2
    elif criterion == 1:
        ua = a2 + 0 * a1
    else:
        ua = np.ones_like(inc)
    out = np.zeros(rinc.shape, np.float32)
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
def clean_data(gt_anno, dt_anno, current_class, difficulty):
    """Ignore flags of one frame (kitti_eval.py:39-92): 0 evaluate, 1 ignore, -1 other class."""
    return clean_gt(gt_anno, current_class, difficulty) + (clean_dt(dt_anno, current_class, difficulty),)


def clean_gt(gt_anno, current_class, difficulty):
    """clean_data's GT side: (valid GT count, GT ignore flags, DontCare boxes)."""
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
    ign_gt = np.where((valid == 1) & ~ignore, 0, np.where((valid == 0) | (ignore & (valid == 1)), 1, -1)).astype(np.int32)
    dc = bbox[np.asarray(gt_anno["name"], dtype=str) == "DontCare"] if len(names) else np.zeros((0, 4))
    return int((ign_gt == 0).sum()), ign_gt, dc


def clean_dt(dt_anno, current_class, difficulty):
    """clean_data's detection side: the detections' ignore flags."""
    cls = CLASS_NAMES[current_class].lower()
    dnames = np.char.lower(np.asarray(dt_anno["name"], dtype=str)) if len(dt_anno["name"]) else np.zeros((0,), str)
    dbox = np.asarray(dt_anno["bbox"], np.float64).reshape(-1, 4)
    height = np.abs(dbox[:, 3] - dbox[:, 1])
    return np.where(height < MIN_HEIGHT[difficulty], 1, np.where(dnames == cls, 0, -1)).astype(np.int32)


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

    def __init__(self, gt_annos, current_class, difficulty):
        prep = [clean_gt(g, current_class, difficulty) for g in gt_annos]
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

    def __init__(self, gt, dt_annos, overlaps, current_class, difficulty):
        ign_dt = [clean_dt(d, current_class, difficulty) for d in dt_annos]
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


def eval_class(gt_annos, dt_annos, current_classes, difficultys, metric, min_overlaps, compute_aos=False,
               overlap_fn=None):
    """precision / recall / orientation [class, difficulty, min_overlap, 41] (eval_class_v3, kitti_eval.py:549-657).
    min_overlaps: [num_minoverlap, metric, class]."""
    return eval_class_many(gt_annos, [dt_annos], current_classes, difficultys, metric, min_overlaps, [compute_aos],
                           overlap_fn)[0]


def eval_class_many(gt_annos, dt_sets, current_classes, difficultys, metric, min_overlaps, compute_aos, overlap_fn=None,
                    gt_sides=None):
    """eval_class for each detection set of ``dt_sets`` against the same GT (``compute_aos``: one flag per set): one
    overlap pass for all sets (calculate_overlaps_many) and one GT side per class and difficulty (``gt_sides``:
    {(class, difficulty): _GtSide}, built here when not given)."""
    assert all(len(gt_annos) == len(d) for d in dt_sets)
    overlaps = calculate_overlaps_many(gt_annos, dt_sets, metric, overlap_fn)
    shape = (len(current_classes), len(difficultys), len(min_overlaps), 41)
    out = [dict(recall=np.zeros(shape), precision=np.zeros(shape), orientation=np.zeros(shape)) for _ in dt_sets]
    for m, cls in enumerate(current_classes):
        for l, diff in enumerate(difficultys):
            gt = _GtSide(gt_annos, cls, diff) if gt_sides is None else gt_sides[cls, diff]
            for dt_annos, ov, aos_s, res in zip(dt_sets, overlaps, compute_aos, out):
                packed = _Packed(gt, dt_annos, ov, cls, diff)
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
    aos_table = None
    if any(aos_flags) and total:
        table = np.zeros((total,), np.float64)
        gt_alpha = gt.alpha.cpu().numpy()
        dt_alpha = torch.cat([d.alpha for d in dts]).cpu().numpy()
        _lib.check(_lib.load().sassd_kitti_aos_table(K, F, _p(gt_off), _p(dt_off), _p(ov_off), _p(gt_alpha),
                                                     _p(dt_alpha), _p(table)), "sassd_kitti_aos_table")
        aos_table = up(table)
    # each job's score region: the next power of two of its (class, difficulty)'s valid GT count
    nv = n_valid.cpu().numpy().astype(np.int64)
    region = np.broadcast_to((1 << np.ceil(np.log2(np.maximum(nv, 1))).astype(np.int64))[None, :, :, None, None],
                             (K, C, Dn, 3, M)).reshape(-1)
    score_off = up(_offsets(region, np.int64))
    desc = _lib.KittiEvalDesc(nsets=K, nframes=F, nclass=C, ndiff=Dn, nover=M, max_nd=int(nd.max()) if len(nd) else 0,
                              max_ng=int(ng.max()) if len(ng) else 0)
    keep = dict(t, ign_gt=ign_gt, ign_dt=ign_dt, n_valid=n_valid, score_off=score_off, ov_bbox=ov[0], ov_bev=ov[1],
                ov_3d=ov[2], aos_table=aos_table)
    for name, _ in desc._fields_[7:]:
        setattr(desc, name, keep[name].data_ptr() if keep[name] is not None else None)
    _, n_thresh, pr = ops.kitti_eval_match(desc, len(region), int(region.sum()))
    n_thresh = n_thresh.cpu().numpy().reshape(K, C, Dn, 3, M)
    pr = pr.cpu().numpy().reshape(K, C, Dn, 3, M, 41, 4)
    # precision, recall and AOS of the sampled thresholds and their monotone envelope, as eval_class_many computes them
    past = np.arange(41) >= n_thresh[..., None]
    with np.errstate(divide="ignore", invalid="ignore"):
        recall = pr[..., 0] / (pr[..., 0] + pr[..., 2])
        precision = pr[..., 0] / (pr[..., 0] + pr[..., 1])
        aos = pr[..., 3] / (pr[..., 0] + pr[..., 1])
    out = []
    for m in range(3):
        per_set = []
        for k in range(K):
            res = {}
            for key, a in (("recall", recall), ("precision", precision), ("orientation", aos)):
                v = np.where(past[k, :, :, m], 0.0, a[k, :, :, m])
                if key == "orientation" and not (m == 0 and aos_flags[k]):
                    v = np.zeros_like(v)
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


def eval_many(gt_annos, dt_sets, classes, tables=(11,), overlap_fn=None, difficultys=(0, 1, 2)):
    """Every table of ``tables`` (11 and 40: the official tables at 11 / 40 recall positions; "coco": the COCO-style
    table) for each of the K detection sets of ``dt_sets`` against the same GT.  Returns one dict per set, {table:
    (text, ap)}.  The official and COCO overlap rows form one list of min overlaps, so the overlaps, the GT side and
    the matching run once for all of them; R11 and R40 read the same precision samples.  The GT and each set are a
    list of annotation dicts or an AnnoBlock."""
    tables = tuple(tables)
    if not tables or any(t not in TABLES for t in tables):
        raise ValueError("tables must be among %r, not %r" % (TABLES, tables))
    classes = _class_ids(classes)
    official = any(t in (11, 40) for t in tables)
    rows = ([np.stack([OVERLAP_0_7, OVERLAP_0_5], axis=0)[:, :, classes]] if official else [])
    if "coco" in tables:
        rows.append(coco_min_overlaps(classes))
    min_overlaps = np.concatenate(rows, 0)
    n_off = 2 if official else 0
    aos_flags = [_aos_flag(d) for d in dt_sets]
    diffs = list(difficultys)
    if overlap_fn is None:
        prec = _eval_device(gt_annos, dt_sets, classes, diffs, min_overlaps, aos_flags)
    else:
        gt_annos, dt_sets = _as_annos(gt_annos), [_as_annos(d) for d in dt_sets]
        gt_sides = {(c, d): _GtSide(gt_annos, c, d) for c in classes for d in diffs}
        prec = [eval_class_many(gt_annos, dt_sets, classes, diffs, metric, min_overlaps,
                                aos_flags if metric == 0 else [False] * len(dt_sets), overlap_fn, gt_sides)
                for metric in (0, 1, 2)]
    out = []
    for s, compute_aos in enumerate(aos_flags):
        r0, r1, r2 = (p[s] for p in prec)
        res = {}
        for rp in (t for t in tables if t in (11, 40)):
            get_mAP_n = get_mAP if rp == 11 else get_mAP_R40
            ap = dict(bbox=get_mAP_n(r0["precision"][:, :, :n_off]),
                      aos=get_mAP_n(r0["orientation"][:, :, :n_off]) if compute_aos else None,
                      bev=get_mAP_n(r1["precision"][:, :, :n_off]), d3=get_mAP_n(r2["precision"][:, :, :n_off]))
            res[rp] = (_ap_text(ap, classes, min_overlaps[:n_off], compute_aos, "AP" if rp == 11 else "AP_R40"), ap)
        if "coco" in tables:
            # do_coco_style_eval (kitti_eval.py:711-729): the mean over the ten overlaps of get_mAP_v2
            ap = dict(bbox=get_mAP(r0["precision"][:, :, n_off:]).mean(-1),
                      aos=get_mAP(r0["orientation"][:, :, n_off:]).mean(-1) if compute_aos else None,
                      bev=get_mAP(r1["precision"][:, :, n_off:]).mean(-1),
                      d3=get_mAP(r2["precision"][:, :, n_off:]).mean(-1))
            res["coco"] = (_coco_text(ap, classes, compute_aos), ap)
        out.append(res)
    return out


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


def _coco_text(ap, classes, compute_aos):
    """get_coco_eval_result's table (kitti_eval.py:904-930)."""
    lines = []
    for j, cls in enumerate(classes):
        start, stop, num = COCO_RANGE[cls]
        lines.append("%s coco AP@%.2f:%.2f:%.2f:" % (CLASS_TO_NAME[cls], start, (stop - start) / (num - 1), stop))
        for key, label in (("bbox", "bbox AP"), ("bev", "bev  AP"), ("d3", "3d   AP")) + ((("aos", "aos  AP"),)
                                                                                           if compute_aos else ()):
            lines.append("%s:%.2f, %.2f, %.2f" % (label, ap[key][j, 0], ap[key][j, 1], ap[key][j, 2]))
    return "".join(l + "\n" for l in lines)


def _ap_text(ap, classes, min_overlaps, compute_aos, tag):
    """The official table of official_eval's AP arrays."""
    lines = []
    for j, cls in enumerate(classes):
        for i in range(min_overlaps.shape[0]):
            lines.append("%s %s@%.2f, %.2f, %.2f:" % ((CLASS_TO_NAME[cls], tag) + tuple(min_overlaps[i, :, j])))
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


def report_sets(entries, labels, evs, class_names, noun, log=print, extra=None):
    """Print each evaluated set's tables (``evs``: eval_many's dicts, with table 11) under ``== label ==``, then one
    summary line per set: moderate 3D AP per class at the class's strict overlap (R11, and R40 / COCO when evaluated).
    Each set's texts and AP lists go into its dict of ``entries`` (returned).  ``extra(k, entry)`` may add to set k's
    entry after its tables and returns more summary fields."""
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
        if extra is not None:
            line += extra(k, entry)
        summary.append("  ".join(line))
    log("summary: %d %s (moderate 3D AP)" % (len(labels), noun))
    for line in summary:
        log(line)
    return entries


def eval_dirs(label_dir, result_dirs, ids, classes, tables=(11,), times=None):
    """Every table of ``tables`` for each directory of KITTI result files in ``result_dirs`` against the label files
    of ``label_dir``, over the frames ``ids``: the GT is read once, every directory is read and parsed on the device
    (read_block), and one eval_many evaluates them all.  Returns eval_many's list, one dict per directory.
    ``times``: a dict whose "read", "parse" and "eval" entries accumulate seconds."""
    times = {} if times is None else times
    gt = read_block(label_dir, ids, times=times)
    dts = [read_block(d, ids, times=times) for d in result_dirs]
    t0 = time.perf_counter()
    out = eval_many(gt, dts, classes, tables)
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
    args = p.parse_args(argv)
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


def main(argv=None, log=print):
    """Evaluate directories of KITTI result files against a split's labels (SECOND's kitti-object-eval-python):

    python -m sassd_b200.kitti_eval --data-root DIR [--split val] --results DIR [DIR ...]
                                    [--classes Car Pedestrian Cyclist] [--r40] [--coco] [--json FILE]

    The labels are ``training/label_2/%06d.txt`` and the frames those of ``ImageSets/<split>.txt``; files a result
    directory holds beyond them are ignored.  Every file is read into pinned memory, copied to the device once and
    parsed there (read_block), and all directories are evaluated in one pass (eval_many) on the device.  Prints each
    directory's tables under ``== DIR ==``, one summary line per directory and the seconds spent reading, parsing and
    evaluating.  Returns the result dict that ``--json`` writes."""
    from .kitti_data import read_split
    args = parse_args(argv)
    ids = read_split(args.data_root, args.split)
    tables = (11,) + ((40,) if args.r40 else ()) + (("coco",) if args.coco else ())
    times = {}
    evs = eval_dirs(os.path.join(args.data_root, "training", "label_2"), args.results, ids, args.classes, tables, times)
    entries = report_sets([dict(dir=d) for d in args.results], args.results, evs, args.classes, "directories", log)
    log("frames: %d, directories: %d, read %.3f s, parse %.3f s, evaluate %.3f s" % (
        len(ids), len(args.results), times["read"], times["parse"], times["eval"]))
    result = dict(split=args.split, frames=len(ids), classes=args.classes, results=entries, times_s=times)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(result, fh, indent=1)
    return result


if __name__ == "__main__":
    main(sys.argv[1:])
