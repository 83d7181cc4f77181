"""Training-time augmentation of labelled KITTI frames: the reference's PointAugmentor
(mmdet/core/point_cloud/point_augmentor.py) as its prepare_train_img applies it (mmdet/datasets/kitti.py:181-256),
with the per-point work and the noise search on the GPU (csrc/augment.cu).

    python -m sassd_b200.augment CONFIG --data-root R [--split train] [--lidar velodyne|velodyne_reduced] [--seed S]
                                 [--batch B] [--frames K] [--out DIR] [--checkpoint CKPT]

With the config's data.train.with_plane, the driver also reads each frame's training/planes/%06d.txt (read_plane).

Per frame, in order, the host makes the reference's draws on ``rng`` (a np.random.RandomState; numpy's global state by
default): the database picks of each class's sampler (and the shuffle when a sampler wraps), the location and rotation
noise of every selected box ([N, 100, 3] normal, then [N, 100] uniform over ``global_rot_range``), the flip choice, the
global rotation and the scaling.  No draw depends on a GPU result, so a batch is drawn first and then launched, with
one synchronisation at the end.  The sampler's collision filter, the box corners and planes, and the box transforms
are small float32 / float64 numpy work on the host, in the reference's dtypes.

Semantics kept from the reference, as it runs with numba compiled:
  * box collisions count a box fully inside another (the compiled ``ret[i, j] is True`` checks);
  * the per-object rotation noise is drawn over ``global_rot_range``; a box with no collision-free try still takes the
    -centre, +centre round trip;
  * the per-class sample count is taken on the raw names, before Van becomes Car, and sampled boxes avoid every
    non-DontCare box;
  * the point masks are taken on the pasted cloud against the selected boxes before noise, in float32 planes;
  * rotations round as numpy's float32 matmul: out_k = fma(z, R2k, fma(y, R1k, fma(x, R0k, +0))).
A frame with no box left after the range filter is reported through the keep mask; the caller picks a replacement.
The reference draws that replacement inside the stream with np.random.choice, so a seeded stream with a rejected frame
differs from the reference's after that frame.  NaN coordinates come out NaN, with the device's NaN bits.

Road planes (the reference's ``with_plane``; ``augment(road_planes=, calibs=)``): once a frame's records are picked,
their boxes move vertically onto its road plane in float64 (plane_shift, the reference's sample_all); the moved float32
boxes replace the database boxes everywhere after the sampler's collision filter, and the records' points move by the
same height on the device, rounded after the centre add and again after the move.  No draw changes.
"""
import argparse
import ctypes
import ctypes.util
import os
import pickle
import sys
import time

import numpy as np

from .create_data import _CORNER_NORM
from .frustum import corner_planes

NUM_TRY = 100
DEFAULT_RANGE = (0.0, -40.0, -3.0, 70.4, 40.0, 1.0)      # the shipped configs' point_cloud_range
_SQUARE = np.array([[-0.5, -0.5], [-0.5, 0.5], [0.5, 0.5], [0.5, -0.5]])   # corners_nd(2-D, origin 0.5), clockwise

_libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
for _f in ("sinf", "cosf"):
    getattr(_libm, _f).restype = ctypes.c_float
    getattr(_libm, _f).argtypes = [ctypes.c_float]


# ---------------------------------------------------------------------------------------------------- host geometry
def bev_corners(centres, dims, angles):
    """[N,2], [N,2], [N] -> clockwise BEV corners [N,4,2] in the inputs' dtype (center_to_corner_box2d)."""
    corners = dims.reshape(-1, 1, 2) * _SQUARE.astype(dims.dtype).reshape(1, 4, 2)
    s, c = np.sin(angles), np.cos(angles)
    corners = np.einsum("aij,jka->aik", corners, np.stack([[c, -s], [s, c]]))
    corners += centres.reshape(-1, 1, 2)
    return corners


def box_corners3d(boxes):
    """LiDAR boxes [N,7] -> corners [N,8,3] in the boxes' dtype (center_to_corner_box3d, origin (0.5, 0.5, 0))."""
    corners = boxes[:, 3:6].reshape(-1, 1, 3) * _CORNER_NORM.astype(boxes.dtype).reshape(1, 8, 3)
    s, c = np.sin(boxes[:, 6]), np.cos(boxes[:, 6])
    z, o = np.zeros_like(c), np.ones_like(c)
    corners = np.einsum("aij,jka->aik", corners, np.stack([[c, -s, z], [s, c, z], [z, z, o]]))
    corners += boxes[:, :3].reshape(-1, 1, 3)
    return corners


def box_planes32(boxes):
    """float32 LiDAR boxes [N,7] -> float32 planes [N,6,4] (n, d), the reference's points_in_rbbox planes: the cross
    products and dot products run in float32, as the reference's surface_equ_3d_jit does on float32 corners."""
    planes = corner_planes(box_corners3d(np.asarray(boxes, np.float32).reshape(-1, 7)))
    assert planes.dtype == np.float32, "the planes of float32 boxes must be computed in float32"
    return planes


def box_collision(boxes, qboxes):
    """BEV corners [N,4,2], [K,4,2] -> [N,K] bool: box_collision_test as numba compiles it, element for element in the
    inputs' dtype: standup boxes overlap, and two edges cross or one box is strictly inside the other."""
    n, k = boxes.shape[0], qboxes.shape[0]
    if n == 0 or k == 0:
        return np.zeros((n, k), bool)
    bs = np.concatenate([boxes.min(1), boxes.max(1)], 1)
    qs = np.concatenate([qboxes.min(1), qboxes.max(1)], 1)
    iw = np.minimum(bs[:, None, 2], qs[None, :, 2]) - np.maximum(bs[:, None, 0], qs[None, :, 0])
    ih = np.minimum(bs[:, None, 3], qs[None, :, 3]) - np.maximum(bs[:, None, 1], qs[None, :, 1])
    A = boxes[:, None, :, None, :]
    B = np.roll(boxes, -1, axis=1)[:, None, :, None, :]
    C = qboxes[None, :, None, :, :]
    D = np.roll(qboxes, -1, axis=1)[None, :, None, :, :]

    def gt(p, q, r):     # (q.y - p.y) * (r.x - p.x) > (r.y - p.y) * (q.x - p.x)
        return (q[..., 1] - p[..., 1]) * (r[..., 0] - p[..., 0]) > (r[..., 1] - p[..., 1]) * (q[..., 0] - p[..., 0])
    edge = ((gt(A, D, C) != gt(B, D, C)) & (gt(A, C, B) != gt(A, D, B))).any((2, 3))

    def inside(a, q):    # every corner of q strictly inside a: a [N,1,4,1,2], q [1,K,1,4,2]
        vec = -(a - np.roll(a, -1, axis=2))
        cross = vec[..., 1] * (a[..., 0] - q[..., 0])
        cross = cross - vec[..., 0] * (a[..., 1] - q[..., 1])
        return (cross < 0).all((2, 3))
    q_in_b = inside(boxes[:, None, :, None, :], qboxes[None, :, None, :, :])
    b_in_q = inside(qboxes[:, None, :, None, :], boxes[None, :, None, :, :]).T
    return (iw > 0) & (ih > 0) & (edge | q_in_b | b_in_q)


def sampler_filter(avoid, sp_boxes):
    """Indices of the sampled boxes [S,7] kept by the reference's sampler: BEV collisions against ``avoid`` [G,7] and
    each other, then a greedy pass in sample order (PointAugmentor.sample)."""
    num_gt = avoid.shape[0]
    boxes = np.concatenate([avoid, sp_boxes], 0)
    sp = boxes[num_gt:]
    total = np.concatenate([bev_corners(avoid[:, 0:2], avoid[:, 3:5], avoid[:, 6]),
                            bev_corners(sp[:, 0:2], sp[:, 3:5], sp[:, 6])], 0)
    coll = box_collision(total, total)
    coll[np.arange(len(total)), np.arange(len(total))] = False
    valid = []
    for i in range(num_gt, len(total)):
        if coll[i].any():
            coll[i] = False
            coll[:, i] = False
        else:
            valid.append(i - num_gt)
    return valid


def in_range(boxes, limit_range):
    """filter_gt_box_outside_range: a box is kept when one of its BEV corners is strictly inside the range's
    rectangle (the corners widened to float64)."""
    lo, hi = np.asarray(limit_range, np.float64)[:2], np.asarray(limit_range, np.float64)[2:]
    poly = lo + (hi - lo) * np.array([[0.0, 0.0], [0.0, 1.0], [1.0, 1.0], [1.0, 0.0]])
    vec = poly - poly[[3, 0, 1, 2]]
    pts = bev_corners(boxes[:, [0, 1]], boxes[:, [3, 4]], boxes[:, 6]).reshape(-1, 1, 2).astype(np.float64)
    cross = vec[:, 1] * (poly[:, 0] - pts[..., 0])
    cross = cross - vec[:, 0] * (poly[:, 1] - pts[..., 1])
    return (cross < 0).all(1).reshape(-1, 4).any(1)


def rotation_z32(angle):
    """float32 rotation_points_single_angle matrix (row vectors, about z)."""
    s, c = np.sin(angle), np.cos(angle)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], dtype=np.float32)


def plane_shift(sampled64, plane, calib):
    """Sampled database boxes [S,7] (their float64 box3d_lidar, in sample order) moved vertically onto the frame's
    road plane (kitti_data.read_plane's float64 (a, b, c, d), rectified camera frame), as the reference's sample_all
    does with road_planes (point_augmentor.py:225-245): each centre goes to the camera frame, takes the plane's height
    there, comes back, and z moves by mv = z - that height.  Returns (boxes [S,7] float32, mv [S] float64); the
    sampled records' points move by -mv after their centre add."""
    from .results import project_rect_to_velo, project_velo_to_rect
    boxes = np.array(sampled64, np.float64).reshape(-1, 7)
    a, b, c, d = np.asarray(plane, np.float64)
    center_cam = project_velo_to_rect(boxes[:, 0:3], calib)
    center_cam[:, 1] = (-d - a * center_cam[:, 0] - c * center_cam[:, 2]) / b
    cur = project_rect_to_velo(center_cam, calib)[:, 2]
    mv = boxes[:, 2] - cur
    boxes[:, 2] -= mv        # not z = cur: z - (z - cur) need not round to cur
    return boxes.astype(np.float32), mv


def check_planes(road_planes, calibs, batch):
    """augment's road_planes / calibs -> per-frame lists (of None without planes): both None, or both one entry per
    frame with each plane 4 finite numbers."""
    if road_planes is None and calibs is None:
        return [None] * batch, [None] * batch
    if road_planes is None or calibs is None:
        raise ValueError("road_planes and calibs go together: pass both or neither")
    road_planes, calibs = list(road_planes), list(calibs)
    if len(road_planes) != batch or len(calibs) != batch:
        raise ValueError("road_planes and calibs need one entry per frame (%d frames; %d planes, %d calibs)"
                         % (batch, len(road_planes), len(calibs)))
    for b, p in enumerate(road_planes):
        p = np.asarray(p)
        if p.shape != (4,) or not np.issubdtype(p.dtype, np.number) or not np.isfinite(p).all():
            raise ValueError("frame %d: a road plane is 4 finite numbers (a, b, c, d), not %r" % (b, p))
    return road_planes, calibs


# ---------------------------------------------------------------------------------------------------- augmentor
class _ClassSampler:
    """The reference's BatchSampler over one class's records: a shuffled index order consumed in runs, reshuffled
    when a run reaches its end."""

    def __init__(self, n, rng):
        self.n, self.rng, self.idx = n, rng, 0
        self.indices = np.arange(n)
        rng.shuffle(self.indices)

    def take(self, num):
        if self.idx + num >= self.n:
            ret = self.indices[self.idx:].copy()
            self.rng.shuffle(self.indices)
            self.idx = 0
        else:
            ret = self.indices[self.idx:self.idx + num].copy()
            self.idx += num
        return ret


class PointAugmentor:
    """The reference's PointAugmentor with its constructor arguments (obj_from_dict builds it from a config's
    ``data.train.augmentor``), plus ``rng`` (np.random.RandomState, numpy's global state by default) and ``device``
    (where the database's points live; None keeps only the host side: ``draw`` and ``finish_boxes``).

    The database records of each sample class are those with num_points_in_gt >= min_num_points and a difficulty
    outside removed_difficulties; their point files are read once into one device buffer [R,4]."""

    def __init__(self, root_path, info_path, sample_classes, min_num_points, sample_max_num, removed_difficulties,
                 gt_rot_range=None, global_rot_range=None, center_noise_std=None, scale_range=None, rng=None,
                 device="cuda", with_plane=False):
        if with_plane:
            raise NotImplementedError("with_plane is a dataset option (data.train.with_plane), not an augmentor "
                                      "argument: pass each frame's road plane and calibration to "
                                      "augment(road_planes=, calibs=)")
        if global_rot_range is None or center_noise_std is None or scale_range is None:
            raise ValueError("global_rot_range, center_noise_std and scale_range are required")
        sample_classes = list(sample_classes)
        if isinstance(min_num_points, int):
            min_num_points = [min_num_points] * len(sample_classes)
        if isinstance(sample_max_num, int):
            sample_max_num = [sample_max_num] * len(sample_classes)
        if not (len(min_num_points) == len(sample_max_num) == len(sample_classes)):
            raise ValueError("min_num_points and sample_max_num need one entry per sample class")
        self.rng = np.random.mtrand._rand if rng is None else rng
        with open(info_path, "rb") as fh:
            infos = pickle.load(fh)
        self.root_path, self.sample_classes = root_path, sample_classes
        self.sample_max_num = [int(v) for v in sample_max_num]
        self.global_rot_range, self.gt_rot_range = list(global_rot_range), gt_rot_range
        self.center_noise_std = list(center_noise_std)
        self.scale_range = list(scale_range)
        self.records, self.class_records, self.samplers = [], [], []
        for cls, mn in zip(sample_classes, min_num_points):
            recs = [r for r in infos.get(cls, []) if r["num_points_in_gt"] >= mn]
            recs = [r for r in recs if r["difficulty"] not in removed_difficulties]
            if not recs:
                raise ValueError("no %s records left in %s after the min_num_points / removed_difficulties filter"
                                 % (cls, info_path))
            self.class_records.append(list(range(len(self.records), len(self.records) + len(recs))))
            self.records += recs
            self.samplers.append(_ClassSampler(len(recs), self.rng))
        self.device = device
        if device is not None:
            self._load_database(device)

    def _load_database(self, device):
        import torch
        from .kitti_data import read_points
        pts = [read_points(os.path.join(self.root_path, r["path"])) for r in self.records]
        self.db_count = np.array([len(p) for p in pts], np.int64)
        self.db_start = np.concatenate([[0], np.cumsum(self.db_count)[:-1]]).astype(np.int64)
        cat = np.concatenate(pts, 0) if pts else np.zeros((0, 4), np.float32)
        self.db = torch.from_numpy(np.ascontiguousarray(cat if len(cat) else np.zeros((1, 4), np.float32))).to(device)

    # -------------------------------------------------------------------------------------------- host, per frame
    def draw(self, gt_boxes, gt_names, class_names, plane=None, calib=None):
        """One frame's host part, in the reference's draw order: gt_boxes [G,7] float32 (every non-DontCare label box,
        LiDAR frame) and their raw names.  Returns a dict: the sampled record ids, the selected boxes (float32, before
        noise), their labels, the noise draws and the frame's flip, rotation and scale.  With the frame's road
        ``plane`` and ``calib``, the sampled boxes are plane_shift's (the collision filter has run on the database
        boxes, as in the reference) and ``mv`` holds each sampled record's height move; otherwise ``mv`` is None."""
        rng = self.rng
        gt_boxes = np.asarray(gt_boxes, np.float32).reshape(-1, 7)
        gt_names = [str(n) for n in gt_names]
        avoid, picked = gt_boxes, []
        for ci, cls in enumerate(self.sample_classes):
            num = int(self.sample_max_num[ci] - np.sum([n == cls for n in gt_names]))
            if num <= 0:
                continue
            recs = [self.class_records[ci][i] for i in self.samplers[ci].take(num)]
            sp = np.stack([self.records[r]["box3d_lidar"] for r in recs], 0)
            valid = [recs[i] for i in sampler_filter(avoid, sp)]
            if valid:
                picked += valid
                avoid = np.concatenate([avoid, np.stack([self.records[r]["box3d_lidar"] for r in valid], 0)], 0)
        sampled = (np.stack([self.records[r]["box3d_lidar"] for r in picked], 0).astype(np.float32) if picked
                   else np.zeros((0, 7), np.float32))
        mv = None
        if plane is not None and picked:
            sampled, mv = plane_shift(np.stack([self.records[r]["box3d_lidar"] for r in picked], 0), plane, calib)
        boxes = np.concatenate([gt_boxes, sampled], 0)
        names = ["Car" if n == "Van" else n for n in gt_names + [self.records[r]["name"] for r in picked]]
        sel = [i for i, n in enumerate(names) if n in class_names]
        boxes = boxes[sel]
        labels = np.array([list(class_names).index(names[i]) + 1 for i in sel], dtype=np.int64)
        n = len(sel)
        loc = rng.normal(scale=np.array(self.center_noise_std, dtype=boxes.dtype), size=[n, NUM_TRY, 3])
        rot = rng.uniform(self.global_rot_range[0], self.global_rot_range[1], size=[n, NUM_TRY])
        flip = bool(rng.choice([False, True], replace=False, p=[0.5, 0.5]))
        angle = rng.uniform(self.global_rot_range[0], self.global_rot_range[1])
        scale = rng.uniform(self.scale_range[0], self.scale_range[1])
        return dict(records=picked, sampled=sampled, mv=mv, boxes=boxes, labels=labels, loc=loc, rot=rot, flip=flip,
                    angle=angle, scale=scale)

    @staticmethod
    def finish_boxes(plan, sel, point_cloud_range=DEFAULT_RANGE):
        """The frame's boxes after the chosen noise (sel [N], -1: none), flip, rotation, scaling, the range filter and
        limit_period: (boxes [M,7] float32, labels [M] int64)."""
        boxes = plan["boxes"].copy()
        n = len(boxes)
        sel = np.asarray(sel).reshape(n)
        ok = sel >= 0
        loc_t, rot_t = np.zeros((n, 3)), np.zeros((n,))
        loc_t[ok] = plan["loc"][ok, sel[ok]]
        rot_t[ok] = plan["rot"][ok, sel[ok]]
        boxes[:, :3] = (boxes[:, :3].astype(np.float64) + loc_t).astype(np.float32)
        boxes[:, 6] = (boxes[:, 6].astype(np.float64) + rot_t).astype(np.float32)
        if plan["flip"]:
            boxes[:, 1] = -boxes[:, 1]
            boxes[:, 6] = -boxes[:, 6] + np.pi
        boxes[:, :3] = boxes[:, :3] @ rotation_z32(plan["angle"])
        boxes[:, 6] += plan["angle"]
        boxes[:, :6] *= plan["scale"]
        r = np.asarray(point_cloud_range, np.float64)
        keep = in_range(boxes, r[[0, 1, 3, 4]]) if n else np.zeros((0,), bool)
        boxes, labels = boxes[keep], plan["labels"][keep]
        boxes[:, 6] = boxes[:, 6] - np.floor(boxes[:, 6] / (2 * np.pi) + 0.5) * (2 * np.pi)
        return boxes, labels

    # -------------------------------------------------------------------------------------------- device, per batch
    def augment(self, points, pt_off, batch, gt_boxes, gt_names, class_names=None, point_cloud_range=DEFAULT_RANGE,
                max_points=None, road_planes=None, calibs=None):
        """points [Ncap,4] f32 and pt_off [batch+1] i32 on the device (frustum_crop's layout); per frame the
        non-DontCare boxes (float32 [G,7], LiDAR frame) and raw KITTI names.  Returns (points [cap,4], pt_off
        [batch+1], boxes list, labels list, keep [batch] bool, sel list): per frame its GT boxes (float32) and labels
        (int64, 1-based over ``class_names``) after the range filter and limit_period, keep false where the reference
        would reject the frame (no box left), and each selected box's chosen noise try (int32, -1: none), in the order
        of the selected boxes before the range filter.  ``max_points`` (default: the input's rows plus every sampled
        row) caps the output rows; overflow raises.

        ``road_planes`` and ``calibs`` (the reference's data.train.with_plane): per frame its road plane
        (kitti_data.read_plane) and its results.Calibration.  The sampled boxes then sit on the frame's road
        (plane_shift) for the scene crop, the noise search, the point masks and the returned boxes, and each sampled
        record's points move by the same height as its box."""
        import torch
        from . import ops
        from .lib import GT_CAP_MAX, raise_on_status
        road_planes, calibs = check_planes(road_planes, calibs, batch)
        if self.device is None:
            raise ValueError("this augmentor was built without a device database")
        class_names = list(self.sample_classes if class_names is None else class_names)
        if len(gt_boxes) != batch or len(gt_names) != batch:
            raise ValueError("gt_boxes and gt_names need one entry per frame")
        dev = points.device
        plans = [self.draw(gt_boxes[b], gt_names[b], class_names, road_planes[b], calibs[b]) for b in range(batch)]
        for p in plans:
            if len(p["boxes"]) > GT_CAP_MAX:
                raise ValueError("a frame has %d boxes after sampling; at most %d are supported"
                                 % (len(p["boxes"]), GT_CAP_MAX))

        def dev_t(a, dtype):
            a = np.ascontiguousarray(a, dtype)
            if a.size == 0:
                a = np.zeros((1,) + a.shape[1:], dtype)
            return torch.from_numpy(a).to(dev, non_blocking=False)

        def offsets(counts):
            return np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)

        # scene crop by the sampled boxes
        samp_off = offsets([len(p["sampled"]) for p in plans])
        samp_planes = np.concatenate([box_planes32(p["sampled"]) for p in plans], 0).reshape(-1, 6, 4)
        kept, kept_off = ops.augment_drop_points(points, pt_off, batch, dev_t(samp_planes, np.float32),
                                                 dev_t(samp_off, np.int32))
        # noise search over the selected boxes
        boxes = np.concatenate([p["boxes"] for p in plans], 0).reshape(-1, 7)
        box_off = offsets([len(p["boxes"]) for p in plans])
        loc = np.concatenate([p["loc"] for p in plans], 0).reshape(-1, NUM_TRY, 3)
        rot = np.concatenate([p["rot"] for p in plans], 0).reshape(-1, NUM_TRY)
        try_trig = np.stack([np.cos(rot), np.sin(rot)], -1).astype(np.float32)
        box_trig = np.array([[_libm.cosf(float(a)), _libm.sinf(float(a))] for a in boxes[:, 6]], np.float32)
        status = torch.zeros((1,), dtype=torch.int32, device=dev)
        d_box_off, d_trig, d_loc = dev_t(box_off, np.int32), dev_t(try_trig, np.float32), dev_t(loc, np.float64)
        if len(boxes):
            sel = ops.augment_noise_search(dev_t(boxes[:, [0, 1, 3, 4, 6]], np.float32), dev_t(box_trig, np.float32),
                                           d_box_off, batch, d_trig, d_loc, status)
        else:
            sel = torch.full((1,), -1, dtype=torch.int32, device=dev)
        # sampled rows, the point pass and the global transforms
        recs = [r for p in plans for r in p["records"]]
        srec_off = offsets([self.db_count[r] for r in recs])
        srow_off = np.concatenate([[0], np.cumsum([sum(self.db_count[r] for r in p["records"]) for p in plans])])
        ctr = np.array([np.asarray(self.records[r]["box3d_lidar"], np.float64)[:3] for r in recs]).reshape(-1, 3)
        tf = np.array([[float(p["flip"]), *rotation_z32(p["angle"])[:2, :2].reshape(-1), np.float32(p["scale"])]
                       for p in plans], np.float32)
        out_cap = int(points.shape[0] + srow_off[-1]) if max_points is None else int(max_points)
        srec_db = torch.from_numpy(np.array([self.db_start[r] for r in recs], np.int32)).to(dev)
        dz = None
        if recs and road_planes[0] is not None:
            dz = dev_t(np.concatenate([p["mv"] for p in plans if p["records"]]), np.float64)
        out, out_off = ops.augment_assemble(
            kept, kept_off, batch, dev_t(srow_off, np.int32), dev_t(srec_off, np.int32), srec_db, dev_t(ctr, np.float64),
            self.db, d_box_off, dev_t(np.concatenate([box_planes32(p["boxes"]) for p in plans], 0).reshape(-1, 6, 4),
                                      np.float32),
            dev_t(boxes[:, :3], np.float32), sel, d_trig, d_loc, dev_t(tf, np.float32), out_cap, status, dz=dz)
        sel_h = sel.cpu().numpy()
        raise_on_status(int(status.cpu()))
        sels = [sel_h[box_off[b]:box_off[b + 1]].copy() for b in range(batch)]
        out_boxes, out_labels = [], []
        for p, sl in zip(plans, sels):
            bx, lb = self.finish_boxes(p, sl, point_cloud_range)
            out_boxes.append(bx)
            out_labels.append(lb)
        keep = np.array([len(bx) > 0 for bx in out_boxes], bool)
        return out, out_off, out_boxes, out_labels, keep, sels


# ---------------------------------------------------------------------------------------------------- driver
def build_augmentor(cfg, data_root, rng=None, device="cuda"):
    """cfg.data.train.augmentor with root_path / info_path under ``data_root``."""
    aug = dict(cfg.data["train"]["augmentor"])
    aug.pop("type", None)
    aug["root_path"] = data_root
    aug["info_path"] = os.path.join(data_root, os.path.basename(aug["info_path"]))
    return PointAugmentor(rng=rng, device=device, **aug)


def main(argv=None):
    ap = argparse.ArgumentParser(prog="python -m sassd_b200.augment", description=__doc__.split("\n\n")[0])
    ap.add_argument("config")
    ap.add_argument("--data-root", required=True)
    ap.add_argument("--split", default="train")
    ap.add_argument("--lidar", default="velodyne", choices=("velodyne", "velodyne_reduced"))
    ap.add_argument("--seed", type=int, default=None)
    ap.add_argument("--batch", type=int, default=1)
    ap.add_argument("--frames", type=int, default=None)
    ap.add_argument("--out", default=None)
    ap.add_argument("--checkpoint", default=None,
                    help="also run the detector's loss_points on the kept frames of every augmented batch and print "
                         "each loss's mean over the batches")
    args = ap.parse_args(argv)
    if args.batch < 1:
        ap.error("--batch must be >= 1")
    import torch
    from . import Config, ops
    from .kitti_data import KittiSplit, Prefetcher, labelled_boxes, read_label, read_plane
    cfg = Config.fromfile(args.config)
    if "train" not in cfg.data:
        ap.error("%s has no data.train section" % args.config)
    with_plane = bool(cfg.data["train"].get("with_plane", False))
    class_names = list(cfg.data["train"].get("class_names", cfg.data["val"]["class_names"]))
    pc_range = cfg.data["train"]["generator"]["point_cloud_range"]
    if args.seed is not None:
        np.random.seed(args.seed)
    aug = build_augmentor(cfg, args.data_root)
    dev = torch.device("cuda")
    model = None
    if args.checkpoint:
        from . import build_from_config
        from .checkpoint import load_params_from_file
        model, _, _ = build_from_config(cfg, device=dev)
        load_params_from_file(model, args.checkpoint)
        model.eval()
        if list(model.class_names) != class_names:
            ap.error("the model's classes %s differ from data.train.class_names %s" % (model.class_names, class_names))
        loss_sum, loss_batches = np.zeros(len(ops.LOSS_KEYS)), 0
    split = KittiSplit(args.data_root, args.split, lidar=args.lidar)
    ids = split.ids[:args.frames] if args.frames is not None else split.ids

    class _Labelled:
        def frame(self, idx):
            pts, meta = split.frame(idx)
            gt = labelled_boxes(read_label(split.path("label_2", idx, "txt")), meta["calib"])
            if with_plane:
                return pts, meta, gt, read_plane(split.path("planes", idx, "txt"))
            return pts, meta, gt

        def pad_frame(self):
            raise AssertionError("frames are not padded")
    batches = [ids[i:i + args.batch] for i in range(0, len(ids), args.batch)]
    pf = Prefetcher(_Labelled(), batches)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
    n_frames, n_kept, t0 = 0, 0, time.perf_counter()
    for bids, pts, metas, gts, *road in pf:
        B = len(bids)
        off = np.concatenate([[0], np.cumsum([len(p) for p in pts])]).astype(np.int32)
        d_pts = torch.from_numpy(np.concatenate(pts, 0) if off[-1] else np.zeros((1, 4), np.float32)).to(dev)
        d_off = torch.from_numpy(off).to(dev)
        if args.lidar == "velodyne":
            planes = np.stack([split.planes(m["calib"], m["img_shape"]) for m in metas])
            d_pts, d_off = ops.frustum_crop(d_pts, d_off, B, torch.from_numpy(planes).to(dev))
        out, out_off, boxes, lbls, keep, _ = aug.augment(
            d_pts, d_off, B, [g[0] for g in gts], [g[1] for g in gts], class_names, pc_range,
            road_planes=road[0] if with_plane else None, calibs=[m["calib"] for m in metas] if with_plane else None)
        n_frames += B
        n_kept += int(keep.sum())
        if args.out or (model is not None and keep.any()):
            o = out_off.cpu().numpy()
            host = out.cpu().numpy()
        if model is not None and keep.any():
            kb = [b for b in range(B) if keep[b]]
            losses = model.loss_points([host[o[b]:o[b + 1]] for b in kb], [boxes[b] for b in kb],
                                       [lbls[b] for b in kb])
            loss_sum += [losses[k] for k in ops.LOSS_KEYS]
            loss_batches += 1
        if args.out:
            for b, idx in enumerate(bids):
                host[o[b]:o[b + 1]].tofile(os.path.join(args.out, "%06d.bin" % idx))
                np.savez(os.path.join(args.out, "%06d.npz" % idx), gt_boxes=boxes[b], gt_labels=lbls[b],
                         keep=keep[b])
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    print("augmented %d frames (%d kept) in %.2f s: %.1f frames/s, read wait %.2f s"
          % (n_frames, n_kept, dt, n_frames / max(dt, 1e-9), pf.wait))
    if model is not None:
        means = loss_sum / max(loss_batches, 1)
        print("losses over %d augmented batches: %s" % (loss_batches, ", ".join(
            "%s %.6f" % (k, v) for k, v in zip(ops.LOSS_KEYS, means))))
    return 0


if __name__ == "__main__":
    sys.exit(main())
