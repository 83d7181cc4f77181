"""Prepare a KITTI root for training and evaluation (the reference's tools/create_data.py), with the point tests on
the GPU:

    python -m sassd_b200.create_data --data-root data/kitti [--db-split train|trainval] [--classes Car ...]
                                     [--batch 16] [--workers 4] [--max-points 131072]

Every frame of ``ImageSets/{train,val,test}.txt`` is read once (full sweep, calibration, PNG header and, under
``training/``, its label) by kitti_data.Prefetcher's reader threads.  Each batch of full sweeps is cropped to the
camera frustum (ops.frustum_crop) and the cropped points are tested against every labelled object's box and gathered
per box (ops.points_in_rbboxes), in one pass that writes:

  * ``kitti_infos_{train,val,trainval,test}.pkl``: the reference's get_kitti_image_info(velodyne=True, calib=True,
    extend_matrix=True, relative_path=True) with add_difficulty_to_annos and _calculate_num_points_in_gt
    (create_data.py:16-104, kitti_common.py:124-212, 476-518): the same keys, dtypes, values and frame order, the
    image shape from the PNG header, num_points_in_gt int32 with -1 for DontCare, trainval = train + val;
  * ``training|testing/velodyne_reduced/%06d.bin``: the cropped sweeps, byte for byte _create_reduced_point_cloud's
    (create_data.py:107-165);
  * ``gt_database/{image_idx}_{name}_{gt_idx}.bin`` for every object that is not DontCare in the ``--db-split``
    frames (its points relative to the box centre), and ``kitti_dbinfos_<db-split>.pkl`` with one record per object of
    ``--classes`` (create_groundtruth_database, create_data.py:168-272): name, path, image_idx, gt_idx, box3d_lidar,
    num_points_in_gt, difficulty, group_id (a counter over the records in frame order) and score.

The default ``--db-split train`` is the database the shipped configs read (``augmentor.info_path``); the reference's
own ``__main__`` writes ``trainval``.  File writes go to a small thread pool.  The output does not depend on
``--batch`` or ``--workers``.

Host geometry, in float64 and bit for bit the reference's: box_camera_to_lidar of anno_to_rbboxes (geometry.py:36-48),
the box corners of center_to_corner_box3d with origin (0.5, 0.5, 0) rotated about z (geometry.py:289-403), and the
faces' planes of corner_to_surfaces_3d + surface_equ_3d_jit (frustum.corner_planes).
"""
import argparse
import os
import pickle
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

# get_class_to_label_map's order (tools/kitti_common.py:222-234)
KITTI_CLASSES = ("Car", "Pedestrian", "Cyclist", "Van", "Person_sitting", "Truck", "Tram", "Misc", "DontCare")
SPLITS = ("train", "val", "test")

# corners_nd(dims, origin=(0.5, 0.5, 0)) per corner, in the reference's corner order: x bit, then (y, z) bits
# (0,0), (0,1), (1,1), (1,0) for each x
_CORNER_NORM = np.array([[x, y, z] for x in (0, 1) for (y, z) in ((0, 0), (0, 1), (1, 1), (1, 0))],
                        np.float64) - np.array([0.5, 0.5, 0.0])


# ---------------------------------------------------------------------------------------------------- host geometry
def lidar_boxes(annos, r0_rect, tr_velo_to_cam):
    """The non-DontCare objects of a label annotation (kitti_data.read_label) as LiDAR boxes [N, 7] float64 (x, y, z,
    w, l, h, ry): camera location through (R0_rect Tr_velo_to_cam)^-1 (4x4 matrices), dimensions l, h, w -> w, l, h."""
    n_obj = int(np.sum(np.asarray(annos["index"]) >= 0))
    loc = np.asarray(annos["location"]).reshape(-1, 3)[:n_obj]
    dims = np.asarray(annos["dimensions"]).reshape(-1, 3)[:n_obj]
    rot = np.asarray(annos["rotation_y"]).reshape(-1)[:n_obj]
    cam = np.concatenate([loc, np.ones((n_obj, 1))], axis=1)
    xyz = (cam @ np.linalg.inv((r0_rect @ tr_velo_to_cam).T))[:, :3]
    return np.concatenate([xyz, dims[:, 2:3], dims[:, 0:1], dims[:, 1:2], rot[:, None]], axis=1)


def box_corners(boxes):
    """LiDAR boxes [N, 7] -> corners [N, 8, 3]: the box of size (w, l, h) with its bottom centre at the origin,
    rotated by ry about z, moved to (x, y, z)."""
    boxes = np.asarray(boxes, np.float64).reshape(-1, 7)
    local = boxes[:, None, 3:6] * _CORNER_NORM[None]
    c, s = np.cos(boxes[:, 6])[:, None], np.sin(boxes[:, 6])[:, None]
    x, y, z = local[..., 0], local[..., 1], local[..., 2]
    rotated = np.stack([x * c + y * s, x * -s + y * c, z], axis=-1)
    return rotated + boxes[:, None, :3]


def box_planes(boxes):
    """LiDAR boxes [N, 7] -> planes [N, 6, 4] float64 (n.x, n.y, n.z, d), normals pointing inside: a point is in box
    i when n.p + d < 0 for its six faces (the reference's points_in_rbbox)."""
    from .frustum import corner_planes
    return corner_planes(box_corners(boxes))


def add_difficulty(annos):
    """annos["difficulty"] int32: 0 easy, 1 moderate, 2 hard, -1 none, from the 2D box height, occlusion and
    truncation (add_difficulty_to_annos: a level needs height > 40 / 25 / 25 px, occlusion <= 0 / 1 / 2 and
    truncation <= 0.15 / 0.3 / 0.5)."""
    bbox = np.asarray(annos["bbox"]).reshape(-1, 4)
    height = bbox[:, 3] - bbox[:, 1]
    occ, trunc = np.asarray(annos["occluded"]), np.asarray(annos["truncated"])
    levels = [~((occ > o) | (height <= h) | (trunc > t)) for o, h, t in ((0, 40, 0.15), (1, 25, 0.3), (2, 25, 0.5))]
    easy, moderate, hard = levels
    diff = np.full(len(bbox), -1, np.int32)
    diff[hard ^ moderate] = 2
    diff[easy ^ moderate] = 1
    diff[easy] = 0
    annos["difficulty"] = diff
    return annos


def num_points_in_gt(annos, counts):
    """annos["num_points_in_gt"] int32: the member counts of the non-DontCare objects, -1 for the DontCare rows."""
    n_ignored = len(annos["name"]) - len(counts)
    annos["num_points_in_gt"] = np.concatenate([counts, -np.ones([n_ignored])]).astype(np.int32)
    return annos


def _ext4(m):
    """A 3x4 or 3x3 matrix as the reference's extend_matrix 4x4: last row (0, 0, 0, 1), zeros beside a 3x3."""
    out = np.zeros((4, 4))
    out[3, 3] = 1.0
    out[:3, :m.shape[1]] = m
    return out


def calib_info(path):
    """``calib/%06d.txt`` -> the info's calibration entries, 4x4 float64: P0-P3, R0_rect, Tr_velo_to_cam,
    Tr_imu_to_velo."""
    from .results import Calibration
    raw = Calibration.read_calib_file(path)
    out = {"calib/P%d" % i: _ext4(raw["P%d" % i].reshape(3, 4)) for i in range(4)}
    out["calib/R0_rect"] = _ext4(raw["R0_rect"].reshape(3, 3))
    out["calib/Tr_velo_to_cam"] = _ext4(raw["Tr_velo_to_cam"].reshape(3, 4))
    out["calib/Tr_imu_to_velo"] = _ext4(raw["Tr_imu_to_velo"].reshape(3, 4))
    return out


def frame_info(root, idx, training):
    """One frame's info dict without num_points_in_gt, and its full sweep: (info, points [N, 4] float32)."""
    from .kitti_data import png_shape, read_label, read_points
    sub = "training" if training else "testing"
    rel = lambda kind, ext: "%s/%s/%06d.%s" % (sub, kind, idx, ext)     # noqa: E731
    info = {"image_idx": idx, "pointcloud_num_features": 4, "velodyne_path": rel("velodyne", "bin"),
            "img_path": rel("image_2", "png")}
    info["img_shape"] = np.array(png_shape(os.path.join(root, info["img_path"]))[:2], dtype=np.int32)
    info.update(calib_info(os.path.join(root, rel("calib", "txt"))))
    if training:
        info["annos"] = add_difficulty(read_label(os.path.join(root, rel("label_2", "txt"))))
    return info, read_points(os.path.join(root, info["velodyne_path"]))


# ---------------------------------------------------------------------------------------------------- driver
class _Frames:
    """What kitti_data.Prefetcher reads: frame keys (split, idx) -> (info, full sweep, LiDAR boxes)."""

    def __init__(self, root):
        self.root = root

    def frame(self, key):
        split, idx = key
        info, points = frame_info(self.root, idx, split != "test")
        boxes = None
        if "annos" in info:
            boxes = lidar_boxes(info["annos"], info["calib/R0_rect"], info["calib/Tr_velo_to_cam"])
        return info, points, boxes

    def pad_frame(self):
        return None, np.zeros((0, 4), np.float32), None


def parse_args(argv=None):
    p = argparse.ArgumentParser(prog="python -m sassd_b200.create_data", description=__doc__.split("\n\n")[0])
    p.add_argument("--data-root", required=True, help="KITTI root holding ImageSets/, training/ and testing/")
    p.add_argument("--db-split", default="train", choices=("train", "trainval"),
                   help="frames of the ground-truth database (default train, the configs' augmentor.info_path)")
    p.add_argument("--classes", nargs="+", default=None,
                   help="classes that get database records (default: every KITTI class but DontCare)")
    p.add_argument("--batch", type=int, default=16, help="frames per GPU batch")
    p.add_argument("--workers", type=int, default=4, help="reader threads")
    p.add_argument("--max-points", type=int, default=131072, help="points per full sweep the device buffers hold")
    args = p.parse_args(argv)
    if args.batch < 1 or args.batch > 256:
        p.error("--batch must be in 1..256")
    if args.workers < 1:
        p.error("--workers must be positive")
    if args.max_points < 1:
        p.error("--max-points must be positive")
    for split in SPLITS:
        path = os.path.join(args.data_root, "ImageSets", split + ".txt")
        if not os.path.isfile(path):
            p.error("%s not found" % path)
    if args.classes is None:
        args.classes = [c for c in KITTI_CLASSES if c != "DontCare"]
    bad = [c for c in args.classes if c not in KITTI_CLASSES or c == "DontCare"]
    if bad:
        p.error("unknown --classes %s (KITTI classes: %s)" % (bad, ", ".join(KITTI_CLASSES[:-1])))
    return args


class _GpuBatch:
    """Device buffers for one batch and the two kernels: frustum crop, then points in the frames' boxes."""

    def __init__(self, batch, max_points, device):
        import torch
        from . import ops
        self.torch, self.ops = torch, ops
        self.batch, self.max_points, self.device = batch, max_points, device
        self.points = torch.zeros((batch * max_points, 4), dtype=torch.float32, device=device)
        self.ws = ops.Workspace()

    def run(self, points, planes, boxes):
        """points: per frame [N, 4] float32; planes [B, 6, 4]; boxes: per frame LiDAR boxes [G, 7] or None.
        Returns per frame (cropped points [M, 4], box counts [G], gathered rows per box)."""
        from . import lib
        torch, B = self.torch, len(points)
        counts = [len(p) for p in points]
        off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
        if off[-1]:
            self.points[:off[-1]].copy_(torch.from_numpy(np.concatenate(points, 0)))
        d_off = torch.from_numpy(off).to(self.device)
        d_planes = torch.from_numpy(np.ascontiguousarray(planes, np.float64)).to(self.device)
        crop, crop_off = self.ops.frustum_crop(self.points[:max(int(off[-1]), 1)], d_off, B, d_planes, ws=self.ws)

        nbox = np.array([0 if b is None else len(b) for b in boxes], np.int32)
        box_cap = max(1, int(nbox.max()))
        if box_cap > lib.GT_CAP_MAX:
            raise ValueError("a frame has %d labelled objects; at most %d are supported" % (box_cap, lib.GT_CAP_MAX))
        bplanes = np.zeros((B, box_cap, 6, 4), np.float64)
        centres = np.zeros((B, box_cap, 3), np.float64)
        for b, bx in enumerate(boxes):
            if bx is not None and len(bx):
                bplanes[b, :len(bx)] = box_planes(bx)
                centres[b, :len(bx)] = bx[:, :3]
        d_bplanes = torch.from_numpy(bplanes).to(self.device)
        d_centres = torch.from_numpy(centres).to(self.device)
        d_nbox = torch.from_numpy(nbox).to(self.device)
        gather_cap = max(int(off[-1]), 1)
        while True:
            cnt, seg_off, gathered, status = self.ops.points_in_rbboxes(crop, crop_off, B, d_bplanes, d_centres, d_nbox,
                                                                        gather_cap, ws=self.ws)
            word, total = int(status.item()), int(seg_off[-1].item())
            if word & ~lib.GATHER_CAP or total <= gather_cap:
                lib.raise_on_status(word)
                break
            gather_cap = total      # boxes overlap: more rows than points; the counts are exact, run again to fit
        crop_off = crop_off.cpu().numpy()
        crop = crop[:int(crop_off[-1])].cpu().numpy()
        cnt, seg_off = cnt.cpu().numpy(), seg_off.cpu().numpy()
        gathered = gathered[:total].cpu().numpy()
        out = []
        for b in range(B):
            g = 0 if boxes[b] is None else len(boxes[b])
            segs = [gathered[seg_off[b * box_cap + j]:seg_off[b * box_cap + j + 1]] for j in range(g)]
            out.append((crop[crop_off[b]:crop_off[b + 1]], cnt[b, :g], segs))
        return out


def create_data(root, db_split="train", classes=None, batch=16, workers=4, max_points=131072, device="cuda:0",
                log=print):
    """Write the infos, reduced clouds and GT database of the KITTI root ``root`` (see the module docstring).
    Returns timings: frames, seconds, read_wait, write_wait."""
    from .kitti_data import PlaneCache, Prefetcher, padded_batches, read_split
    from .results import Calibration
    classes = [c for c in KITTI_CLASSES if c != "DontCare"] if classes is None else list(classes)
    ids = {s: read_split(root, s) for s in SPLITS}
    db_splits = ("train",) if db_split == "train" else ("train", "val")
    keys = [(s, i) for s in SPLITS for i in ids[s]]
    for sub, splits in (("training", ("train", "val")), ("testing", ("test",))):
        if any(ids[s] for s in splits):
            os.makedirs(os.path.join(root, sub, "velodyne_reduced"), exist_ok=True)
    db_dir = os.path.join(root, "gt_database")
    os.makedirs(db_dir, exist_ok=True)

    planes = PlaneCache()
    gpu = _GpuBatch(batch, max_points, device)
    infos = {s: [] for s in SPLITS}
    dbinfos = {c: [] for c in classes}
    group = 0
    writes, write_wait = [], 0.0
    t0 = time.perf_counter()
    reader = Prefetcher(_Frames(root), padded_batches(keys, batch), depth=4, workers=workers)
    with ThreadPoolExecutor(max_workers=4) as writer:
        for bkeys, frame_infos, points, boxes in reader:
            for k, p in zip(bkeys, points):
                if k is not None and len(p) > max_points:
                    raise ValueError("frame %s has %d points; --max-points is %d" % (k, len(p), max_points))
            fplanes = np.stack([planes(Calibration({"P2": inf["calib/P2"][:3], "Tr_velo_to_cam":
                                                    inf["calib/Tr_velo_to_cam"][:3], "R0_rect": inf["calib/R0_rect"][:3, :3]}),
                                       inf["img_shape"]) if inf is not None else np.zeros((6, 4))
                                for inf in frame_infos])
            results = gpu.run(points, fplanes, boxes)
            t = time.perf_counter()
            for w in writes:
                w.result()
            write_wait += time.perf_counter() - t
            writes = []
            for key, info, box, (reduced, counts, segs) in zip(bkeys, frame_infos, boxes, results):
                if key is None:
                    continue
                split, idx = key
                sub = "testing" if split == "test" else "training"
                writes.append(writer.submit(reduced.tofile, os.path.join(root, sub, "velodyne_reduced", "%06d.bin" % idx)))
                infos[split].append(info)
                if "annos" not in info:
                    continue
                annos = num_points_in_gt(info["annos"], counts)
                if split not in db_splits:
                    continue
                group_of = {}
                for i in range(len(counts)):
                    name, gt_idx = annos["name"][i], annos["index"][i]
                    filename = "%d_%s_%d.bin" % (idx, name, gt_idx)
                    writes.append(writer.submit(segs[i].tofile, os.path.join(db_dir, filename)))
                    if name not in dbinfos:
                        continue
                    gid = annos["group_ids"][i]
                    if gid not in group_of:
                        group_of[gid] = group
                        group += 1
                    dbinfos[name].append({"name": name, "path": "gt_database/" + filename, "image_idx": idx,
                                          "gt_idx": gt_idx, "box3d_lidar": box[i], "num_points_in_gt": len(segs[i]),
                                          "difficulty": annos["difficulty"][i], "group_id": group_of[gid],
                                          "score": annos["score"][i]})
        t = time.perf_counter()
        for w in writes:
            w.result()
        write_wait += time.perf_counter() - t
    infos["trainval"] = infos["train"] + infos["val"]
    for s in ("train", "val", "trainval", "test"):
        with open(os.path.join(root, "kitti_infos_%s.pkl" % s), "wb") as fh:
            pickle.dump(infos[s], fh)
    with open(os.path.join(root, "kitti_dbinfos_%s.pkl" % db_split), "wb") as fh:
        pickle.dump(dbinfos, fh)
    seconds = time.perf_counter() - t0
    for c, v in dbinfos.items():
        log("%d %s database records" % (len(v), c))
    log("%d frames in %.2f s: %.1f frames/s (read wait %.2f s, write wait %.2f s)" % (
        len(keys), seconds, len(keys) / max(seconds, 1e-9), reader.wait, write_wait))
    return dict(frames=len(keys), seconds=seconds, read_wait=reader.wait, write_wait=write_wait)


def main(argv=None):
    args = parse_args(argv)
    create_data(args.data_root, db_split=args.db_split, classes=args.classes, batch=args.batch, workers=args.workers,
                max_points=args.max_points)
    return 0


if __name__ == "__main__":
    sys.exit(main())
