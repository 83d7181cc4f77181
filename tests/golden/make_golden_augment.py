"""Generate tests/golden/augment.npz with the REFERENCE's own PointAugmentor (mmdet/core/point_cloud/point_augmentor.py)
and the augmentation part of KittiLiDAR.prepare_train_img (mmdet/datasets/kitti.py:181-256), on the synthetic KITTI
root of tests/kitti_root.py, in the build container.

    python tests/golden/make_golden_augment.py          # writes the fixture
    python tests/golden/make_golden_augment.py --time   # the reference's CPU time per frame instead (no fixture)

numba is COMPILED here, as the reference trains (box_collision_test's `is True` / `is False` checks only behave as
written when compiled).  The functions numba 0.65 cannot compile in nopython mode (the object-mode
points_in_convex_polygon_3d_jit, surface_equ_3d_jit, corner_to_surfaces_3d and points_in_convex_polygon_jit) run as
their .py_func, which is the same float32 / float64 scalar arithmetic.  The root's info files, reduced clouds and GT
database come from the reference's create_data.  A frame without a non-DontCare box gives the augmentor a [0, 7] box
array (the reference's 1-D empty array fails to index).

Stored, per (config, seed) run over the train frames in ImageSets order, read as velodyne_reduced:
  * the draws: sha256 of the location and rotation noise, the flip, rotation angle and scale;
  * the sampled records (database paths), the chosen noise index per box;
  * the final GT boxes and labels, the keep flag, the sha256 of the augmented cloud; two clouds in full;
and adversarial cases: box collision tests (contained, identical, edge- and corner-touching boxes), a noise search in
which every try fails, and boundary points (face points with their 1-ulp neighbours, non-finite points) with their
float32 points_in_rbbox masks.
"""
import hashlib
import os
import shutil
import struct
import sys
import tempfile
import time
import types

import numpy as np
import numpy.ma  # noqa: F401  (numba imports it on first use; before make_golden shims np.bool)

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from make_golden import import_reference_mmdet  # noqa: E402
from tests import kitti_root as K  # noqa: E402

CONFIGS = {
    "car": dict(sample_classes=["Car"], min_num_points=[5], sample_max_num=[15], class_names=["Car"]),
    # multi_cfg's classes and counts; the synthetic root has few small objects with 5 points or more, so the
    # Pedestrian and Cyclist thresholds are lowered to keep a record of each
    "multi": dict(sample_classes=["Car", "Pedestrian", "Cyclist"], min_num_points=[5, 0, 0],
                  sample_max_num=[15, 10, 10], class_names=["Car", "Pedestrian", "Cyclist"]),
}
COMMON = dict(removed_difficulties=[-1], global_rot_range=[-0.78539816, 0.78539816],
              gt_rot_range=[-0.78539816, 0.78539816], center_noise_std=[1., 1., .5], scale_range=[0.95, 1.05])
SEEDS = (0, 1, 2)
BV_RANGE = np.array([0., -40., -3., 70.4, 40., 1.])[[0, 1, 3, 4]]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _imread(path):
    with open(path, "rb") as fh:
        head = fh.read(26)
    w, h = struct.unpack(">II", head[16:24])
    return np.zeros((h, w, 3), np.uint8)


def reference():
    import_reference_mmdet()
    sys.modules["imageio"].imread = _imread
    tq = types.ModuleType("tqdm")
    tq.tqdm = lambda it, *a, **k: it
    sys.modules["tqdm"] = tq
    from mmdet.core.bbox3d import geometry as G
    from mmdet.core.point_cloud import point_augmentor as PA
    from mmdet.datasets import kitti_utils as KU
    from tools import create_data as C
    for name in ("points_in_convex_polygon_3d_jit", "surface_equ_3d_jit", "corner_to_surfaces_3d",
                 "points_in_convex_polygon_jit"):
        setattr(G, name, getattr(G, name).py_func)
        if hasattr(PA, name):
            setattr(PA, name, getattr(G, name))
    return G, PA, KU, C


def frame_inputs(KU, root, idx):
    objects = KU.read_label(os.path.join(root, "training", "label_2", "%06d.txt" % idx))
    calib = KU.Calibration(os.path.join(root, "training", "calib", "%06d.txt" % idx))
    gt = np.array([o.box3d for o in objects if o.type not in ["DontCare"]], dtype=np.float32).reshape(-1, 7)
    types_ = [o.type for o in objects if o.type not in ["DontCare"]]
    if len(gt):
        gt[:, :3] = KU.project_rect_to_velo(gt[:, :3], calib)
    pts = KU.read_lidar(os.path.join(root, "training", "velodyne_reduced", "%06d.bin" % idx))
    return gt, types_, pts


def augment_frame(G, PA, aug, gt_bboxes, gt_types, points, class_names, rec):
    """prepare_train_img's augmentation part, its range filter and limit_period (kitti.py:180-256)."""
    sampled_gt_boxes, sampled_gt_types, sampled_points = aug.sample_all(gt_bboxes, gt_types, None, None)
    gt_bboxes = np.concatenate([gt_bboxes, sampled_gt_boxes])
    gt_types = gt_types + sampled_gt_types
    masks = G.points_in_rbbox(points, sampled_gt_boxes)
    points = points[np.logical_not(masks.any(-1))]
    points = np.concatenate([sampled_points, points], axis=0)
    gt_types = np.array(['Car' if n == 'Van' else n for n in gt_types])
    selected = [i for i in range(len(gt_types)) if gt_types[i] in class_names]
    gt_bboxes = gt_bboxes[selected, :]
    gt_types = gt_types[selected]
    gt_labels = np.array([class_names.index(n) + 1 for n in gt_types], dtype=np.int64)
    aug.noise_per_object_(gt_bboxes, points, num_try=100)
    gt_bboxes, points = aug.random_flip(gt_bboxes, points)
    gt_bboxes, points = aug.global_rotation(gt_bboxes, points)
    gt_bboxes, points = aug.global_scaling(gt_bboxes, points)
    mask = G.filter_gt_box_outside_range(gt_bboxes, BV_RANGE) if len(gt_bboxes) else np.zeros((0,), bool)
    gt_bboxes, gt_labels = gt_bboxes[mask], gt_labels[mask]
    if len(gt_bboxes):
        gt_bboxes[:, 6] = G.limit_period(gt_bboxes[:, 6], offset=0.5, period=2 * np.pi)
    return gt_bboxes, gt_labels, len(gt_bboxes) > 0, points


def run_stream(G, PA, KU, root, cfg_name, seed, out):
    cfg = CONFIGS[cfg_name]
    np.random.seed(seed)
    aug = PA.PointAugmentor(root, os.path.join(root, "kitti_dbinfos_train.pkl"), cfg["sample_classes"],
                            cfg["min_num_points"], cfg["sample_max_num"], **COMMON)
    rec = {}
    orig_npb, orig_sample = PA.noise_per_box, aug.sample
    draws = {}
    orig_normal, orig_uniform, orig_choice = np.random.normal, np.random.uniform, np.random.choice

    def normal(*a, **k):
        v = orig_normal(*a, **k)
        draws["loc"] = sha(v)
        return v

    def uniform(*a, **k):
        v = orig_uniform(*a, **k)
        draws.setdefault("uniform", []).append(v)
        return v

    def choice(*a, **k):
        v = orig_choice(*a, **k)
        draws["flip"] = bool(v)
        return v

    def npb(*a):
        s = orig_npb(*a)
        rec["sel"] = s.copy()
        return s

    def sample(gt_boxes, num, i):
        v = orig_sample(gt_boxes, num, i)
        rec.setdefault("paths", []).extend(r["path"] for r in v)
        return v
    PA.noise_per_box, aug.sample = npb, sample
    np.random.normal, np.random.uniform, np.random.choice = normal, uniform, choice
    key = "%s_s%d" % (cfg_name, seed)
    try:
        rows = []
        for fi, idx in enumerate(K.TRAIN):
            rec.clear()
            draws.clear()
            gt, types_, pts = frame_inputs(KU, root, idx)
            boxes, labels, keep, cloud = augment_frame(G, PA, aug, gt, types_, pts, cfg["class_names"], rec)
            u = draws["uniform"]
            rows.append(dict(paths=";".join(rec.get("paths", [])), sel=rec["sel"].astype(np.int32), boxes=boxes,
                             labels=labels, keep=keep, cloud=sha(cloud), loc=draws["loc"], rot=sha(u[0]),
                             flip=draws["flip"], angle=float(u[1]), scale=float(u[2])))
            if fi < 2 and seed == SEEDS[0] and cfg_name == "car":
                out["%s_cloud%d" % (key, fi)] = cloud
        out[key + "_paths"] = np.array([r["paths"] for r in rows])
        out[key + "_sel"] = np.concatenate([r["sel"] for r in rows])
        out[key + "_nsel"] = np.array([len(r["sel"]) for r in rows], np.int32)
        out[key + "_boxes"] = np.concatenate([r["boxes"].reshape(-1, 7) for r in rows]).astype(np.float32)
        out[key + "_labels"] = np.concatenate([r["labels"] for r in rows]).astype(np.int64)
        out[key + "_nbox"] = np.array([len(r["labels"]) for r in rows], np.int32)
        out[key + "_keep"] = np.array([r["keep"] for r in rows])
        out[key + "_cloud_sha"] = np.array([r["cloud"] for r in rows])
        out[key + "_loc_sha"] = np.array([r["loc"] for r in rows])
        out[key + "_rot_sha"] = np.array([r["rot"] for r in rows])
        out[key + "_flip"] = np.array([r["flip"] for r in rows])
        out[key + "_angle"] = np.array([r["angle"] for r in rows])
        out[key + "_scale"] = np.array([r["scale"] for r in rows])
        print(key, "kept", out[key + "_keep"].sum(), "boxes", out[key + "_nbox"], "sel", out[key + "_nsel"])
    finally:
        PA.noise_per_box = orig_npb
        np.random.normal, np.random.uniform, np.random.choice = orig_normal, orig_uniform, orig_choice


def adversarial(G, PA, out):
    # collision pairs: contained, identical, edge-touching, corner-touching, crossing, apart
    def sq(cx, cy, s, a=0.0):
        return [cx, cy, s, s, a]
    pairs = [(sq(0, 0, 4), sq(0, 0, 1)), (sq(0, 0, 1), sq(0, 0, 4)), (sq(0, 0, 2), sq(0, 0, 2)),
             (sq(0, 0, 2), sq(2, 0, 2)), (sq(0, 0, 2), sq(2, 2, 2)), (sq(0, 0, 2), sq(1, 1, 2, 0.3)),
             (sq(0, 0, 2), sq(5, 5, 2)), (sq(0, 0, 2, 0.7), sq(0.5, 0, 0.5, 1.1)), (sq(0, 0, 3), sq(1.0, 0, 1.0))]
    a = np.array([p[0] for p in pairs], np.float32)
    b = np.array([p[1] for p in pairs], np.float32)
    ca, cb = G.box2d_to_corner_jit(a), G.box2d_to_corner_jit(b)
    out["coll_a"], out["coll_b"] = ca, cb
    out["coll"] = np.array([G.box_collision_test(ca[i:i + 1], cb[i:i + 1])[0, 0] for i in range(len(pairs))])
    out["coll_f64"] = np.array([G.box_collision_test(ca[i:i + 1].astype(np.float64),
                                                     cb[i:i + 1].astype(np.float64))[0, 0] for i in range(len(pairs))])
    # a noise search in which every try of the first two boxes fails: their edges cross whatever the small noise
    rng = np.random.RandomState(3)
    boxes = np.array([[0, 0, 4, 4, 0], [1.0, 0, 4, 4, 0], [8, 0, 4, 4, 0], [30, 0, 2, 4, 0.2]], np.float32)
    loc = rng.normal(scale=np.array([0.3, 0.3, 0.2], np.float32), size=[4, 100, 3])
    rot = rng.uniform(-0.78539816, 0.78539816, size=[4, 100])
    out["ns_boxes"], out["ns_loc"], out["ns_rot"] = boxes, loc, rot
    out["ns_sel"] = PA.noise_per_box(boxes, np.ones((4,), np.bool_), loc, rot).astype(np.int32)
    # boundary points of float32 boxes with their 1-ulp neighbours, and non-finite points
    bb = np.array([[10.0, 2.0, -1.7, 1.6, 3.9, 1.56, 0.3], [10.5, 2.5, -1.6, 1.9, 5.0, 2.1, -3.1415926],
                   [20.0, -4.0, -1.5, 0.6, 1.8, 0.7, 3.14]], np.float32)
    r = np.random.default_rng(5)
    base = []
    for surf in G.corner_to_surfaces_3d(G.center_to_corner_box3d(bb, origin=[0.5, 0.5, 0], axis=2)):
        for q in surf:
            u, v = r.random((31, 1)).astype(np.float32), r.random((31, 1)).astype(np.float32)
            base.append((1 - u) * (1 - v) * q[0] + u * (1 - v) * q[1] + u * v * q[2] + (1 - u) * v * q[3])
    base = np.concatenate(base, 0).astype(np.float32)
    axis = r.integers(0, 3, base.shape[0])
    up, down = base.copy(), base.copy()
    rows = np.arange(base.shape[0])
    up[rows, axis] = np.nextafter(base[rows, axis], np.float32(np.inf))
    down[rows, axis] = np.nextafter(base[rows, axis], np.float32(-np.inf))
    odd = np.array([[np.nan, 0, 0], [10, np.nan, -1], [np.inf, 0, 0], [10, -np.inf, 0]], np.float32)
    xyz = np.concatenate([np.stack([base, up, down], 1).reshape(-1, 3), odd], 0)
    pts = np.concatenate([xyz, r.random((len(xyz), 1)).astype(np.float32)], 1)
    with np.errstate(invalid="ignore", over="ignore"):
        mask = G.points_in_rbbox(pts, bb)
    out["bnd_boxes"], out["bnd_points"], out["bnd_mask"] = bb, pts, np.packbits(mask.T.reshape(-1))
    print("collisions", out["coll"], "f64", out["coll_f64"], "all-fail sel", out["ns_sel"], "boundary members",
          mask.sum(0))


def prepared_root(C, work):
    root = os.path.join(work, "kitti")
    K.write_tree(root)
    C.create_kitti_info_file(root)
    for sub in ("training", "testing"):
        os.makedirs(os.path.join(root, sub, "velodyne_reduced"))
    C.create_reduced_point_cloud(root)
    C.create_groundtruth_database(root)
    return root + os.sep     # the configs' data_root ends with a separator; the augmentor joins with pathlib


def time_reference(G, PA, KU, root, reps=10):
    """CPU time per frame of the reference's augmentation (the same steps as the fixture), numba compiled, after one
    warm-up pass that compiles it."""
    for cfg_name, cfg in CONFIGS.items():
        np.random.seed(0)
        aug = PA.PointAugmentor(root, os.path.join(root, "kitti_dbinfos_train.pkl"), cfg["sample_classes"],
                                cfg["min_num_points"], cfg["sample_max_num"], **COMMON)
        frames = [frame_inputs(KU, root, i) for i in K.TRAIN]
        for rep in range(reps + 1):
            if rep == 1:
                t0 = time.process_time()
            for gt, types_, pts in frames:
                augment_frame(G, PA, aug, gt.copy(), list(types_), pts.copy(), cfg["class_names"], {})
        n = reps * len(frames)
        print("%s: %.1f ms of CPU time per frame over %d frames of %d points on average" % (
            cfg_name, (time.process_time() - t0) * 1e3 / n, n, int(np.mean([len(f[2]) for f in frames]))))


def main():
    G, PA, KU, C = reference()
    out = {}
    work = tempfile.mkdtemp(prefix="kitti_aug_golden_")
    try:
        root = prepared_root(C, work)
        if "--time" in sys.argv[1:]:
            time_reference(G, PA, KU, root)
            return
        for cfg_name in CONFIGS:
            for seed in SEEDS:
                run_stream(G, PA, KU, root, cfg_name, seed, out)
    finally:
        shutil.rmtree(work)
    adversarial(G, PA, out)
    np.savez_compressed(os.path.join(HERE, "augment.npz"), **out)


if __name__ == "__main__":
    main()
