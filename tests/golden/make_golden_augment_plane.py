"""Generate tests/golden/augment_plane.npz: the augmentation of make_golden_augment.py with road planes, as the
reference runs it when a config sets data.train.with_plane = True: KittiLiDAR.get_road_plane reads each frame's
``training/planes/%06d.txt`` (mmdet/datasets/kitti.py:96-108, 176-179) and PointAugmentor.sample_all moves the sampled
boxes and their points onto it (mmdet/core/point_cloud/point_augmentor.py:220-245).  The root is tests/kitti_root.py's
with tests/kitti_planes.py's plane files and overhang; numba is compiled, with make_golden_augment.py's shims.

    python tests/golden/make_golden_augment_plane.py

Stored, per (config, seed) run over the train frames in ImageSets order, read as velodyne_reduced:
  * the plane as read, each sampled record's height move mv (float64), the sampled boxes sample_all returns;
  * the draws: sha256 of the location and rotation noise, the flip, rotation angle and scale;
  * the sampled records (database paths), the chosen noise index per box;
  * the final GT boxes and labels, the keep flag, the sha256 of the augmented cloud; two clouds in full;
  * the number of scene points the corrected boxes crop that the database boxes would not (``lift_crop``).
"""
import os
import shutil
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_augment import COMMON, CONFIGS, SEEDS, augment_frame, frame_inputs, reference, sha  # noqa: E402
from tests import kitti_planes as KP  # noqa: E402
from tests import kitti_root as K  # noqa: E402


def run_stream(G, PA, KU, get_road_plane, root, cfg_name, seed, out):
    cfg = CONFIGS[cfg_name]
    np.random.seed(seed)
    aug = PA.PointAugmentor(root, os.path.join(root, "kitti_dbinfos_train.pkl"), cfg["sample_classes"],
                            cfg["min_num_points"], cfg["sample_max_num"], **COMMON)
    rec, draws = {}, {}
    orig_npb, orig_sample, orig_sample_all = PA.noise_per_box, aug.sample, aug.sample_all
    orig_normal, orig_uniform, orig_choice = np.random.normal, np.random.uniform, np.random.choice
    orig_to_velo = PA.project_rect_to_velo

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
        rec.setdefault("z", []).extend(float(r["box3d_lidar"][2]) for r in v)
        return v

    def to_velo(pts, calib):
        v = orig_to_velo(pts, calib)
        rec["cur"] = v[:, 2].copy()
        return v

    def sample_all(gt_boxes, gt_types, road_planes=None, calib=None):
        assert road_planes is None
        s = orig_sample_all(gt_boxes, gt_types, rec["plane"], rec["calib"])
        rec["sampled"] = s[0].copy()
        return s
    PA.noise_per_box, PA.project_rect_to_velo, aug.sample, aug.sample_all = npb, to_velo, sample, sample_all
    np.random.normal, np.random.uniform, np.random.choice = normal, uniform, choice
    key = "%s_s%d" % (cfg_name, seed)
    try:
        rows = []
        for fi, idx in enumerate(K.TRAIN):
            rec.clear()
            draws.clear()
            gt, types_, pts = frame_inputs(KU, root, idx)
            rec["plane"] = get_road_plane(None, os.path.join(root, "training", "planes", "%06d.txt" % idx))
            rec["calib"] = KU.Calibration(os.path.join(root, "training", "calib", "%06d.txt" % idx))
            boxes, labels, keep, cloud = augment_frame(G, PA, aug, gt, types_, pts, cfg["class_names"], rec)
            # mv as sample_all computes it: the database box's float64 z minus the plane height it projected
            mv = np.array(rec.get("z", []), np.float64) - rec["cur"] if rec.get("z") else np.zeros((0,))
            sampled = rec["sampled"].reshape(-1, 7)
            lift = 0
            if len(sampled):
                db = sampled.copy()
                db[:, 2] = np.array(rec["z"], np.float64).astype(np.float32)
                lift = int((G.points_in_rbbox(pts, sampled).any(-1) & ~G.points_in_rbbox(pts, db).any(-1)).sum())
            u = draws["uniform"]
            rows.append(dict(paths=";".join(rec.get("paths", [])), sel=rec["sel"].astype(np.int32), boxes=boxes,
                             labels=labels, keep=keep, cloud=sha(cloud), loc=draws["loc"], rot=sha(u[0]),
                             flip=draws["flip"], angle=float(u[1]), scale=float(u[2]), plane=rec["plane"], mv=mv,
                             sampled=sampled, lift=lift))
            if fi in (1, 3) and seed == SEEDS[0] and cfg_name == "car":
                out["%s_cloud%d" % (key, fi)] = cloud
        out[key + "_plane"] = np.stack([r["plane"] for r in rows])
        out[key + "_mv"] = np.concatenate([r["mv"] for r in rows])
        out[key + "_sampled"] = np.concatenate([r["sampled"] for r in rows]).astype(np.float32)
        out[key + "_nsampled"] = np.array([len(r["mv"]) for r in rows], np.int32)
        out[key + "_lift_crop"] = np.array([r["lift"] for r in rows], np.int32)
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
        print(key, "kept", out[key + "_keep"].sum(), "sampled", out[key + "_nsampled"], "lift crop",
              out[key + "_lift_crop"])
    finally:
        PA.noise_per_box, PA.project_rect_to_velo = orig_npb, orig_to_velo
        np.random.normal, np.random.uniform, np.random.choice = orig_normal, orig_uniform, orig_choice


def prepared_root(C, work):
    """make_golden_augment's root with write_planes' planes and add_overhang's points (before create_data, so that
    the reduced cloud has them)."""
    root = os.path.join(work, "kitti")
    K.write_tree(root)
    KP.write_planes(root)
    KP.add_overhang(root)
    C.create_kitti_info_file(root)
    for sub in ("training", "testing"):
        os.makedirs(os.path.join(root, sub, "velodyne_reduced"))
    C.create_reduced_point_cloud(root)
    C.create_groundtruth_database(root)
    return root + os.sep


def main():
    G, PA, KU, C = reference()
    from mmdet.datasets.kitti import KittiLiDAR
    out = {}
    work = tempfile.mkdtemp(prefix="kitti_aug_plane_golden_")
    try:
        root = prepared_root(C, work)
        for cfg_name in CONFIGS:
            for seed in SEEDS:
                run_stream(G, PA, KU, KittiLiDAR.get_road_plane, root, cfg_name, seed, out)
    finally:
        shutil.rmtree(work)
    assert max(int(out[k].max()) for k in out if k.endswith("_lift_crop")) > 0, \
        "no plane lifts a sampled box onto scene points its database box leaves alone"
    np.savez_compressed(os.path.join(HERE, "augment_plane.npz"), **out)


if __name__ == "__main__":
    main()
