"""Generate tests/golden/create_data.npz with the REFERENCE's own tools/create_data.py (create_kitti_info_file,
create_reduced_point_cloud, create_groundtruth_database) run on the synthetic KITTI root of tests/kitti_root.py, in the
build container.  The reference checkout is absent on the GPU box, so the fixture is committed.

    python tests/golden/make_golden_create_data.py

The reference runs with NUMBA_DISABLE_JIT=1 (numba 0.65 cannot compile surface_equ_3d_jit), imageio.imread stubbed to
zeros of the PNG header's shape, tqdm stubbed as the identity and np.bool shimmed (make_golden.import_reference_mmdet).

Stored (data only):
  * the digest of every input file of the tree (sweeps, calibrations, PNGs, labels), which guards its rebuild;
  * kitti_infos_{train,val,trainval,test} and kitti_dbinfos_{train,trainval}, flattened to arrays with their Python
    types (kitti_root.flatten);
  * the name and digest of every reduced cloud and database file (train; trainval on a copy of the tree);
  * random LiDAR boxes (and the label boxes) with the reference's planes: center_to_corner_box3d +
    corner_to_surfaces_3d + surface_equ_3d_jit;
  * a boundary cloud stored in full: points on the faces of a few boxes rounded to float32, each with its two 1-ulp
    neighbours along one axis, the corners and non-finite points; its points_in_rbbox masks.
"""
import os
import shutil
import struct
import sys
import tempfile
import types

os.environ["NUMBA_DISABLE_JIT"] = "1"

import numpy as np  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from make_golden import import_reference_mmdet  # noqa: E402
from tests import kitti_root as K  # noqa: E402


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
    from tools import create_data as C
    return G, C


def ref_planes(G, boxes):
    corners = G.center_to_corner_box3d(boxes, origin=[0.5, 0.5, 0], axis=2)
    n, d = G.surface_equ_3d_jit(G.corner_to_surfaces_3d(corners)[:, :, :3, :])
    return np.concatenate([n, d[..., None]], axis=-1)


def random_boxes(rng, n=48):
    b = np.concatenate([rng.uniform([-40, -40, -3], [70, 40, 1], (n, 3)), rng.uniform(0.2, 5.0, (n, 3)),
                        rng.uniform(-np.pi, np.pi, (n, 1))], axis=1)
    b[:6, 6] = [np.pi, -np.pi, 3.14, -3.14, np.nextafter(np.pi, 0), -np.nextafter(np.pi, 0)]
    b[6, 5] = 0.0
    b[7, 3:6] = 0.0
    return b


def boundary_cloud(G, boxes, rng, per_face=97):
    base = []
    for surf in G.corner_to_surfaces_3d(G.center_to_corner_box3d(boxes, origin=[0.5, 0.5, 0], axis=2)):
        for q in surf:
            u, v = rng.random((per_face, 1)), rng.random((per_face, 1))
            base.append((1 - u) * (1 - v) * q[0] + u * (1 - v) * q[1] + u * v * q[2] + (1 - u) * v * q[3])
    base = np.concatenate(base, 0).astype(np.float32)
    axis = rng.integers(0, 3, base.shape[0])
    up, down = base.copy(), base.copy()
    rows = np.arange(base.shape[0])
    up[rows, axis] = np.nextafter(base[rows, axis], np.float32(np.inf))
    down[rows, axis] = np.nextafter(base[rows, axis], np.float32(-np.inf))
    xyz = np.stack([base, up, down], 1).reshape(-1, 3)
    corners = G.center_to_corner_box3d(boxes, origin=[0.5, 0.5, 0], axis=2).reshape(-1, 3).astype(np.float32)
    odd = np.array([[np.nan, 0, 0], [10, np.nan, -1], [10, 0, np.nan], [np.inf, 0, 0], [-np.inf, 0, 0],
                    [10, np.inf, 0], [10, 0, -np.inf]], np.float32)
    xyz = np.concatenate([xyz, odd, corners], 0)
    inten = rng.random((xyz.shape[0], 1)).astype(np.float32)
    return np.ascontiguousarray(np.concatenate([xyz, inten], 1).astype(np.float32))


def main():
    G, C = reference()
    import pickle
    from oracle.frustum import inside_frustum
    out = {}
    work = tempfile.mkdtemp(prefix="kitti_golden_")
    try:
        root = os.path.join(work, "kitti")
        K.write_tree(root)
        inputs = [os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs]
        inputs = sorted(inputs)
        out["input_files"] = np.array(inputs)
        out["input_sha"] = np.array([K.file_digest(os.path.join(root, f)) for f in inputs])

        C.create_kitti_info_file(root)
        for sub in ("training", "testing"):
            os.makedirs(os.path.join(root, sub, "velodyne_reduced"))
        C.create_reduced_point_cloud(root)
        tv = os.path.join(work, "kitti_tv")
        shutil.copytree(root, tv)
        C.create_groundtruth_database(root)
        C.create_groundtruth_database(tv, info_path=os.path.join(tv, "kitti_infos_trainval.pkl"),
                                      db_info_save_path=os.path.join(tv, "kitti_dbinfos_trainval.pkl"))
        for s in ("train", "val", "trainval", "test"):
            with open(os.path.join(root, "kitti_infos_%s.pkl" % s), "rb") as fh:
                K.flatten(pickle.load(fh), "infos_" + s, out)
        db_boxes = []
        for s, r in (("train", root), ("trainval", tv)):
            with open(os.path.join(r, "kitti_dbinfos_%s.pkl" % s), "rb") as fh:
                db = pickle.load(fh)
            K.flatten(db, "dbinfos_" + s, out)
            db_boxes += [rec["box3d_lidar"] for v in db.values() for rec in v]
            files = K.output_files(r)
            if s == "trainval":
                files = [f for f in files if f.startswith("gt_database/")]
            out["files_" + s] = np.array(files)
            out["files_sha_" + s] = np.array([K.file_digest(os.path.join(r, f)) for f in files])
            print("%s: %d output files, %s" % (s, len(files), {k: len(v) for k, v in db.items()}))
    finally:
        shutil.rmtree(work)

    rng = np.random.default_rng(11)
    boxes = np.concatenate([random_boxes(rng), np.stack(db_boxes)], 0)
    out["boxes"] = boxes
    out["box_planes"] = ref_planes(G, boxes)

    bboxes = np.array([[10.0, 2.0, -1.7, 1.6, 3.9, 1.56, 0.3], [10.5, 2.5, -1.6, 1.9, 5.0, 2.1, -3.1415926],
                       [20.0, -4.0, -1.5, 0.6, 1.8, 0.0, 3.14], [-5.0, 7.0, 0.5, 0.05, 0.07, 0.03, 1.0]])
    bnd = boundary_cloud(G, bboxes, np.random.default_rng(5))
    with np.errstate(invalid="ignore", over="ignore"):
        mask = G.points_in_rbbox(bnd[:, :3], bboxes)
        bplanes = ref_planes(G, bboxes)
        for j in range(len(bboxes)):
            assert np.array_equal(inside_frustum(bnd, bplanes[j]), mask[:, j]), "numpy restatement differs, box %d" % j
    out["boundary_boxes"] = bboxes
    out["boundary_points"] = bnd
    out["boundary_mask"] = np.packbits(mask.T.reshape(-1))
    print("boundary cloud: %d points, members per box %s" % (bnd.shape[0], mask.sum(0)))
    np.savez_compressed(os.path.join(HERE, "create_data.npz"), **out)


if __name__ == "__main__":
    main()
