"""Generate tests/golden/gt_lidar.npz from the REFERENCE's labelled test path, KittiLiDAR.prepare_test_img with
with_label=True (mmdet/datasets/kitti.py:265-293): read_label -> box3d -> project_rect_to_velo -> Van as Car -> class
selection, on synthetic label_2 and calib files.  The reference checkout is absent where the tests run, so the fixture
is committed; it holds the files' text, the reference's C2V of each calibration and its gt_bboxes / gt_labels.

    python tests/golden/make_golden_gt.py

The dataset object is made without its constructor (which builds anchors and reads ImageSets) and given only what
prepare_test_img reads on this path; the image read and transform and mmcv's DataContainer are stubbed.  A frame whose
only rows are DontCare makes the reference fail (its empty box array is 1-D and cannot be indexed by column); the
fixture records that frame with an ``error`` flag.
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import import_reference_mmdet  # noqa: E402

CLASS_LISTS = (["Car"], ["Car", "Pedestrian", "Cyclist"])


def calib_text(rng):
    """A KITTI object calib file: P0..P3, R0_rect, Tr_velo_to_cam, Tr_imu_to_velo, values near the real ones."""
    def rot(a, b, c):
        ca, sa, cb, sb, cc, sc = np.cos(a), np.sin(a), np.cos(b), np.sin(b), np.cos(c), np.sin(c)
        rx = np.array([[1, 0, 0], [0, ca, -sa], [0, sa, ca]])
        ry = np.array([[cb, 0, sb], [0, 1, 0], [-sb, 0, cb]])
        rz = np.array([[cc, -sc, 0], [sc, cc, 0], [0, 0, 1]])
        return rz @ ry @ rx
    f = rng.uniform(700, 730)
    p2 = np.array([[f, 0, rng.uniform(600, 615), rng.uniform(40, 50)], [0, f, rng.uniform(170, 185), rng.uniform(-0.5, 0.5)],
                   [0, 0, 1, rng.uniform(0.002, 0.006)]])
    r0 = rot(*rng.uniform(-0.01, 0.01, 3))
    # velo (x fwd, y left, z up) -> camera (x right, y down, z fwd), slightly perturbed
    base = np.array([[0, -1, 0], [0, 0, -1], [1, 0, 0]], np.float64)
    v2c = np.concatenate([rot(*rng.uniform(-0.02, 0.02, 3)) @ base,
                          np.array([[rng.uniform(-0.01, 0.01)], [rng.uniform(-0.08, -0.06)], [rng.uniform(-0.3, -0.25)]])], 1)
    fmt = lambda a: " ".join("%.12e" % v for v in np.asarray(a).reshape(-1))    # noqa: E731
    lines = ["P0: " + fmt(p2), "P1: " + fmt(p2), "P2: " + fmt(p2), "P3: " + fmt(p2), "R0_rect: " + fmt(r0),
             "Tr_velo_to_cam: " + fmt(v2c), "Tr_imu_to_velo: " + fmt(np.eye(3, 4))]
    return "".join(l + "\n" for l in lines)


def label_text(rng, names):
    out = []
    for name in names:
        if name == "DontCare":
            vals = [-1, -1, -10] + list(np.round(rng.uniform(0, 1200, 4), 2)) + [-1, -1, -1, -1000, -1000, -1000, -10]
        else:
            vals = [round(float(rng.uniform(0, 1)), 2), int(rng.integers(0, 4)), round(float(rng.uniform(-3.1, 3.1)), 2)]
            vals += list(np.round(rng.uniform(0, 1200, 4), 2)) + list(np.round(rng.uniform(0.5, 4.5, 3), 2))
            vals += [round(float(rng.uniform(-20, 20)), 2), round(float(rng.uniform(0.5, 2.5)), 2),
                     round(float(rng.uniform(3, 70)), 2), round(float(rng.uniform(-3.14, 3.14)), 2)]
        out.append(" ".join([name] + [str(v) for v in vals]))
    return "".join(l + "\n" for l in out)


FRAMES = [
    ["Car", "Van", "Pedestrian", "DontCare", "DontCare"],
    ["Car"],
    ["Cyclist", "Person_sitting", "Car", "Truck", "Van", "Tram", "Misc", "DontCare"],
    ["DontCare"],
    ["Pedestrian", "Pedestrian", "Person_sitting"],
    ["Van", "Van", "Car", "Cyclist", "Car", "Car", "DontCare"],
]


def main():
    import_reference_mmdet()
    import torch  # noqa: F401
    from mmdet.datasets import kitti as K
    from mmdet.datasets.kitti_utils import Calibration
    K.DC = lambda x, **kw: x
    K.mmcv.imread = lambda path: np.zeros((375, 1242, 3), np.uint8)
    rng = np.random.default_rng(5)
    calibs = [calib_text(rng) for _ in range(3)]
    labels = [label_text(rng, names) for names in FRAMES]
    out = {"nframes": np.array(len(FRAMES)), "ncalib": np.array(len(calibs))}
    with tempfile.TemporaryDirectory() as d:
        for sub in ("calib", "label_2", "image_2"):
            os.makedirs(os.path.join(d, sub))
        for i in range(len(FRAMES)):
            with open(os.path.join(d, "calib", "%06d.txt" % i), "w") as fh:
                fh.write(calibs[i % len(calibs)])
            with open(os.path.join(d, "label_2", "%06d.txt" % i), "w") as fh:
                fh.write(labels[i])
        for c, text in enumerate(calibs):
            out["calib_txt_%d" % c] = np.array(text)
            out["c2v_%d" % c] = Calibration(os.path.join(d, "calib", "%06d.txt" % c)).C2V
        for i in range(len(FRAMES)):
            out["label_txt_%d" % i] = np.array(labels[i])
        for ci, names in enumerate(CLASS_LISTS):
            ds = K.KittiLiDAR.__new__(K.KittiLiDAR)
            ds.sample_ids = list(range(len(FRAMES)))
            ds.img_prefix, ds.calib_prefix = os.path.join(d, "image_2"), os.path.join(d, "calib")
            ds.label_prefix = os.path.join(d, "label_2")
            ds.img_transform = lambda img, scale, flip: (img, img.shape, img.shape, 1.0)
            ds.with_label, ds.with_mask, ds.with_point = True, False, False
            ds.class_names, ds.anchors, ds.generator = names, None, None
            for i in range(len(FRAMES)):
                key = "%d_%d" % (ci, i)
                try:
                    data = ds.prepare_test_img(i)
                except IndexError:
                    out["error_" + key] = np.array(1)
                    continue
                out["error_" + key] = np.array(0)
                out["boxes_" + key] = data["gt_bboxes"].numpy()
                out["labels_" + key] = data["gt_labels"].numpy()
    np.savez_compressed(os.path.join(HERE, "gt_lidar.npz"), **out)
    print("wrote", len(FRAMES), "frames x", len(CLASS_LISTS), "class lists;",
          sum(int(v) for k, v in out.items() if k.startswith("error_")), "reference failures")


if __name__ == "__main__":
    main()
