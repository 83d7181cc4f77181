"""Road-plane additions to the synthetic KITTI root of tests/kitti_root.py, for the augmentation's with_plane tests:
``write_planes`` writes a plane file for every training frame and ``add_overhang`` puts points above the road where a
lifted database box reaches them.  kitti_root.write_tree is left as it is, so no fixture built on it moves."""
import os

import numpy as np

from tests.kitti_root import TRAIN, VAL

# Per training frame: the road plane's tilt (added to a and c), its height (added to d; -1 lifts the road by ~1 m), the
# factor the coefficients are written with (the reader normalises the normal), and whether the file's normal faces
# down (b > 0, which the reader turns up).
PLANES = {0: (0.01, 0.02, 0.0, 1.0, False), 1: (-0.015, 0.01, 0.05, 2.5, True), 2: (0.0, -0.02, 0.1, 0.7, False),
          3: (0.02, 0.0, -1.0, 1.3, False), 4: (-0.01, -0.01, -0.3, 3.0, True), 5: (0.005, 0.005, 0.0, 1.1, False),
          6: (0.03, 0.015, -0.2, 0.5, False), 7: (0.0, 0.0, 0.2, 1.9, True)}
OVERHANG_FRAME = 3
assert sorted(PLANES) == sorted(TRAIN + VAL)


def write_planes(root):
    """Write ``training/planes/%06d.txt`` for every training frame of write_tree's root, in the planes format AVOD
    ships for KITTI (three header lines, then ``a b c d`` of a x + b y + c z + d = 0 in the rectified camera frame):
    the synthetic ground (y = 1.658 - 0.0106 x + 0.0105 z in both rigs' camera frames) tilted and moved per frame."""
    d = os.path.join(root, "training", "planes")
    os.makedirs(d, exist_ok=True)
    for idx, (da, dc, dd, scale, down) in sorted(PLANES.items()):
        plane = scale * np.array([-0.0106 + da, -1.0, 0.0105 + dc, 1.658 + dd])
        if down:
            plane = -plane
        with open(os.path.join(d, "%06d.txt" % idx), "w") as fh:
            fh.write("# Plane\nWidth 4\nHeight 1\n%s\n" % " ".join("%.6e" % v for v in plane))


def add_overhang(root):
    """Append an overhang to frame OVERHANG_FRAME's sweep: a 1.0 x 0.6 m grid of points at z = 0, above the road
    where every augmentation run of the tests pastes a database Car (centre (15, 2)).  The database box ends 0.2 m
    below it and leaves it alone; lifted ~1 m by that frame's road plane, the box crops it.  The frame has only
    DontCare labels, so the GT database does not change."""
    x, y = np.meshgrid(np.linspace(14.5, 15.5, 11), np.linspace(1.7, 2.3, 7))
    grid = np.stack([x.ravel(), y.ravel(), np.zeros(x.size), np.full(x.size, 0.5)], 1).astype(np.float32)
    with open(os.path.join(root, "training", "velodyne", "%06d.bin" % OVERHANG_FRAME), "ab") as fh:
        grid.tofile(fh)
