"""Camera-frustum crop restated in numpy: the per-point test of points_in_convex_polygon_3d_jit
(mmdet/core/bbox3d/geometry.py:190-222) for one 6-face polygon given its planes, as remove_outside_points
(geometry.py:50-61) applies it.  Each numpy operation rounds on its own, so this is the reference's fp64 evaluation
order bit for bit: s = ((x*n.x + y*n.y) + z*n.z) + d, and `s >= 0` rejects."""
import numpy as np


def inside_frustum(points, planes):
    """points [N,>=3] float32, planes [6,4] float64 -> bool [N]."""
    p = np.asarray(points)[:, :3].astype(np.float64)
    planes = np.asarray(planes, np.float64)
    keep = np.ones(p.shape[0], dtype=bool)
    with np.errstate(invalid="ignore", over="ignore"):
        for nx, ny, nz, d in planes:
            s = ((p[:, 0] * nx + p[:, 1] * ny) + p[:, 2] * nz) + d
            keep &= ~(s >= 0)
    return keep


def kept_indices(points, planes):
    return np.flatnonzero(inside_frustum(points, planes))
