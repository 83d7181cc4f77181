"""Image-FOV crop restated in numpy: get_lidar_in_image_fov(points, calib, 0, 0, w, h, clip_distance=0.1)
(mmdet/datasets/kitti_utils.py:252-263) as the reference's raw-drive dataset applies it (mmdet/datasets/kitti.py:394).

The reference projects with three fp64 matrix products, ref = [x,y,z,1] V2C^T, rect = ref R0^T, uvw = [rect,1] P2^T
(kitti_utils.py:165-202).  numpy hands these to its BLAS, which evaluates each dot product as a sequential FMA chain
from k = 0: fma(a3,b3, fma(a2,b2, fma(a1,b1, a0*b0))).  That is the order the device kernel uses (csrc/frustum.cu).
numpy has no fused multiply-add, so ``fma`` below computes it exactly: an error-free product (Dekker), an error-free
sum, and a final rounding through round-to-odd (Boldo & Melquiond, "Emulation of FMA and correctly rounded sums:
proved algorithms using rounding to odd", IEEE Trans. Computers 57(4), 2008).  The fixture's generator checks the
three products against numpy's own on every row it stores.

Then u = uvw0/uvw2, v = uvw1/uvw2 (IEEE division), and a point is kept when u < w, u >= 0, v < h, v >= 0 and its fp32
x > 0.1 compared in fp32 (numpy compares a float32 array with a Python float in float32)."""
import numpy as np

CLIP_X = 0.1
_SPLITTER = 134217729.0        # 2**27 + 1


def _split(a):
    c = _SPLITTER * a
    hi = c - (c - a)
    return hi, a - hi


def _two_prod(a, b):
    """p + e == a * b exactly (no overflow or underflow at the magnitudes of a point cloud and a calibration)."""
    p = a * b
    ah, al = _split(a)
    bh, bl = _split(b)
    return p, ((ah * bh - p) + ah * bl + al * bh) + al * bl


def _two_sum(a, b):
    s = a + b
    bb = s - a
    return s, (a - (s - bb)) + (b - bb)


def _add_round_odd(a, b):
    """a + b rounded to odd: exact sums as they are, else the neighbouring float of the two around the sum whose last
    significand bit is 1."""
    s, e = _two_sum(a, b)
    other = np.nextafter(s, np.where(e > 0, np.inf, -np.inf))
    odd = (s.view(np.int64) & 1) == 1
    return np.where((e == 0) | odd, s, other)


def fma(a, b, c):
    """Correctly rounded a * b + c, elementwise on float64 arrays (finite operands; non-finite ones go through
    a * b + c, which gives the same infinities and NaNs)."""
    a, b, c = np.broadcast_arrays(np.asarray(a, np.float64), np.asarray(b, np.float64), np.asarray(c, np.float64))
    with np.errstate(invalid="ignore", over="ignore"):
        uh, ul = _two_prod(a, b)
        th, tl = _two_sum(c, uh)
        z = th + _add_round_odd(tl, ul)
        plain = a * b + c
    return np.where(np.isfinite(a) & np.isfinite(b) & np.isfinite(c), z, plain)


def chain_matmul(x, m):
    """x [N,K] @ m.T for m [R,K], every entry the sequential FMA chain from k = 0 (numpy's BLAS order)."""
    x = np.asarray(x, np.float64)
    m = np.asarray(m, np.float64)
    out = np.empty((x.shape[0], m.shape[0]))
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(m.shape[0]):
            acc = x[:, 0] * m[r, 0]
            for k in range(1, m.shape[1]):
                acc = fma(x[:, k], m[r, k], acc)
            out[:, r] = acc
    return out


def _hom(x):
    return np.concatenate([x, np.ones((x.shape[0], 1))], axis=1)


def project(points, P2, V2C, R0):
    """points [N,>=3] float32 -> (ref [N,3], rect [N,3], uvw [N,3]) in fp64, the reference's three products."""
    xyz = np.asarray(points)[:, :3].astype(np.float64)
    ref = chain_matmul(_hom(xyz), V2C)
    rect = chain_matmul(ref, R0)
    uvw = chain_matmul(_hom(rect), P2)
    return ref, rect, uvw


def in_image_fov(points, P2, V2C, R0, img_shape, clip_x=CLIP_X):
    """points [N,>=3] float32, calibration matrices, image (h, w, ...) -> bool [N]: the kept points."""
    points = np.asarray(points)
    _, _, uvw = project(points, P2, V2C, R0)
    h, w = float(img_shape[0]), float(img_shape[1])
    with np.errstate(invalid="ignore", divide="ignore"):
        u = uvw[:, 0] / uvw[:, 2]
        v = uvw[:, 1] / uvw[:, 2]
        return (u < w) & (u >= 0) & (v < h) & (v >= 0) & (points[:, 0] > np.float32(clip_x))
