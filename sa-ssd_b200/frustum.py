"""Camera frustum of a KITTI calibration as six plane equations in the LiDAR frame, for cropping full sweeps on the
device (ops.frustum_crop, csrc/frustum.cu).

The reference makes its ``velodyne_reduced`` clouds offline with ``remove_outside_points``
(mmdet/core/bbox3d/geometry.py:50-61, called by tools/create_data.py:107-140).  This module computes the same planes
on the host in float64:
  * P2[:, :3] = K R with K upper triangular, found by a QR factorisation of its inverse, and T = K^-1 P2[:, 3]
    (geometry.py:23-34);
  * the image box (0, 0, w, h) at the near and far clip depths 0.001 m and 100 m: 8 corners (geometry.py:4-21);
  * the corners moved by -T, rotated by R^-1 and taken from the rectified camera frame to the LiDAR frame through
    (R0_rect Tr_velo_to_cam)^-1 (geometry.py:43-48, 56-58);
  * one plane per face from its first three corners, n = (c0 - c1) x (c1 - c2), d = -n.c0, the normals pointing into
    the frustum (corner_to_surfaces_3d_jit geometry.py:562, surface_equ_3d_jit :177-187).
A point is inside when n.p + d < 0 for all six faces.
"""
import numpy as np

NEAR_CLIP, FAR_CLIP = 0.001, 100.0

# corners: 0-3 near, 4-7 far, each in the image-box order (0,0), (0,h), (w,h), (w,0); faces in the reference's order
# near, far, and the four sides, each listed so that the first three corners give an inward normal
_FACES = np.array([[0, 1, 2, 3], [7, 6, 5, 4], [0, 3, 7, 4], [1, 5, 6, 2], [0, 4, 5, 1], [3, 2, 6, 7]])


def _homogeneous4(m):
    out = np.eye(4)
    out[:m.shape[0], :m.shape[1]] = m
    return out


def frustum_corners(calib, img_shape):
    """The 8 corners [8, 3] (LiDAR frame, float64) of the camera frustum of image size img_shape = (h, w, ...)."""
    P = calib.P2
    q, u = np.linalg.qr(np.linalg.inv(P[:, :3]))        # inv(K R) = R^-1 K^-1: orthogonal times upper triangular
    K, R = np.linalg.inv(u), np.linalg.inv(q)
    T = u @ P[:, 3]
    h, w = float(img_shape[0]), float(img_shape[1])
    uv = np.array([[0.0, 0.0], [0.0, h], [w, h], [w, 0.0]])
    corners = []
    for z in (NEAR_CLIP, FAR_CLIP):
        xy = (uv - K[0:2, 2]) / np.array([K[0, 0] / z, K[1, 1] / z])
        corners.append(np.concatenate([xy, np.full((4, 1), z)], axis=1))
    cam = np.linalg.inv(R) @ (np.concatenate(corners, axis=0) - T).T           # [3, 8], rectified camera frame
    rect_to_velo = np.linalg.inv(_homogeneous4(calib.R0) @ _homogeneous4(calib.V2C))
    return (np.concatenate([cam.T, np.ones((8, 1))], axis=1) @ rect_to_velo.T)[:, :3]


def corner_planes(corners):
    """Corners [..., 8, 3] in the reference's layout (near/bottom face 0-3, far/top face 4-7) -> planes [..., 6, 4] in
    the corners' dtype: one plane per face from its first three corners, n = (c0 - c1) x (c1 - c2), d = -n.c0, normals
    pointing inside.  Nothing is widened: float32 corners give the reference's float32 planes (augment.box_planes32),
    as its np.cross and einsum on float32 surfaces do."""
    c = corners[..., _FACES, :]                                               # [..., 6, 4, 3]
    n = np.cross(c[..., 0, :] - c[..., 1, :], c[..., 1, :] - c[..., 2, :])
    d = -(n * c[..., 0, :]).sum(axis=-1)
    return np.concatenate([n, d[..., None]], axis=-1)


def camera_frustum_planes(calib, img_shape):
    """results.Calibration + image (h, w) -> float64 [6, 4]: (n.x, n.y, n.z, d) per face, normals pointing inside.
    One frame's entry of the ``frustum_planes`` argument of SingleStageDetector.forward_points / detect_stream."""
    return corner_planes(frustum_corners(calib, img_shape))
