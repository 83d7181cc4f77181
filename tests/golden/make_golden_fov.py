"""Generate tests/golden/fov.npz with the REFERENCE's own raw-drive calibration and image-FOV crop
(mmdet/datasets/kitti_utils.py: Calibration(..., from_video=True) :75-79,128-144, get_lidar_in_image_fov :252-263,
the crop KittiVideo applies to every sweep, mmdet/datasets/kitti.py:394) run in the build container.
The reference checkout is absent on the GPU box, so the fixture is committed.

    python tests/golden/make_golden_fov.py

kitti_utils imports cv2 for its drawing helpers only; a stub stands in when OpenCV is not installed.

Every row stored here is also projected by oracle/image_fov.py, the sequential-FMA restatement the device kernel
follows; the generator asserts that its three products equal numpy's (the reference's) on every row, so a BLAS that
sums in another order fails here, not on the GPU.

Stored (data only):
  * calib{0,1}_cam_to_cam / calib{0,1}_velo_to_cam: raw-drive calibration files (with date lines) of the calibration
    of make_golden_results.py and of the perturbed rig of make_golden_frustum.py; calib{0,1}_{P2,Tr,R0}: the
    reference's matrices read from them;
  * set_calib / set_shape: the four crop sets, calib x image shape (375x1242, 370x1224);
  * sweeps synth_cloud(seed, fov_deg=180) for 3 seeds: their digests, and per set the kept points as a packed bit mask;
  * a boundary cloud stored in full (boundary_points, boundary_kind) and its kept masks per set:
      kind 0: points whose u or v sits on 0, w or h of a set: the float32 point on one side of the edge and its two
              1-ulp neighbours along lidar y (u edges) or z (v edges), the triple straddling the edge;
      kind 1: x = 0.1f and its 1-ulp neighbours, on a (y, z) grid around the camera axis;
      kind 2: near-field points, 0.1 < x < 0.35 m, whose rectified depth is negative (their flipped projection can
              land in the image);
      kind 3: rectified depth and uvw2 at zero: the float32 x nearest to each zero and its 1-ulp neighbours;
      kind 4: non-finite points.
"""
import os
import sys
import tempfile
import unittest.mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
from make_golden import digest, import_reference_mmdet  # noqa: E402
from make_golden_frustum import SEEDS, SHAPES, parse_calib, perturbed  # noqa: E402
from make_golden_results import CALIB_TXT  # noqa: E402

from oracle.image_fov import in_image_fov, project  # noqa: E402

CLIP = 0.1
EDGE_BASES = 40           # per edge and set
WALK = 256                # ulps searched on each side of a rounded edge point


def _fmt(a):
    return " ".join(repr(float(v)) for v in np.ravel(a))


def raw_calib_texts(c, p3):
    cam = ("calib_time: 09-Jan-2012 13:57:47\ncorner_dist: 9.950000e-02\n"
           "S_00: 1.392000e+03 5.120000e+02\nR_rect_00: %s\nP_rect_00: %s\nP_rect_02: %s\nP_rect_03: %s\n"
           % (_fmt(c["R0"]), _fmt(np.concatenate([c["P2"][:, :3], np.zeros((3, 1))], 1)), _fmt(c["P2"]), _fmt(p3)))
    velo = ("calib_time: 15-Mar-2012 11:37:16\nR: %s\nT: %s\ndelta_f: 0.000000e+00 0.000000e+00\n"
            "delta_c: 0.000000e+00 0.000000e+00\n" % (_fmt(c["Tr"][:, :3]), _fmt(c["Tr"][:, 3])))
    return cam, velo


def reference_calibration(K, cam, velo):
    with tempfile.TemporaryDirectory() as d:
        for name, text in (("calib_cam_to_cam.txt", cam), ("calib_velo_to_cam.txt", velo)):
            with open(os.path.join(d, name), "w") as fh:
                fh.write(text)
        return K.Calibration(d, from_video=True)


def reference_keep(K, pts, calib, shape):
    """get_lidar_in_image_fov as KittiVideo calls it, its mask, and the check that the oracle's three products are
    numpy's on every row."""
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        kept, _, mask = K.get_lidar_in_image_fov(pts, calib, 0, 0, shape[1], shape[0], return_more=True,
                                                 clip_distance=CLIP)
        ref = K.project_velo_to_ref(pts[:, :3], calib)
        rect = K.project_ref_to_rect(ref, calib)
        uvw = K.cart2hom(rect) @ calib.P2.T
    assert np.array_equal(kept, pts[mask], equal_nan=True)
    o_ref, o_rect, o_uvw = project(pts, calib.P2, calib.V2C, calib.R0)
    for what, a, b in (("V2C", o_ref, ref), ("R0", o_rect, rect), ("P2", o_uvw, uvw)):
        same = (a == b) | (np.isnan(a) & np.isnan(b))
        assert same.all(), "oracle %s product differs from numpy's on %d of %d entries" % (what, (~same).sum(), a.size)
    o_mask = in_image_fov(pts, calib.P2, calib.V2C, calib.R0, shape)
    assert np.array_equal(o_mask, mask), "oracle mask differs on %d points" % (o_mask != mask).sum()
    return mask


def _rect_to_velo(rect, calib):
    ref = rect @ np.linalg.inv(calib.R0).T
    return np.concatenate([ref, np.ones((ref.shape[0], 1))], 1) @ calib.C2V.T


def _walk(base, axis):
    """[n, 2*WALK+1, 4] float32: each base point moved by -WALK..WALK ulps along ``axis``."""
    bits = base[:, axis].view(np.int32).astype(np.int64)
    steps = np.arange(-WALK, WALK + 1)
    sign = np.where(base[:, axis] < 0, -1, 1)[:, None]
    moved = (bits[:, None] + sign * steps[None]).astype(np.int32).view(np.float32)
    out = np.repeat(base[:, None, :], steps.size, 1)
    out[:, :, axis] = moved
    return out


def edge_points(calib, shape, rng):
    """Triples straddling the four image edges of one set (kind 0)."""
    h, w = shape
    out = []
    for edge in range(4):
        t = rng.uniform(0.05, 0.95, EDGE_BASES)
        d = rng.uniform(2.0, 60.0, EDGE_BASES)
        u = np.full(EDGE_BASES, (0.0, float(w))[edge]) if edge < 2 else t * w
        v = t * h if edge < 2 else np.full(EDGE_BASES, (0.0, float(h))[edge - 2])
        P = calib.P2                                            # rectified: P[0,1] = P[1,0] = P[2,:2] = 0
        wz = d + P[2, 3]
        rect = np.stack([(u * wz - P[0, 2] * d - P[0, 3]) / P[0, 0], (v * wz - P[1, 2] * d - P[1, 3]) / P[1, 1], d], 1)
        base = np.concatenate([_rect_to_velo(rect, calib), np.zeros((EDGE_BASES, 1))], 1).astype(np.float32)
        axis = 1 if edge < 2 else 2
        walk = _walk(base, axis)
        keep = in_image_fov(walk.reshape(-1, 4), calib.P2, calib.V2C, calib.R0, shape).reshape(walk.shape[:2])
        for b in range(EDGE_BASES):
            flips = np.flatnonzero(keep[b, 1:] != keep[b, :-1])
            if flips.size:
                k = flips[np.argmin(np.abs(flips - WALK))]
                out.append(walk[b, k - 1:k + 2] if k > 0 else walk[b, k:k + 3])
    return np.concatenate(out, 0)


def _grid():
    y, z = np.meshgrid(np.linspace(-0.3, 0.3, 9), np.linspace(-0.2, 0.05, 9))
    return y.ravel(), z.ravel()


def clip_points():
    """x = 0.1f and its neighbours on a (y, z) grid (kind 1)."""
    x0 = np.float32(CLIP)
    xs = np.array([np.nextafter(x0, np.float32(-1)), x0, np.nextafter(x0, np.float32(1))], np.float32)
    y, z = _grid()
    return np.array([[x, yy, zz, 0.0] for yy, zz in zip(y, z) for x in xs], np.float32)


def near_points():
    """0.1 < x < 0.35 m in front of the LiDAR: behind the camera plane, negative rectified depth (kind 2)."""
    y, z = _grid()
    return np.array([[x, yy, zz, 0.0] for x in np.linspace(0.11, 0.34, 11) for yy, zz in zip(y, z)], np.float32)


def zero_depth_points(calib):
    """Per (y, z) of the grid the float32 x nearest to rect z = 0 and to uvw2 = 0, each with its neighbours (kind 3)."""
    M = calib.R0 @ calib.V2C                                   # rect = M [x, y, z, 1]
    y, z = _grid()
    out = []
    for target in (0.0, -calib.P2[2, 3]):                      # uvw2 = rect z + P2[2, 3]
        x = (target - M[2, 1] * y - M[2, 2] * z - M[2, 3]) / M[2, 0]
        for xx, yy, zz in zip(x.astype(np.float32), y, z):
            for xn in (np.nextafter(xx, np.float32(-1)), xx, np.nextafter(xx, np.float32(1))):
                out.append([xn, yy, zz, 0.0])
    return np.array(out, np.float32)


def odd_points():
    return np.array([[np.nan, 0, 0, 0], [10, np.nan, -1, 0], [10, 0, np.nan, 0], [np.inf, 0, 0, 0], [-np.inf, 0, 0, 0],
                     [10, np.inf, 0, 0], [10, -np.inf, 0, 0], [10, 0, np.inf, 0], [10, 0, -np.inf, 0],
                     [np.inf, np.inf, np.inf, 0], [np.nan, np.nan, np.nan, 0]], np.float32)


def main():
    import_reference_mmdet()
    try:
        import cv2  # noqa: F401
    except ImportError:
        sys.modules["cv2"] = unittest.mock.MagicMock(name="cv2")
    from mmdet.datasets import kitti_utils as K
    from sassd_b200.synth import synth_cloud

    base = parse_calib(CALIB_TXT)
    p3 = np.array([float(v) for v in CALIB_TXT.split("P3:")[1].splitlines()[0].split()]).reshape(3, 4)
    rigs = [base, perturbed(base)]
    out, calibs = {}, []
    for i, c in enumerate(rigs):
        cam, velo = raw_calib_texts(c, p3)
        calib = reference_calibration(K, cam, velo)
        assert np.array_equal(calib.P2, c["P2"]) and np.array_equal(calib.V2C, c["Tr"]) and np.array_equal(calib.R0, c["R0"])
        out["calib%d_cam_to_cam" % i] = np.array(cam)
        out["calib%d_velo_to_cam" % i] = np.array(velo)
        out["calib%d_P2" % i], out["calib%d_Tr" % i], out["calib%d_R0" % i] = calib.P2, calib.V2C, calib.R0
        calibs.append(calib)
    sets = [(ci, s) for ci in range(2) for s in SHAPES]
    out["set_calib"] = np.array([ci for ci, _ in sets], np.int32)
    out["set_shape"] = np.array([s for _, s in sets], np.int32)

    out["sweep_seed"] = np.array(SEEDS, np.int64)
    out["sweep_npts"] = np.zeros(len(SEEDS), np.int64)
    out["sweep_sha"] = np.array([""] * len(SEEDS), dtype="<U64")
    for si, seed in enumerate(SEEDS):
        pts = synth_cloud(seed, fov_deg=180.0)
        out["sweep_npts"][si] = pts.shape[0]
        out["sweep_sha"][si] = digest(pts)
        for k, (ci, shape) in enumerate(sets):
            m = reference_keep(K, pts, calibs[ci], shape)
            out["kept_s%d_k%d" % (si, k)] = np.packbits(m)
            print("sweep seed %d, set %d: %d -> %d points" % (seed, k, pts.shape[0], m.sum()))

    rng = np.random.default_rng(11)
    parts = [(0, edge_points(calibs[ci], shape, rng)) for ci, shape in sets]
    parts += [(1, clip_points()), (2, near_points())]
    parts += [(3, zero_depth_points(c)) for c in calibs]
    parts += [(4, odd_points())]
    bnd = np.concatenate([p for _, p in parts], 0)
    bnd[:, 3] = rng.random(bnd.shape[0]).astype(np.float32)
    kind = np.concatenate([np.full(p.shape[0], k, np.int8) for k, p in parts])
    out["boundary_points"] = np.ascontiguousarray(bnd)
    out["boundary_kind"] = kind
    for k, (ci, shape) in enumerate(sets):
        m = reference_keep(K, bnd, calibs[ci], shape)
        out["boundary_kept_k%d" % k] = np.packbits(m)
        print("boundary cloud, set %d: %d -> %d points;" % (k, bnd.shape[0], m.sum()),
              " ".join("kind %d: %d/%d" % (j, m[kind == j].sum(), (kind == j).sum()) for j in range(5)))
    np.savez_compressed(os.path.join(HERE, "fov.npz"), **out)


if __name__ == "__main__":
    main()
