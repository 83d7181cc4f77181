"""Generate tests/golden/frustum.npz with the REFERENCE's own camera-frustum crop
(mmdet/core/bbox3d/geometry.py: remove_outside_points :50-61, corner_to_surfaces_3d_jit :562,
surface_equ_3d_jit :177-187, points_in_convex_polygon_3d_jit :190-222) run in the build container.
The reference checkout is absent on the GPU box, so the fixture is committed.

    python tests/golden/make_golden_frustum.py

numba 0.65 cannot compile surface_equ_3d_jit (np.einsum, and object mode is gone), so the reference runs with
NUMBA_DISABLE_JIT=1, set before numba is imported: plain Python, about a second per sweep.

Stored (data only):
  * calib{0,1}_{P2,Tr,R0}: the KITTI calibration of make_golden_results.py and a perturbed copy;
  * planes [4,6,4]: the reference's (normal, d) per face for calib x image shape (375x1242, 370x1224);
  * sweeps synth_cloud(seed, fov_deg=180) for 3 seeds: their digests, and per plane set the kept points as a packed
    bit mask (kept indices = flatnonzero);
  * a boundary cloud stored in full: points drawn on the six faces of plane set 0 and rounded to float32, each with
    its two 1-ulp neighbours along one axis, plus a few non-finite points; its kept masks for every plane set.
"""
import os
import sys

os.environ["NUMBA_DISABLE_JIT"] = "1"

import numpy as np  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import digest, import_reference_mmdet  # noqa: E402
from make_golden_results import CALIB_TXT  # noqa: E402

SEEDS = (0, 1, 2)
SHAPES = ((375, 1242), (370, 1224))


def parse_calib(txt):
    out = {}
    for line in txt.strip().splitlines():
        key, value = line.split(":", 1)
        out[key] = np.array([float(v) for v in value.split()])
    return dict(P2=out["P2"].reshape(3, 4), Tr=out["Tr_velo_to_cam"].reshape(3, 4), R0=out["R0_rect"].reshape(3, 3))


def perturbed(c):
    """Another rig: 1.3 % longer focal length, principal point moved, LiDAR yawed by 0.8 deg and shifted."""
    P2 = c["P2"].copy()
    P2[0, 0] *= 1.013; P2[1, 1] *= 1.013
    P2[0, 2] += 3.7; P2[1, 2] -= 2.1
    a = np.deg2rad(0.8)
    yaw = np.array([[np.cos(a), -np.sin(a), 0.0], [np.sin(a), np.cos(a), 0.0], [0.0, 0.0, 1.0]])
    Tr = c["Tr"].copy()
    Tr[:, :3] = Tr[:, :3] @ yaw
    Tr[:, 3] += [0.02, -0.015, 0.03]
    return dict(P2=P2, Tr=Tr, R0=c["R0"].copy())


def ext4(m):
    out = np.eye(4)
    out[:m.shape[0], :m.shape[1]] = m
    return out


def reference_frustum(G, c, shape):
    """The steps of remove_outside_points before the point test: corners [8,3] and surfaces [1,6,4,3] (LiDAR)."""
    C, R, T = G.projection_matrix_to_CRT_kitti(ext4(c["P2"]))
    frustum = G.get_frustum([0, 0, shape[1], shape[0]], C)
    frustum -= T
    frustum = np.linalg.inv(R) @ frustum.T
    frustum = G.camera_to_lidar(frustum.T, ext4(c["R0"]), ext4(c["Tr"]))
    return frustum, G.corner_to_surfaces_3d_jit(frustum[np.newaxis, ...])


def reference_keep(G, pts, c, shape, surfaces):
    mask = G.points_in_convex_polygon_3d_jit(pts[:, :3], surfaces).reshape(-1)
    reduced = G.remove_outside_points(pts, ext4(c["R0"]), ext4(c["Tr"]), ext4(c["P2"]), shape)
    assert np.array_equal(reduced, pts[mask], equal_nan=True), "remove_outside_points disagrees with its own point test"
    return mask


def boundary_cloud(corners, surfaces, rng, per_face=567):
    base = []
    for f in range(6):
        q = surfaces[0, f]                                              # [4,3] face corners
        u, v = rng.random((per_face, 1)), rng.random((per_face, 1))
        base.append((1 - u) * (1 - v) * q[0] + u * (1 - v) * q[1] + u * v * q[2] + (1 - u) * v * q[3])
    base = np.concatenate(base, 0).astype(np.float32)
    axis = rng.integers(0, 3, base.shape[0])
    up, down = base.copy(), base.copy()
    rows = np.arange(base.shape[0])
    up[rows, axis] = np.nextafter(base[rows, axis], np.float32(np.inf))
    down[rows, axis] = np.nextafter(base[rows, axis], np.float32(-np.inf))
    xyz = np.stack([base, up, down], 1).reshape(-1, 3)
    odd = np.array([[np.nan, 0, 0], [10, np.nan, -1], [10, 0, np.nan], [np.inf, 0, 0], [-np.inf, 0, 0],
                    [10, np.inf, 0], [10, 0, -np.inf]], np.float32)
    xyz = np.concatenate([xyz, odd, corners.astype(np.float32)], 0)
    inten = rng.random((xyz.shape[0], 1)).astype(np.float32)
    return np.ascontiguousarray(np.concatenate([xyz, inten], 1).astype(np.float32))


def main():
    import_reference_mmdet()
    from mmdet.core.bbox3d import geometry as G
    from sassd_b200.synth import synth_cloud

    calibs = [parse_calib(CALIB_TXT)]
    calibs.append(perturbed(calibs[0]))
    out = {}
    for i, c in enumerate(calibs):
        for k, v in c.items():
            out["calib%d_%s" % (i, k)] = v
    sets = [(ci, s) for ci in range(2) for s in SHAPES]
    planes, surfs, corners0 = [], [], None
    for ci, shape in sets:
        corners, surfaces = reference_frustum(G, calibs[ci], shape)
        n, d = G.surface_equ_3d_jit(surfaces[:, :, :3, :])
        planes.append(np.concatenate([n[0], d[0][:, None]], 1))
        surfs.append(surfaces)
        if corners0 is None:
            corners0, surf0 = corners, surfaces
    out["planes"] = np.stack(planes).astype(np.float64)
    out["planeset_calib"] = np.array([ci for ci, _ in sets], np.int32)
    out["planeset_shape"] = np.array([s for _, s in sets], np.int32)

    out["sweep_seed"] = np.array(SEEDS, np.int64)
    out["sweep_npts"] = np.zeros(len(SEEDS), np.int64)
    out["sweep_sha"] = np.array([""] * len(SEEDS), dtype="<U64")
    for si, seed in enumerate(SEEDS):
        pts = synth_cloud(seed, fov_deg=180.0)
        out["sweep_npts"][si] = pts.shape[0]
        out["sweep_sha"][si] = digest(pts)
        for pi, (ci, shape) in enumerate(sets):
            m = reference_keep(G, pts, calibs[ci], shape, surfs[pi])
            out["kept_s%d_p%d" % (si, pi)] = np.packbits(m)
            print("sweep seed %d, plane set %d: %d -> %d points" % (seed, pi, pts.shape[0], m.sum()))

    bnd = boundary_cloud(corners0, surf0, np.random.default_rng(5))
    out["boundary_points"] = bnd
    for pi, (ci, shape) in enumerate(sets):
        with np.errstate(invalid="ignore", over="ignore"):
            m = reference_keep(G, bnd, calibs[ci], shape, surfs[pi])
        out["boundary_kept_p%d" % pi] = np.packbits(m)
        print("boundary cloud, plane set %d: %d -> %d points" % (pi, bnd.shape[0], m.sum()))
    np.savez_compressed(os.path.join(HERE, "frustum.npz"), **out)


if __name__ == "__main__":
    main()
