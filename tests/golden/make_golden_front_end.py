"""Generate tests/golden/front_end_edges.npz by running the REFERENCE's own numba points_to_voxel and its
sparse_sum_for_anchors_mask / fused_get_anchors_area on the edge constructions of tests/test_front_end_edges.py: cells
of up to 10 000 points in shuffled order at max_points 1 / 5 / 8, the max_voxels cut at 1, m - 1, m, m + 1 and with its
opener at index 8191 / 8192, coordinates at and one ulp around the range limits, the 16 frames of the batch case, and
the anchor masks of 16 frames with empty frames and grid-border cells (1 and 3 classes).  The non-finite cloud is left
out: the reference's result is undefined there.  Run once where the original project is checked out; the fixture is
committed.  Inputs are stored as sha256 digests (the constructions regenerate them from their seeds), voxel outputs as
digests and counts, masks in full (packed bits).

    python tests/golden/make_golden_front_end.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden import import_reference_mmdet, load_ref_points_ops  # noqa: E402
from tests import test_front_end_edges as E  # noqa: E402


def main():
    ops = load_ref_points_ops()
    out = {}
    for tag, (pts, rg, mp, mv) in E.voxel_cases().items():
        v, c, n = ops.points_to_voxel(pts, E.VS, rg, mp, True, mv)
        out["vox_%s_points_sha" % tag] = np.array(E.digest(pts))
        out["vox_%s_M" % tag] = np.int64(c.shape[0])
        out["vox_%s_sha" % tag] = np.array(E.digest(v, c, n))

    import_reference_mmdet()
    from mmdet.core.anchor.anchor3d_generator import AnchorGeneratorStride
    from mmdet.core.bbox3d import geometry as G
    frames = E.anchor_frames()
    out["anchor_frames_sha"] = np.array(E.digest(*frames))
    vs, rg = np.array(E.VS, np.float32), np.array(E.RG, np.float32)
    grid = np.round((rg[3:] - rg[:3]) / vs).astype(np.int64)
    for tag, cfgs in E.ANCHOR_CFGS.items():
        anchors = np.concatenate([AnchorGeneratorStride(**c)([1, 200, 176]).reshape(-1, 7) for c in cfgs], 0)
        bv = G.rbbox2d_to_near_bbox(anchors[..., [0, 1, 3, 4, 6]])
        for b, f in enumerate(frames):
            dm = G.sparse_sum_for_anchors_mask(f, tuple(grid[::-1][1:])).cumsum(0).cumsum(1)
            out["mask_%s_%d" % (tag, b)] = np.packbits(G.fused_get_anchors_area(dm, bv, vs, rg, grid) > 1)
    path = os.path.join(HERE, "front_end_edges.npz")
    np.savez_compressed(path, **out)
    print("front_end_edges: %d arrays, %d bytes" % (len(out), os.path.getsize(path)))


if __name__ == "__main__":
    main()
