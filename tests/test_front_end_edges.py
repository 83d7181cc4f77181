"""The front of the step at its edges, one kernel at a time through the C ABI: the voxelizer, the hash and rulebooks,
the BEV scatter and the anchor masks.  Every output there is an integer or a copied value, so every assertion is bit for
bit.  Outputs are pre-filled with a sentinel, so that both "written" and "left untouched" are asserted.

Voxelizer: against oracle/voxelize.c frame by frame and against tests/golden/front_end_edges.npz (the reference's own
numba points_to_voxel on these constructions, made by make_golden_front_end.py): one cell holding up to 10 000 points
over several rank chunks in shuffled order, max_points 1 / 5 / 8, the max_voxels cut at 1, m - 1, m, m + 1 and with its
opener at frame index 8191 / 8192, coordinates one ulp inside and outside the range, non-finite rows, batches of 16 and
256 frames with empty, one-point and chunk-spanning frames, VOXEL_CAP and HASH_FULL.  The mean is bit-exact against a
sequential fp32 sum of all max_points slots.  Rulebooks: against the oracle's SubM / strided tables on the faces,
edges and corners of the four real level shapes, on degenerate shapes where one bitmap word spans rows, planes and
frames, on solid blocks and odd / even lattices, at ragged row capacities and output capacities, and at 23 frames of the
level-0 grid (keys past 2e9).  BEV scatter: the three scatter kernels against dense_bev in the d*C + c channel order and
their tile distances against test_constant_region_rule.tile_distances.  Anchor masks: the batched kernel against the
reference's per-frame mask at B = 2 and 16."""
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import ref_pipeline as O
from tests.test_constant_region_rule import tile_distances

f32 = np.float32
SENT = 0x7F7F7F7F                          # sentinel word of every pre-filled output
VS = [0.05, 0.05, 0.1]
RG = [0, -40., -3., 70.4, 40., 1.]         # the detector's grid: 1408 x 1600 x 40
RG_S = [0, -3.2, -3., 6.4, 3.2, 1.]        # a 128 x 128 x 40 grid: the oracle's dense table stays small
VR_CHUNK = 8192                            # points per rank chunk of vox_rank_kernel
COUNTS = (1, 4, 5, 6, 33, 300, 10000)      # points of the crowded cells
CUT_VOXELS = 300
VOXEL_CAP, ROWS_CAP, HASH_FULL = 1, 2, 16
LEVELS = [[40, 1600, 1408], [20, 800, 704], [10, 400, 352], [5, 200, 176]]
CAR = dict(sizes=[1.6, 3.9, 1.56], anchor_strides=[0.4, 0.4, 1.0], anchor_offsets=[0.2, -39.8, -1.78],
           rotations=[0, 1.57])
PED = dict(CAR, sizes=[0.6, 0.8, 1.73])
CYC = dict(CAR, sizes=[0.6, 1.76, 1.73])
ANCHOR_CFGS = {"car": [CAR], "multi": [CAR, PED, CYC]}


def digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        a = np.ascontiguousarray(a)
        h.update(str(a.dtype).encode()); h.update(str(a.shape).encode()); h.update(a.tobytes())
    return h.hexdigest()


# ====================================================================== constructions (shared with the fixture script)
def cells_of(points, vs, rg):
    """(z, y, x) of every point with the voxelizer's fp32 arithmetic, and whether it is inside the grid."""
    p = np.asarray(points, f32)
    lo, v = np.asarray(rg[:3], f32), np.asarray(vs, f32)
    grid = np.round((np.asarray(rg[3:], f32) - lo) / v).astype(np.int64)
    with np.errstate(invalid="ignore"):
        c = np.floor((p[:, :3] - lo) / v)
        ok = np.all((c >= 0) & (c < grid), 1)
    c = np.where(ok[:, None], c, 0).astype(np.int64)
    return c[:, ::-1], ok


def openers(points, vs, rg):
    """Indices of the points that open a voxel, in the reference's first-touch order (no cut)."""
    zyx, ok = cells_of(points, vs, rg)
    seen, out = set(), []
    for i in np.nonzero(ok)[0]:
        k = tuple(zyx[i])
        if k not in seen:
            seen.add(k); out.append(int(i))
    return out


def _points_in(cells_zyx, vs, rg, rng):
    """One point strictly inside each (z, y, x) cell, away from its faces; a distinct intensity per point."""
    c = np.asarray(cells_zyx, np.float64)[:, ::-1]
    u = rng.uniform(0.2, 0.8, c.shape)
    xyz = np.asarray(rg[:3], np.float64) + (c + u) * np.asarray(vs, np.float64)
    w = rng.uniform(0, 1, (c.shape[0], 1))
    return np.concatenate([xyz, w], 1).astype(f32)


def _random_cells(rng, n, grid_zyx):
    return np.stack([rng.integers(0, g, n) for g in grid_zyx], 1)


def crowded_cloud(order):
    """Cells holding COUNTS points among 15 000 points of random cells; `order` "shuffled" (a random permutation) or
    "strided" (the big cell on every other index from the start, the others dealt round-robin behind it)."""
    rng = np.random.default_rng(11)
    crowd, tags = [], []
    for k, n in enumerate(COUNTS):
        cell = (5 + k, 20 + 3 * k, 10 + 7 * k)
        crowd.append(_points_in(np.repeat([cell], n, 0), VS, RG_S, rng))
        tags += [k] * n
    filler = _points_in(_random_cells(rng, 15000, (40, 128, 128)), VS, RG_S, rng)
    pts = np.concatenate(crowd + [filler], 0)
    tags = np.array(tags + [-1] * filler.shape[0])
    if order == "shuffled":
        perm = rng.permutation(pts.shape[0])
    else:
        big = np.nonzero(tags == len(COUNTS) - 1)[0]
        rest = np.nonzero(tags != len(COUNTS) - 1)[0]
        rest = rest[np.argsort(np.arange(rest.shape[0]) % 7, kind="stable")]
        perm = np.empty(pts.shape[0], np.int64)
        perm[0:2 * big.shape[0]:2] = big
        perm[1:2 * big.shape[0]:2] = rest[:big.shape[0]]
        perm[2 * big.shape[0]:] = rest[big.shape[0]:]
    return pts[perm], tags[perm]


def cut_cloud(opener):
    """CUT_VOXELS cells opened first, repeats of them up to index `opener`, where a new cell opens voxel number
    CUT_VOXELS (the cut), then points into the open cells and into new cells: the hard stop drops all of them."""
    rng = np.random.default_rng(opener)
    cells = np.unique(_random_cells(rng, 2 * CUT_VOXELS, (40, 128, 128)), axis=0)[:CUT_VOXELS]
    rng.shuffle(cells)
    first = _points_in(cells, VS, RG_S, rng)
    again = _points_in(cells[rng.integers(0, CUT_VOXELS, opener - CUT_VOXELS)], VS, RG_S, rng)
    new = cells[0] + np.array([0, 1, 1])
    while (np.all(cells == new, 1)).any():
        new = new + np.array([0, 0, 1])
    tail_old = _points_in(cells[rng.integers(0, CUT_VOXELS, 1500)], VS, RG_S, rng)
    tail_new = _points_in(_random_cells(rng, 1500, (40, 128, 128)), VS, RG_S, rng)
    tail = np.concatenate([tail_old, tail_new], 0)[rng.permutation(3000)]
    return np.concatenate([first, again, _points_in([new], VS, RG_S, rng), tail], 0)


def edge_cloud():
    """On the detector's grid: each axis at lo, one ulp either side of lo, one ulp below hi and at hi; values
    lo + k*vs (fp32) and one ulp either side, where (p - lo) / vs rounds onto the integer k or just off it."""
    lo, hi, vs = np.asarray(RG[:3], f32), np.asarray(RG[3:], f32), np.asarray(VS, f32)
    grid = np.round((hi - lo) / vs).astype(np.int64)
    base = np.array([35.21, 0.13, -1.04, 0.5], f32)
    rows = []
    for j in range(3):
        vals = [lo[j], np.nextafter(lo[j], f32(-np.inf)), np.nextafter(lo[j], f32(np.inf)),
                np.nextafter(hi[j], f32(-np.inf)), hi[j], np.nextafter(hi[j], f32(np.inf))]
        for k in (1, 2, 3, 7, 10, 19, 100, 333, 777, int(grid[j]) - 1):
            q = f32(lo[j] + f32(k) * vs[j])
            vals += [q, np.nextafter(q, f32(-np.inf)), np.nextafter(q, f32(np.inf))]
        for v in vals:
            p = base.copy(); p[j] = v; p[3] = f32(len(rows) / 256.0)
            rows.append(p)
    return np.stack(rows).astype(f32)


def nonfinite_cloud():
    """A random cloud with NaN and +-inf in some coordinates; returns (cloud, cloud without those rows)."""
    rng = np.random.default_rng(5)
    pts = _points_in(_random_cells(rng, 3000, (40, 128, 128)), VS, RG_S, rng)
    bad = rng.choice(3000, 60, replace=False)
    for t, i in enumerate(bad):
        pts[i, t % 3] = (np.nan, np.inf, -np.inf)[(t // 3) % 3]
    keep = np.all(np.isfinite(pts[:, :3]), 1)
    return pts, pts[keep]


B16_SIZES = [0, 37, 1, 45, 0, 20000, 1, 3, 0, 100, 31, 33, 1, 500, 64, 0]


def batch_frames(kind):
    """"b16": empty frames first, in the middle and last, one-point frames, frame borders off the warp grid, a frame of
    20 000 points (three rank chunks) at an unaligned offset; "b256": 256 frames of 0..5 points.  The first point of
    every frame lies in the cell of the previous frame's last point."""
    rng = np.random.default_rng(16 if kind == "b16" else 256)
    sizes = B16_SIZES if kind == "b16" else list(rng.integers(0, 6, 256))
    frames, last = [], None
    for n in sizes:
        cells = _random_cells(rng, n, (40, 128, 128))
        if n and last is not None:
            cells[0] = last
        if n > 8:
            cells[n // 2:n // 2 + 4] = cells[1]              # a few shared cells inside the frame
        f = _points_in(cells, VS, RG_S, rng)
        if n:
            last = cells[-1]
        frames.append(f)
    return frames


def _blobs(rng, n_blobs, per_blob, grid_zyx, spread=4):
    ctr = _random_cells(rng, n_blobs, grid_zyx)
    c = np.repeat(ctr, per_blob, 0) + rng.integers(-spread, spread + 1, (n_blobs * per_blob, 3))
    return np.clip(c, 0, np.asarray(grid_zyx) - 1)


def anchor_frames():
    """16 frames of (z, y, x) cells on the detector's grid: empty frames 0, 7 and 15, blobs, and cells along the four
    grid borders and in its corners."""
    rng = np.random.default_rng(1600)
    frames = []
    for b in range(16):
        if b in (0, 7, 15):
            frames.append(np.zeros((0, 3), np.int32))
            continue
        c = [_blobs(rng, 60, 25, (40, 1600, 1408))]
        if b % 2:
            for y, x in ((0, 0), (0, 1407), (1599, 0), (1599, 1407)):
                c.append(_blobs(rng, 1, 40, (40, 1600, 1408), 0) * [1, 0, 0] + [0, y, x] +
                         rng.integers(-3, 4, (40, 3)) * [0, 1, 1])
        else:
            for _ in range(6):
                y = rng.integers(0, 1600)
                c.append(np.stack([rng.integers(0, 40, 30), np.full(30, y), rng.choice([0, 1, 1406, 1407], 30)], 1))
                x = rng.integers(0, 1408)
                c.append(np.stack([rng.integers(0, 40, 30), rng.choice([0, 1, 1598, 1599], 30), np.full(30, x)], 1))
        c = np.unique(np.clip(np.concatenate(c, 0), 0, [39, 1599, 1407]), axis=0)
        frames.append(c[rng.permutation(c.shape[0])].astype(np.int32))
    return frames


def voxel_cases():
    """The single-cloud voxelizer cases held to the fixture: tag -> (points, range, max_points, max_voxels)."""
    out = {}
    for order in ("shuffled", "strided"):
        pts, _ = crowded_cloud(order)
        for mp in (1, 5, 8):
            out["crowded_%s_p%d" % (order, mp)] = (pts, RG_S, mp, 20000)
    pts, _ = crowded_cloud("shuffled")
    m = len(openers(pts, VS, RG_S))
    for tag, mv in (("1", 1), ("m-1", m - 1), ("m", m), ("m+1", m + 1)):
        out["maxv_%s" % tag] = (pts, RG_S, 5, mv)
    for op in (8191, 8192):
        out["cut_%d" % op] = (cut_cloud(op), RG_S, 5, CUT_VOXELS)
    out["edge"] = (edge_cloud(), RG, 8, 20000)
    for b, f in enumerate(batch_frames("b16")):
        out["b16_%d" % b] = (f, RG_S, 5, 20000)
    return out


def mean_sequential(voxels, num):
    """SimpleVoxel's mean as the kernel computes it: from +0, every one of the max_points slots added in order in
    fp32 (empty slots are zeros), then one IEEE division."""
    acc = np.zeros((voxels.shape[0], voxels.shape[2]), f32)
    for s in range(voxels.shape[1]):
        acc = (acc + voxels[:, s]).astype(f32)
    return (acc / num.astype(f32)[:, None]).astype(f32)


def oracle_anchor_masks(cfgs, frames):
    _, bv = O.make_anchors(cfgs)
    vs, rg = np.asarray(VS, f32), np.asarray(RG, f32)
    grid = np.round((rg[3:] - rg[:3]) / vs).astype(np.int64)
    return [O.anchors_mask(f, bv, vs, rg, grid) for f in frames]


# ====================================================================== CPU self-checks
def test_crowded_cells_span_warps_ctas_and_rank_chunks():
    for order in ("shuffled", "strided"):
        pts, tags = crowded_cloud(order)
        zyx, ok = cells_of(pts, VS, RG_S)
        assert ok.all()
        for k, n in enumerate(COUNTS):
            idx = np.nonzero(tags == k)[0]
            assert idx.shape[0] == n
            assert np.unique(zyx[idx], axis=0).shape[0] == 1, "a crowded cell's points share one cell"
            if n >= 33:
                assert idx.min() // 256 != idx.max() // 256, "spans several CTAs of 256 points"
        big = np.nonzero(tags == len(COUNTS) - 1)[0]
        assert big.max() // VR_CHUNK - big.min() // VR_CHUNK >= 1, "the 10 000-point cell spans rank chunks"
        if order == "shuffled":
            assert not np.all(np.diff(big[:8]) == 2)


def test_cut_openers_sit_at_8191_and_8192():
    for op in (8191, 8192):
        pts = cut_cloud(op)
        o = openers(pts, VS, RG_S)
        assert len(o) > CUT_VOXELS and o[CUT_VOXELS] == op
        zyx, _ = cells_of(pts, VS, RG_S)
        opened = {tuple(z) for z in zyx[:op]}
        assert sum(tuple(z) in opened for z in zyx[op + 1:]) >= 1000, "points after the cut land in open voxels"
        _, c, _ = O.points_to_voxel(pts, VS, RG_S, 5, CUT_VOXELS)
        assert c.shape[0] == CUT_VOXELS


def test_edge_cloud_straddles_the_range_and_the_cell_faces():
    pts = edge_cloud()
    zyx, ok = cells_of(pts, VS, RG)
    assert ok.any() and (~ok).any()
    lo, vs = np.asarray(RG[:3], f32), np.asarray(VS, f32)
    q = ((pts[:, :3] - lo) / vs).astype(f32)
    assert ((q == np.floor(q)) & (q > 0)).sum() >= 10, "several quotients land exactly on an integer in fp32"
    assert ((q < np.round(q)) & (np.round(q) - q < 1e-3)).any(), "and some one ulp below one"


def test_batches_cross_warps_and_chunks():
    fr = batch_frames("b16")
    sizes = [f.shape[0] for f in fr]
    off = np.concatenate([[0], np.cumsum(sizes)])
    assert sizes[0] == 0 and sizes[-1] == 0 and 0 in sizes[1:-1] and 1 in sizes
    assert off[5] % 32 and (off[6] - off[5] + VR_CHUNK - 1) // VR_CHUNK == 3
    assert any(o % 32 for o in off[1:-1])
    for b in range(1, len(fr)):
        prev = [f for f in fr[:b] if f.shape[0]]
        if fr[b].shape[0] and prev:
            a, c = cells_of(np.stack([prev[-1][-1], fr[b][0]]), VS, RG_S)[0]
            assert np.array_equal(a, c), "frame b starts in the cell where the previous frame ended"
    assert len(batch_frames("b256")) == 256


def test_b23_keys_exceed_2e9_and_b24_would_overflow():
    coords = b23_coords()
    D, H, W = LEVELS[0]
    keys = ((coords[:, 0].astype(np.int64) * D + coords[:, 1]) * H + coords[:, 2]) * W + coords[:, 3]
    assert keys.max() > 2_000_000_000 and keys.max() == 23 * D * H * W - 1
    assert 23 * D * H * W < 2 ** 31 - 1 <= 24 * D * H * W
    per_frame = np.bincount(coords[:, 0])
    assert per_frame.shape[0] == 23 and per_frame.min() >= 2000


def test_lattices_mark_eight_and_one_outputs():
    for kind, fan in (("odd", 8), ("even", 1)):
        c = lattice(kind)
        _, onbr, _ = O.sparse_conv_rulebook(c, [9, 9, 9])
        uses = np.bincount(onbr[onbr >= 0], minlength=c.shape[0])
        assert np.all(uses == fan), kind
    c = solid_block()
    nbr = O.subm_rulebook(c, [8, 8, 8])
    assert ((nbr >= 0).sum(1) == 27).sum() == 64         # the 4^3 interior has all 27 neighbours


def test_tile_distance_cases_reach_9_and_10():
    for H, W in ((200, 176), (13, 21)):
        coords = bev_coords(2, H, W, 5, 7)
        yx = coords[coords[:, 0] == 0][:, 2:]
        d = tile_distances([tuple(v) for v in yx], H, W)
        if H == 13:
            assert (coords[:, 2] == H - 1).any() and (coords[:, 2] == 0).any(), "rows next to the frame border"
        else:
            (y9, x9), (y10, x10) = ISO
            assert d[y9 // 8 + 2, x9 // 16] == 9, "the tile 9 rows below the first isolated cell"
            assert d[y10 // 8 + 2, x10 // 16] == 1 << 20, "the tile 10 rows below the second keeps the sentinel"
            assert d[y10 // 8 + 1, x10 // 16] == 2


def test_oracle_reproduces_the_reference_fixture(golden_dir):
    z = np.load(os.path.join(golden_dir, "front_end_edges.npz"))
    for tag, (pts, rg, mp, mv) in voxel_cases().items():
        assert digest(pts) == str(z["vox_%s_points_sha" % tag]), "the construction %s differs from the fixture" % tag
        v, c, n = O.points_to_voxel(pts, VS, rg, mp, mv)
        assert c.shape[0] == int(z["vox_%s_M" % tag]), tag
        assert digest(v, c, n) == str(z["vox_%s_sha" % tag]), tag
    # the oracle keeps the same points as the reference where a cell holds more than max_points
    assert int(z["vox_crowded_shuffled_p8_M"]) > 1000
    frames = anchor_frames()
    assert digest(*frames) == str(z["anchor_frames_sha"])
    for tag, cfgs in ANCHOR_CFGS.items():
        for b, m in enumerate(oracle_anchor_masks(cfgs, frames)):
            assert np.array_equal(np.packbits(m), z["mask_%s_%d" % (tag, b)]), (tag, b)
        assert sum(int(np.unpackbits(z["mask_%s_%d" % (tag, b)]).sum()) for b in range(16)) > 1000


# ====================================================================== GPU helpers
def _lib():
    from sassd_b200 import lib
    return lib.load()


def _ptr(t):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(rc, what):
    from sassd_b200 import lib
    lib.check(rc, what)


def _sent(shape, dtype=torch.int32):
    """A CUDA buffer every byte of which is 0x7F."""
    t = torch.full(shape, SENT, dtype=torch.int32, device="cuda")
    return t.view(dtype) if dtype != torch.int32 else t


def _bits(a):
    return np.ascontiguousarray(a).view(np.int32)


def _dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


# ====================================================================== voxelizer
PAD_ROWS = 64


def run_voxelize(frames, rg, mp, mv, rows_cap=None, slots=None):
    from sassd_b200 import ops
    L = _lib()
    B = len(frames)
    counts = [f.shape[0] for f in frames]
    total = int(sum(counts))
    pts = torch.zeros((max(total, 1), 4), dtype=torch.float32, device="cuda")
    if total:
        pts[:total] = _dev(np.concatenate(frames, 0))
    off = _dev(np.concatenate([[0], np.cumsum(counts)]).astype(np.int32))
    params, _ = ops.make_voxel_params(VS, rg, mp, mv)
    rows_cap = max(total, 1) if rows_cap is None else rows_cap
    slots = ops.next_pow2(2 * max(max(counts), 1)) if slots is None else slots
    cap = rows_cap + PAD_ROWS
    vox, coors, num = _sent((cap, mp, 4), torch.float32), _sent((cap, 4)), _sent((cap,))
    mean, frame_rows = _sent((cap, 4), torch.float32), _sent((B + 1 + 8,))
    status = torch.zeros((1,), dtype=torch.int32, device="cuda")
    ws = torch.empty((L.sassd_voxelize_workspace_bytes(pts.shape[0], B, slots),), dtype=torch.uint8, device="cuda")
    _check(L.sassd_voxelize(_ptr(pts), _ptr(off), pts.shape[0], B, ctypes.byref(params), slots, _ptr(vox), _ptr(coors),
                            _ptr(num), _ptr(mean), rows_cap, _ptr(frame_rows), _ptr(status), _ptr(ws), ws.numel(),
                            _stream()), "sassd_voxelize")
    torch.cuda.synchronize()
    return dict(vox=vox.cpu().numpy(), coors=coors.cpu().numpy(), num=num.cpu().numpy(), mean=mean.cpu().numpy(),
                frame_rows=frame_rows.cpu().numpy(), status=int(status.item()), rows_cap=rows_cap)


def check_voxelize(got, frames, rg, mp, mv, fixture=None, tags=None):
    B, rows_cap = len(frames), got["rows_cap"]
    exp = [O.points_to_voxel(f, VS, rg, mp, mv) for f in frames]
    cum = np.concatenate([[0], np.cumsum([e[1].shape[0] for e in exp])])
    fr = got["frame_rows"]
    assert np.array_equal(fr[:B + 1], np.minimum(cum, rows_cap)), "frame_rows: clamped running voxel counts"
    assert np.all(np.diff(fr[:B + 1]) >= 0) and fr[B] <= rows_cap
    assert np.all(fr[B + 1:] == SENT)
    assert got["status"] == (VOXEL_CAP if cum[-1] > rows_cap else 0)
    R = int(min(cum[-1], rows_cap))
    ev, ec, en = O.merge_batch([e[0] for e in exp], [e[1] for e in exp], [e[2] for e in exp]) if B else (None,) * 3
    ev, ec, en = ev[:R], ec[:R], en[:R]
    assert np.array_equal(got["coors"][:R], ec)
    assert np.array_equal(got["num"][:R], en)
    assert np.array_equal(_bits(got["vox"][:R]), _bits(ev))
    if R:
        assert np.array_equal(_bits(got["mean"][:R]), _bits(mean_sequential(ev, en)))
        np.testing.assert_allclose(got["mean"][:R], O.simple_voxel(ev, en).numpy(), rtol=1e-6, atol=1e-6)
    for k in ("vox", "coors", "num", "mean"):
        assert np.all(_bits(got[k][R:]) == SENT), k + ": rows past the last voxel are untouched"
    if fixture is not None:
        for b, tag in enumerate(tags):
            s, e = fr[b], fr[b + 1]
            d = digest(got["vox"][s:e], np.ascontiguousarray(got["coors"][s:e, 1:]), got["num"][s:e])
            assert d == str(fixture["vox_%s_sha" % tag]), tag


@pytest.fixture(scope="module")
def fixture(golden_dir):
    return np.load(os.path.join(golden_dir, "front_end_edges.npz"))


@pytest.mark.gpu
@pytest.mark.parametrize("order", ["shuffled", "strided"])
@pytest.mark.parametrize("mp", [1, 5, 8])
def test_voxelize_crowded_cells_keep_the_smallest_indices(fixture, order, mp):
    pts, _ = crowded_cloud(order)
    tag = "crowded_%s_p%d" % (order, mp)
    check_voxelize(run_voxelize([pts], RG_S, mp, 20000), [pts], RG_S, mp, 20000, fixture, [tag])


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["1", "m-1", "m", "m+1"])
def test_voxelize_max_voxels_cut(fixture, which):
    pts, _ = crowded_cloud("shuffled")
    m = len(openers(pts, VS, RG_S))
    mv = {"1": 1, "m-1": m - 1, "m": m, "m+1": m + 1}[which]
    check_voxelize(run_voxelize([pts], RG_S, 5, mv), [pts], RG_S, 5, mv, fixture, ["maxv_" + which])


@pytest.mark.gpu
@pytest.mark.parametrize("opener", [8191, 8192])
def test_voxelize_cut_opener_at_a_rank_chunk_border(fixture, opener):
    pts = cut_cloud(opener)
    check_voxelize(run_voxelize([pts], RG_S, 5, CUT_VOXELS), [pts], RG_S, 5, CUT_VOXELS, fixture, ["cut_%d" % opener])
    # the same cut one frame later, at an unaligned offset
    fr = [batch_frames("b16")[1], pts]
    check_voxelize(run_voxelize(fr, RG_S, 5, CUT_VOXELS), fr, RG_S, 5, CUT_VOXELS)


@pytest.mark.gpu
def test_voxelize_range_edges_and_nonfinite_rows(fixture):
    pts = edge_cloud()
    check_voxelize(run_voxelize([pts], RG, 8, 20000), [pts], RG, 8, 20000, fixture, ["edge"])
    # non-finite coordinates are dropped (the reference's result is undefined there): equal to the oracle on the
    # cloud without those rows
    bad, clean = nonfinite_cloud()
    got = run_voxelize([bad], RG_S, 5, 20000)
    check_voxelize(got, [clean], RG_S, 5, 20000)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["b16", "b256"])
def test_voxelize_batches(fixture, kind):
    frames = batch_frames(kind)
    got = run_voxelize(frames, RG_S, 5, 20000)
    if kind == "b16":
        check_voxelize(got, frames, RG_S, 5, 20000, fixture, ["b16_%d" % b for b in range(16)])
    else:
        check_voxelize(got, frames, RG_S, 5, 20000)
    # a max_voxels cut in every frame at once
    check_voxelize(run_voxelize(frames, RG_S, 5, 3), frames, RG_S, 5, 3)


@pytest.mark.gpu
@pytest.mark.parametrize("cut_frame", [1, 7, 14])
def test_voxelize_rows_cap_clamps_every_frame_offset(cut_frame):
    frames = batch_frames("b16")
    m = np.cumsum([O.points_to_voxel(f, VS, RG_S, 5, 20000)[1].shape[0] for f in frames])
    rows_cap = int(m[cut_frame - 1]) - 2 if m[cut_frame - 1] >= 2 else 1
    got = run_voxelize(frames, RG_S, 5, 20000, rows_cap=rows_cap)
    assert got["status"] & VOXEL_CAP
    assert (got["frame_rows"][:17] == rows_cap).sum() >= 2, "frames that start past rows_cap sit at rows_cap"
    check_voxelize(got, frames, RG_S, 5, 20000)


@pytest.mark.gpu
def test_voxelize_full_hash_is_flagged_and_returns():
    from sassd_b200 import ops
    rng = np.random.default_rng(2)
    pts = _points_in([[1, 1, 1], [2, 2, 2], [3, 3, 3], [1, 1, 1]], VS, RG_S, rng)
    params, _ = ops.make_voxel_params(VS, RG_S, 5, 20000)
    status = torch.zeros((1,), dtype=torch.int32, device="cuda")
    off = torch.tensor([0, 4], dtype=torch.int32, device="cuda")
    ops.voxelize(_dev(pts), off, 1, params, 4, 2, status)
    torch.cuda.synchronize()
    assert int(status.item()) & HASH_FULL


# ====================================================================== hash and rulebooks
def _flat(c, shape):
    c = np.asarray(c, np.int64)
    return ((c[:, 0] * shape[0] + c[:, 1]) * shape[1] + c[:, 2]) * shape[2] + c[:, 3]


def _tile_masks(nbr):
    """per 128-row tile: bit k set when some row of the tile has a neighbour at offset k."""
    n = nbr.shape[0]
    nt = (n + 127) // 128
    pad = np.full((nt * 128, 27), -1, np.int64)
    pad[:n] = nbr
    return (((pad.reshape(nt, 128, 27) >= 0).any(1)) * (1 << np.arange(27))[None, :]).sum(1).astype(np.int32)


def _nbr_table(L, fn, coors, d_rows, rows_cap, shape, index):
    """fn = sassd_rulebook_subm / _conv_nbr into sentinel-filled nbr [rows_cap + 8, 27] and tile masks."""
    nt = (rows_cap + 127) // 128
    nbr, tm = _sent((rows_cap + 8, 27)), _sent((nt + 2,))
    _check(getattr(L, fn)(_ptr(coors), _ptr(d_rows), rows_cap, *shape, _ptr(index.keys), _ptr(index.vals), index.slots,
                          _ptr(nbr), _ptr(tm), _stream()), fn)
    return nbr, tm


def _assert_table(nbr, tm, exp, rows_cap, what):
    n = exp.shape[0]
    live = min((n + 127) // 128 * 128, rows_cap)
    got = nbr.cpu().numpy()
    assert np.array_equal(got[:n], exp), what
    assert np.all(got[n:live] == -1), what + ": rows past d_rows up to the end of the last live tile are -1"
    assert np.all(got[live:] == SENT), what + ": rows of later tiles and past rows_cap are untouched"
    t = tm.cpu().numpy()
    nt = (n + 127) // 128
    assert np.array_equal(t[:nt], _tile_masks(exp)), what
    assert np.all(t[nt:] == SENT), what


def check_rulebooks(coords, B, shape, rows_cap=None, cap_out=None, n_live=None):
    """Hash, SubM table, strided output set (fused next-level hash), strided table and pair tables of one level
    against the oracle.  coords [n,4]; rows_cap >= n (rows past n hold other valid cells); cap_out defaults to the exact
    output count.  Returns (oracle output rows truncated to cap_out, output shape)."""
    from sassd_b200 import ops
    L = _lib()
    coords = np.asarray(coords, np.int32)
    n = coords.shape[0]
    rows_cap = max(n, 1) if rows_cap is None else rows_cap
    buf = np.zeros((rows_cap, 4), np.int32)
    buf[:n] = coords
    if rows_cap > n:                           # cells outside the set: a kernel reading past d_rows would differ
        free = np.setdiff1d(np.arange(B * int(np.prod(shape))), _flat(coords, shape))[:rows_cap - n]
        r = free.copy()
        for j, s in ((3, shape[2]), (2, shape[1]), (1, shape[0])):
            buf[n:n + free.shape[0], j] = r % s; r //= s
        buf[n:n + free.shape[0], 0] = r
    cin, d_rows = _dev(buf), torch.tensor([n], dtype=torch.int32, device="cuda")
    status = torch.zeros((1,), dtype=torch.int32, device="cuda")
    idx = ops.hash_build(ops.HashIndex(rows_cap, "cuda"), cin, d_rows, B, shape, status)
    nbr, tm = _nbr_table(L, "sassd_rulebook_subm", cin, d_rows, rows_cap, shape, idx)
    _assert_table(nbr, tm, O.subm_rulebook(coords, shape), rows_cap, "subm %s" % (shape,))

    oc, onbr, oshape = O.sparse_conv_rulebook(coords, shape)
    count = oc.shape[0]
    cap_out = max(count, 1) if cap_out is None else cap_out
    R = min(count, cap_out)
    Do, Ho, Wo = oshape
    co, dro = _sent((cap_out + 8, 4)), _sent((1,))
    iout = ops.HashIndex(cap_out, "cuda")
    ws = torch.empty((L.sassd_rulebook_conv_workspace_bytes(B, Do, Ho, Wo),), dtype=torch.uint8, device="cuda")
    _check(L.sassd_rulebook_conv_outputs_hash(_ptr(cin), _ptr(d_rows), rows_cap, B, *shape, _ptr(co), _ptr(dro),
                                              cap_out,
                                              _ptr(iout.keys), _ptr(iout.vals), iout.slots, _ptr(status), _ptr(ws),
                                              ws.numel(), _stream()), "conv_outputs_hash")
    torch.cuda.synchronize()
    assert int(dro.item()) == R
    assert int(status.item()) == (ROWS_CAP if count > cap_out else 0), (count, cap_out)
    cog = co.cpu().numpy()
    assert np.array_equal(cog[:R], oc[:R]), "output rows sorted by flattened (b,z,y,x)"
    assert np.all(cog[R:] == SENT)
    # the fused next-level hash holds exactly the first R rows, each with its row
    keys, vals = iout.keys.cpu().numpy(), iout.vals.cpu().numpy()
    used = keys != -1
    okeys = _flat(oc[:R], oshape)
    assert used.sum() == R and np.array_equal(np.sort(keys[used]), okeys)
    assert np.array_equal(vals[used], np.searchsorted(okeys, keys[used]))

    nbr2, tm2 = _nbr_table(L, "sassd_rulebook_conv_nbr", co, dro, cap_out, shape, idx)
    _assert_table(nbr2, tm2, onbr[:R], cap_out, "conv %s" % (shape,))
    pairs = _sent((2, 27, cap_out))
    pnum = _sent((27 + 1,))
    _check(L.sassd_rulebook_pairs(_ptr(nbr2), _ptr(dro), cap_out, _ptr(pairs), _ptr(pnum), _stream()), "pairs")
    op, on = O.nbr_to_indice_pairs(onbr[:R], n_cap=cap_out)
    assert np.array_equal(pnum.cpu().numpy()[:27], on) and int(pnum[27].item()) == SENT
    assert np.array_equal(pairs.cpu().numpy(), op)

    # SubM of the output level on the fused hash == the oracle's == the one on a separate hash_build
    nbr3, tm3 = _nbr_table(L, "sassd_rulebook_subm", co, dro, cap_out, oshape, iout)
    _assert_table(nbr3, tm3, O.subm_rulebook(oc[:R], oshape), cap_out, "subm on the fused hash")
    isep = ops.hash_build(ops.HashIndex(cap_out, "cuda"), co[:cap_out], dro, B, oshape, status)
    nbr4, _ = _nbr_table(L, "sassd_rulebook_subm", co, dro, cap_out, oshape, isep)
    assert torch.equal(nbr3, nbr4)
    torch.cuda.synchronize()
    assert int(status.item()) == (ROWS_CAP if count > cap_out else 0)
    return oc[:R], oshape


def _with_batch(cells_per_frame):
    return np.concatenate([np.pad(c, ((0, 0), (1, 0)), constant_values=b) for b, c in enumerate(cells_per_frame)],
                          0).astype(np.int32)


def level_cells(shape, rng=None):
    """Every combination of {0, 1, mid, n-2, n-1} per axis: corners, the cells next to them, edge and face centres."""
    axes = [sorted({0, 1, s // 2, s - 2, s - 1} & set(range(s))) for s in shape]
    c = np.stack(np.meshgrid(*axes, indexing="ij"), -1).reshape(-1, 3)
    if rng is not None:
        c = c[rng.random(c.shape[0]) < 0.6]
    return c


def solid_block():
    g = np.arange(1, 7)
    return _with_batch([np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)])


def lattice(kind):
    g = np.arange(1, 9, 2) if kind == "odd" else np.arange(0, 9, 2)
    return _with_batch([np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3)])


def b23_coords():
    rng = np.random.default_rng(23)
    frames = []
    for b in range(23):
        c = _blobs(rng, 40, 60, LEVELS[0], spread=3)
        if b == 0:
            c = np.concatenate([c, [[0, 0, 0]]])
        if b == 22:
            c = np.concatenate([c, [[39, 1599, 1407], [39, 1599, 1406], [38, 1598, 1407]]])
        frames.append(np.unique(c, axis=0))
    return _with_batch(frames)


@pytest.mark.gpu
@pytest.mark.parametrize("level", range(4))
@pytest.mark.parametrize("B", [1, 2])
def test_rulebooks_on_the_faces_edges_and_corners_of_the_level_grids(level, B):
    rng = np.random.default_rng(level)
    shape = LEVELS[level]
    cells = [level_cells(shape)] + [level_cells(shape, rng) for _ in range(B - 1)]
    check_rulebooks(_with_batch(cells), B, shape)


ODD_SHAPES = [[1, 1, 1], [1, 1, 3], [3, 1, 1], [2, 3, 1], [5, 3, 2], [7, 5, 33]]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", ODD_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("B", [1, 3, 16])
def test_rulebooks_on_degenerate_shapes(shape, B):
    rng = np.random.default_rng(B * 100 + sum(shape))
    allc = np.stack(np.meshgrid(*[np.arange(s) for s in shape], indexing="ij"), -1).reshape(-1, 3)
    cells = [allc[rng.random(allc.shape[0]) < 0.6] for _ in range(B)]
    if not any(c.shape[0] for c in cells):
        cells[0] = allc[:1]
    check_rulebooks(_with_batch(cells), B, shape)
    check_rulebooks(_with_batch([allc] * B), B, shape)      # every cell of every frame


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["solid", "odd", "even"])
def test_rulebooks_on_blocks_and_lattices(kind):
    if kind == "solid":
        check_rulebooks(solid_block(), 1, [8, 8, 8])
        c = solid_block()
        check_rulebooks(np.concatenate([c, c + [1, 0, 0, 0]]), 2, [8, 8, 8])
    else:
        check_rulebooks(lattice(kind), 1, [9, 9, 9])


@pytest.mark.gpu
@pytest.mark.parametrize("rows_cap", [1, 2, 3, 127, 128, 129, 130, 131, 255, 256, 257])
@pytest.mark.parametrize("below", [False, True])
def test_rulebooks_at_ragged_row_capacities(rows_cap, below):
    rng = np.random.default_rng(rows_cap)
    shape, B = [9, 21, 17], 3
    n = rows_cap - (rows_cap + 2) // 3 if below else rows_cap
    cells = rng.choice(B * 9 * 21 * 17, n, replace=False)
    c = np.zeros((n, 4), np.int32)
    r = cells.copy()
    for j, s in ((3, 17), (2, 21), (1, 9)):
        c[:, j] = r % s; r //= s
    c[:, 0] = r
    oc, _ = check_rulebooks(c, B, shape, rows_cap=rows_cap)
    # the strided table at a ragged output capacity: d_rows_out = count, rows_cap_out = count + 1 .. + 3
    for extra in (1, 2, 3):
        check_rulebooks(c, B, shape, rows_cap=rows_cap, cap_out=max(oc.shape[0], 1) + extra)


@pytest.mark.gpu
@pytest.mark.parametrize("delta", [-1, 0, 1])
@pytest.mark.parametrize("case", ["random", "corners"])
def test_rulebooks_output_capacity_at_the_count(delta, case):
    if case == "random":
        rng = np.random.default_rng(9)
        shape, B = [9, 21, 17], 3
        c = _with_batch([np.unique(_blobs(rng, 12, 20, shape, 2), axis=0) for _ in range(B)])
    else:
        shape, B = LEVELS[1], 2
        c = _with_batch([level_cells(shape), level_cells(shape, np.random.default_rng(1))])
    count = O.sparse_conv_rulebook(c, shape)[0].shape[0]
    check_rulebooks(c, B, shape, cap_out=count + delta)


@pytest.mark.gpu
def test_rulebooks_at_23_frames_of_the_level0_grid_and_24_refused():
    from sassd_b200 import ops
    from sassd_b200.lib import SassdError
    coords = b23_coords()
    shape = LEVELS[0]
    for level in range(4):
        assert shape == LEVELS[level]
        coords, shape = check_rulebooks(coords, 23, shape)
    c24 = _dev(np.concatenate([b23_coords(), [[23, 0, 0, 0]]]).astype(np.int32))
    status = torch.zeros((1,), dtype=torch.int32, device="cuda")
    with pytest.raises(SassdError, match="UNSUPPORTED"):
        ops.hash_build(ops.HashIndex(c24.shape[0], "cuda"), c24, torch.tensor([c24.shape[0]], dtype=torch.int32,
                                                                              device="cuda"), 24, LEVELS[0], status)


# ====================================================================== BEV scatter
ISO = [(111, 95), (166, 134)]              # isolated cells at 200 x 176: y % 8 == 7 (a tile 9 rows below), 6 (10)


def bev_coords(B, H, W, D, seed):
    """(b, d, y, x) rows: random cells, each frame's last row beside the next frame's first row, and on the 200 x 176
    map an isolated cell whose tiles lie at distances 9 and 10."""
    rng = np.random.default_rng(seed)
    rows = []
    for b in range(B):
        n = max(3, H * W // 60)
        cy = rng.integers(0, H // 2, n) if H > 100 else rng.integers(0, H, n)
        rows.append(np.stack([np.full(n, b), rng.integers(0, D, n), cy, rng.integers(0, W, n)], 1))
        xs = rng.integers(0, W, 4)
        rows.append(np.stack([np.full(4, b), rng.integers(0, D, 4), np.full(4, H - 1), xs], 1))
        rows.append(np.stack([np.full(4, b), rng.integers(0, D, 4), np.zeros(4, int), xs], 1))
        if H > 100:
            rows.append(np.array([[b, 0, ISO[0][0], ISO[0][1]], [b, 2, ISO[0][0], ISO[0][1]],
                                  [b, 4, ISO[1][0], ISO[1][1]]]))
            rows.append(np.array([[b, 1, H - 1 - (b % 3), W - 1 - 9 * (b % 2)]]))
    c = np.unique(np.concatenate(rows, 0), axis=0)
    return c[rng.permutation(c.shape[0])].astype(np.int32)


def _split(x):
    hi = x.half()
    lo = ((x - hi.float()) * 2048.0).half()
    return hi, lo


@pytest.mark.gpu
@pytest.mark.parametrize("hw", [(200, 176), (13, 21)], ids=["200x176", "13x21"])
@pytest.mark.parametrize("B", [1, 2, 16, 24])
def test_bev_scatter_matches_dense_bev_and_tile_distances(hw, B):
    from sassd_b200 import ops
    L = _lib()
    H, W = hw
    D, C = 5, 64
    coords = bev_coords(B, H, W, D, B * 7 + H)
    n = coords.shape[0]
    rng = np.random.default_rng(n)
    feat = (rng.standard_normal((n, C)) * 10.0 ** rng.uniform(-3, 3, (n, C))).astype(f32)
    # rows past d_rows: other cells with other values, which must not be scattered
    extra = 5
    junk = bev_coords(B, H, W, D, B * 7 + H + 1)[:extra]
    cap = n + extra
    cd = _dev(np.concatenate([coords, junk], 0))
    fd = _dev(np.concatenate([feat, np.full((extra, C), 7.0, f32)], 0))
    d_rows = torch.tensor([n], dtype=torch.int32, device="cuda")

    exp = torch.zeros((B * H * W * D, C), dtype=torch.float32, device="cuda")
    flat = ((cd[:n, 0].long() * H + cd[:n, 2].long()) * W + cd[:n, 3].long()) * D + cd[:n, 1].long()
    exp[flat] = fd[:n]
    exp = exp.view(B, H, W, D * C)
    if B * H * W <= 2 * 200 * 176:
        ref = O.dense_bev(torch.from_numpy(feat), coords, (D, H, W), B)          # channel c*D + d
        ref = ref.view(B, C, D, H, W).permute(0, 3, 4, 2, 1).reshape(B, H, W, D * C)
        assert torch.equal(exp.cpu(), ref)
    touched = torch.zeros((B * H * W * D,), dtype=torch.bool, device="cuda")
    touched[flat] = True
    touched = touched.view(B, H, W, D, 1).expand(B, H, W, D, C).reshape(B, H, W, D * C)

    th, tw = ops._lib.CONV2D_TILE_H, ops._lib.CONV2D_TILE_W
    nt = B * ((H + th - 1) // th) * ((W + tw - 1) // tw)
    exp_dist = np.concatenate([tile_distances([tuple(v) for v in coords[coords[:, 0] == b][:, 2:]], H, W).ravel()
                               for b in range(B)]).astype(np.int64)
    exp_dist = np.where(exp_dist > ops._lib.TILE_DIST_MAX, ops._TILE_FAR, exp_dist)
    ehi, elo = _split(exp)

    def dist_buf():
        t = torch.full((nt + 4,), ops._TILE_FAR, dtype=torch.int32, device="cuda")
        t[nt:] = SENT
        return t

    def check_dist(t, what):
        got = t.cpu().numpy()
        assert np.array_equal(got[:nt], exp_dist), what
        assert np.all(got[nt:] == SENT), what

    # fp32 scatter into a sentinel map: active slices written, every other value untouched
    bev = _sent((B, H, W, D * C), torch.float32)
    _check(L.sassd_sparse_to_bev(_ptr(fd), _ptr(cd), _ptr(d_rows), cap, C, D, H, W, _ptr(bev), _stream()), "bev")
    sent = torch.full_like(bev.view(torch.int32), SENT)
    assert torch.equal(bev.view(torch.int32), torch.where(touched, exp.view(torch.int32), sent))
    del bev, sent

    # fp32 rows -> split map (product: zero-filled), split = (half(x), half((x - hi) * 2048))
    planes = torch.zeros((2, B, H, W, D * C), dtype=torch.float16, device="cuda")
    dist = dist_buf()
    _check(L.sassd_sparse_to_bev_split(_ptr(fd), _ptr(cd), _ptr(d_rows), cap, C, D, H, W, B, _ptr(planes), _ptr(dist),
                                       _stream()), "bev_split")
    assert torch.equal(planes[0].view(torch.int16), ehi.view(torch.int16))
    assert torch.equal(planes[1].view(torch.int16), elo.view(torch.int16))
    check_dist(dist, "sparse_to_bev_split")

    # split rows -> split map: the row bits copied
    rhi, rlo = _split(fd)
    rows = torch.stack([rhi, rlo]).contiguous()
    planes.zero_()
    dist = dist_buf()
    _check(L.sassd_split_rows_to_bev(_ptr(rows), _ptr(cd), _ptr(d_rows), cap, C, D, H, W, B, _ptr(planes), _ptr(dist),
                                     _stream()), "split_rows_to_bev")
    assert torch.equal(planes[0].view(torch.int16), ehi.view(torch.int16))
    assert torch.equal(planes[1].view(torch.int16), elo.view(torch.int16))
    check_dist(dist, "split_rows_to_bev")


# ====================================================================== anchor masks
@pytest.mark.gpu
@pytest.mark.parametrize("cls", ["car", "multi"])
@pytest.mark.parametrize("B", [2, 16])
def test_anchor_masks_batched_match_the_per_frame_reference(fixture, cls, B):
    from sassd_b200.anchors import AnchorGeneratorStride, AnchorSet
    from sassd_b200.voxel_generator import VoxelGenerator
    L = _lib()
    vg = VoxelGenerator(VS, RG, 5, 20000, device="cuda:0")
    aset = AnchorSet([AnchorGeneratorStride(**c) for c in ANCHOR_CFGS[cls]], vg, device="cuda:0")
    frames = anchor_frames()
    ids = list(range(16)) if B == 16 else [1, 2]
    sel = [frames[i] for i in ids]
    exp = oracle_anchor_masks(ANCHOR_CFGS[cls], sel)
    coors = _with_batch(sel)
    n = coors.shape[0]
    cd = _dev(np.concatenate([coors, np.tile([[0, 0, 5, 5]], (9, 1))], 0).astype(np.int32))   # rows past d_rows
    d_rows = torch.tensor([n], dtype=torch.int32, device="cuda")
    got = aset.mask_device(cd, d_rows, B).cpu().numpy().astype(bool)
    _, rects = aset.device_tensors()
    H, W = aset.grid_hw
    na = rects.shape[0]
    mask = torch.full((B * na + 64,), 0x7F, dtype=torch.uint8, device="cuda")
    ws = torch.empty((L.sassd_anchor_mask_workspace_bytes(B, H, W),), dtype=torch.uint8, device="cuda")
    _check(L.sassd_anchor_mask(_ptr(cd), _ptr(d_rows), cd.shape[0], B, H, W, _ptr(rects), na, aset.threshold,
                               _ptr(mask),
                               _ptr(ws), ws.numel(), _stream()), "anchor_mask")
    m = mask.cpu().numpy()
    assert np.all(m[B * na:] == 0x7F) and set(np.unique(m[:B * na])) <= {0, 1}
    m = m[:B * na].reshape(B, na).astype(bool)
    for j, b in enumerate(ids):
        assert np.array_equal(got[j], exp[j]), (cls, b)
        assert np.array_equal(m[j], exp[j]), (cls, b)
        assert np.array_equal(np.packbits(exp[j]), fixture["mask_%s_%d" % (cls, b)]), (cls, b)
    assert sum(e.sum() for e in exp) > 0
