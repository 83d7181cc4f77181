"""The tensor-core convolutions bit for bit: the TMA-fed dense conv (csrc/conv2d_tma.cu), the split-row sparse conv
(csrc/spconv_split.cu) and the gathered GEMM (csrc/gconv_tc.cu, with csrc/gconv.cu's FFMA path beside it).

All three use the 3xFP16 split: hi = half(x), a lo plane holding half((x - hi) * 2048), and
x * w ~ a_hi * w_hi + (a_hi * w_lo + a_lo * w_hi) / 2048 summed in two fp32 accumulators (big, small).  The tolerance
tests (test_bev_conv_feed.py, test_sparse_chunk_deal.py) accept ~2e-5 relative error, far above what a wrong lo path,
a single lost channel or a mis-reduced piece costs.  Here the operands are chosen so that every product and every
partial sum is exact in fp32, whatever the summation order or the split of the sum over CTAs:

* split grid: every hi part is an integer in [-AMAX, AMAX] and every stored lo value a multiple of 1/4; every output
  column has at most BUDGET // AMAX nonzero weights w = i + j * 2^-13 (i in {-1, 1}, j in {-1, 0, 1}), so
  sum max|a_hi| * |w_hi| <= BUDGET over the column.  The big accumulator then holds integers below 2^11, the small one
  multiples of 1/4 below 2^11, and big + small / 2048 is a multiple of 2^-13 below 2^10: exact in fp32.  A power-of-two
  scale and a shift on a 2^-6 grid keep the epilogue exact.
* coarse grid: multiples of 1/4 in [-1, 1] with lo = 0, the same column bound: FFMA, 3xTF32 and 3xFP16 agree.

A correct kernel must return exactly the fp64 value of the three-product formula (without the lo * lo term; computed
here by fp64 GEMMs, exact in any order), its fmaf(., scale, shift) and ReLU, and numpy's round-to-nearest-even split
of that fp32 value.  Every GPU assertion is an exact equality.  The fixtures assert that the reference is exactly
representable in fp32, so a broken fixture fails as a fixture error and not as a kernel mismatch."""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_background_tiles import tile_kinds
from tests.test_sparse_chunk_deal import _tile_masks, active_chunks, takes_deal

AMAX = 2                 # max |a_hi| on the split grid
BUDGET = 900             # bound on sum max|a_hi| * |w_hi| per output column
LO_SCALE = 2048.0
TH, TW = 8, 16           # SASSD_CONV2D_TILE_H / _W

# dense layers (taps, cin, cin_stored, cout): the BEV neck's, the heads' and PSWarp's shapes
DENSE_LAYERS = {
    "3x3_320_256": (9, 320, 320, 256),
    "3x3_256_256": (9, 256, 256, 256),
    "1x1_256_256": (1, 256, 256, 256),
    "1x1_256_20": (1, 256, 256, 20),
    "1x1_256_72": (1, 256, 256, 72),
    "3x3_256_28": (9, 256, 256, 28),
    "1x1_28_28_stored64": (1, 28, 64, 28),
}
# sparse layers (cin, cin_stored, cout) with 27 taps: the backbone's channel pairs
SPARSE_PAIRS = [(4, 8, 16), (16, 16, 16), (16, 16, 32), (32, 32, 32), (32, 32, 64), (64, 64, 64)]
# (relu, scale given, shift given)
OPTIONS = [(True, True, True), (False, True, True), (True, False, False), (False, False, True)]


# ------------------------------------------------------------------------------------------------ grids (CPU-tested)
def split16_np(x):
    """numpy's round-to-nearest-even split of fp32 values: (hi, lo) fp16 with lo = half((x - hi) * 2048)."""
    x = np.asarray(x, np.float32)
    hi = x.astype(np.float16)
    lo = ((x - hi.astype(np.float32)) * np.float32(LO_SCALE)).astype(np.float16)
    return hi, lo


def split16(x):
    """The same split of an fp32 torch tensor (SplitMap.from_float's arithmetic), on its device."""
    hi = x.half()
    return hi, ((x - hi.float()) * LO_SCALE).half()


def grid_weights(taps, cin, cout, seed, amax=AMAX, coarse=False):
    """fp32 weights [taps, cin, cout]: per output column BUDGET // amax nonzero entries at random (tap, channel)
    positions, i + j * 2^-13 on the split grid, or +-{1/4 .. 1} on the coarse grid."""
    g = torch.Generator().manual_seed(seed)
    K = taps * cin
    nnz = min(K, BUDGET // amax)
    rows = torch.rand(K, cout, generator=g).argsort(0)[:nnz]
    sign = torch.randint(0, 2, (nnz, cout), generator=g).float() * 2 - 1
    if coarse:
        vals = sign * torch.randint(1, 5, (nnz, cout), generator=g).float() / 4
    else:
        vals = sign + torch.randint(-1, 2, (nnz, cout), generator=g).float() * 2.0 ** -13
    return torch.zeros(K, cout).scatter_(0, rows, vals).view(taps, cin, cout)


def grid_planes(shape, cin, seed, device="cpu", amax=AMAX, lo_from=1, coarse=False):
    """Split planes [2, *shape] fp16 (last dim = stored channels, those >= cin zero).  Split grid: hi an integer in
    [-amax, amax], stored lo in {-3/4 .. 3/4}, zero where |hi| < lo_from.  lo_from = 1 keeps lo = 0 where hi = 0, so
    that the planes are the split of their own fp32 value (what gconv, which splits fp32 inputs, needs).  Coarse grid:
    hi a multiple of 1/4 in [-1, 1], lo = 0."""
    g = torch.Generator(device=device).manual_seed(seed)
    if coarse:
        hi = torch.randint(-4, 5, shape, generator=g, device=device).float() / 4
        lo = torch.zeros_like(hi)
    else:
        hi = torch.randint(-amax, amax + 1, shape, generator=g, device=device).float()
        lo = torch.randint(-3, 4, shape, generator=g, device=device).float() / 4
        # fp16's spacing halves below 1: beside hi = +-1 only |lo| <= 1/4 keeps half(hi + lo / 2048) == hi
        lo = torch.where(hi.abs() == 1, lo.clamp(-0.25, 0.25), lo)
        if lo_from:
            lo = torch.where(hi.abs() >= lo_from, lo, torch.zeros_like(lo))
    p = torch.stack([hi, lo]).half()
    p[..., cin:] = 0
    return p.contiguous()


def planes_value(planes):
    """fp32 value of split planes, hi + lo / 2048 (exact on both grids)."""
    return planes[0].float() + planes[1].float() / LO_SCALE


def grid_bn(cout, seed, device):
    """Power-of-two scales and shifts on a 2^-6 grid in [-4, 4]: fmaf(v, scale, shift) stays exact."""
    g = torch.Generator().manual_seed(seed)
    scale = 2.0 ** torch.randint(-1, 2, (cout,), generator=g).float()
    shift = torch.randint(-256, 257, (cout,), generator=g).float() / 64
    return scale.to(device), shift.to(device)


def column_bound(w, amax):
    """max over output columns of sum max|a_hi| * |w_hi| (the big accumulator's bound) and of the small one's bound."""
    hi, lo = split16(w.float())
    hi = hi.double().abs().reshape(-1, w.shape[-1])
    lo = lo.double().abs().reshape(-1, w.shape[-1])
    return float((amax * hi).sum(0).max()), float((amax * lo + 0.75 * hi).sum(0).max())


# ------------------------------------------------------------------------------------------------ exact references
def exact32(t):
    return bool(torch.equal(t.float().double(), t))


def _operands(planes, cin, w):
    """fp64 GEMM operands whose product is a_hi*w_hi + (a_hi*w_lo + a_lo*w_hi)/2048: [a_hi | a_lo/2048] and
    [w_hi + w_lo/2048 ; w_hi] per tap."""
    x = torch.cat([planes[0, ..., :cin].double(), planes[1, ..., :cin].double() / LO_SCALE], -1)
    hi, lo = split16(w.float())
    hi, lo = hi.double(), lo.double()
    return x, torch.cat([hi + lo / LO_SCALE, hi], 1)


def conv_ref(planes, cin, w):
    """planes [2, B, H, W, Cs] -> fp64 [B, H, W, cout] before the epilogue (3x3 pad 1 or 1x1)."""
    x, wt = _operands(planes, cin, w.to(planes.device))
    if w.shape[0] == 1:
        return x @ wt[0]
    B, H, W, _ = x.shape
    xp = torch.nn.functional.pad(x, (0, 0, 1, 1, 1, 1))
    v = None
    for t in range(9):
        ky, kx = divmod(t, 3)
        part = xp[:, ky:ky + H, kx:kx + W] @ wt[t]
        v = part if v is None else v + part
    return v


def rows_ref(planes, cin, w, nbr, n_rows):
    """Split rows [2, in_rows, Cs] through the neighbour table nbr [rows, taps] (None: row m reads row m) -> fp64
    [n_rows, cout] before the epilogue."""
    x, wt = _operands(planes, cin, w.to(planes.device))
    if nbr is None:
        return x[:n_rows] @ wt[0]
    v = torch.zeros((n_rows, w.shape[2]), dtype=torch.float64, device=planes.device)
    nb = nbr[:n_rows].long()
    for t in range(w.shape[0]):
        o = torch.nonzero(nb[:, t] >= 0).view(-1)
        v.index_add_(0, o, x[nb[o, t]] @ wt[t])
    return v


def epilogue(v, scale, shift, relu):
    """fmaf(v, scale, shift) and ReLU in fp64, asserting that v and the result are exact fp32 values."""
    assert exact32(v), "fixture: the accumulated value is not an fp32 value (grid broken)"
    o = v
    if scale is not None:
        o = o * scale.double()
    if shift is not None:
        o = o + shift.double()
    assert exact32(o), "fixture: the epilogue's result is not an fp32 value (grid broken)"
    return o.clamp_min(0) if relu else o


def assert_split_out(planes, ref, cout, what):
    """Split planes [2, ..., Cs]: channels < cout equal the split of the fp32 reference, the rest zero."""
    hi, lo = split16(ref.float())
    for k, (got, want) in enumerate(((planes[0, ..., :cout], hi), (planes[1, ..., :cout], lo))):
        if not torch.equal(got, want):
            bad = (got != want).nonzero()[:4].tolist()
            raise AssertionError("%s: %s plane differs at %s: %s vs %s" % (
                what, ("hi", "lo")[k], bad, [float(got[tuple(i)]) for i in bad], [float(want[tuple(i)]) for i in bad]))
    assert bool((planes[..., cout:] == 0).all()), "%s: stored channels past cout are not zero" % what


def assert_f32_out(f32, ref, cout, what):
    got = f32[..., :cout]
    want = ref.float()
    if not torch.equal(got, want):
        bad = (got != want).nonzero()[:4].tolist()
        g = [float(got[tuple(i)]) for i in bad]
        e = [float(want[tuple(i)]) for i in bad]
        raise AssertionError("%s: fp32 output differs at %s: %s vs %s (bits %s vs %s)" % (
            what, bad, g, e, [hex(np.float32(x).view(np.uint32)) for x in g],
            [hex(np.float32(x).view(np.uint32)) for x in e]))
    assert bool((f32[..., cout:] == 0).all()), "%s: fp32 columns past cout are not zero" % what


# ------------------------------------------------------------------------------------------------ CPU tests
def test_weight_split_gives_integer_hi_and_quarter_lo():
    """w = i + j * 2^-13 splits into hi = i and stored lo = j / 4, in numpy and in torch alike."""
    i = np.array([-1, -1, -1, 0, 1, 1, 1], np.float32)
    j = np.array([-1, 0, 1, 0, -1, 0, 1], np.float32)
    w = i + j * np.float32(2.0 ** -13)
    hi, lo = split16_np(w)
    assert np.array_equal(hi.astype(np.float32), i) and np.array_equal(lo.astype(np.float32), j / 4)
    th, tl = split16(torch.from_numpy(w))
    assert np.array_equal(th.numpy(), hi) and np.array_equal(tl.numpy(), lo)
    w = grid_weights(9, 64, 32, seed=1)
    hi, lo = split16_np(w.numpy())
    assert np.array_equal(hi.astype(np.float32), np.round(w.numpy()))
    assert set(np.unique(lo.astype(np.float32) * 4)) <= {-1.0, 0.0, 1.0}
    assert not np.any((hi == 0) & (lo != 0)), "j = 0 where i = 0"


@pytest.mark.parametrize("coarse", [False, True])
def test_planes_are_the_split_of_their_value(coarse):
    """Planes with lo = 0 where hi = 0 are the round-to-nearest split of their own fp32 value (numpy, torch and
    SplitMap.from_float alike), so kernels that split fp32 inputs see the same operands; hi integer, lo in quarters."""
    from sassd_b200 import ops
    p = grid_planes((3, 5, 7, 64), 40, seed=2, coarse=coarse)
    v = planes_value(p)
    hi, lo = split16_np(v.numpy())
    assert np.array_equal(hi, p[0].numpy()) and np.array_equal(lo, p[1].numpy())
    sm = ops.SplitMap.from_float(v[..., :40])
    assert torch.equal(sm.planes, p)
    if coarse:
        assert bool((p[1] == 0).all()) and bool(((p[0].float() * 4).frac() == 0).all())
        assert float(p[0].float().abs().max()) <= 1
    else:
        assert bool((p[0].float().frac() == 0).all()) and bool(((p[1].float() * 4).frac() == 0).all())
        assert float(p[0].float().abs().max()) <= AMAX and float(p[1].float().abs().max()) <= 0.75
    # lo_from = 0: lo beside a zero hi too (planes written directly, not the split of a value)
    p0 = grid_planes((4000,), 4000, seed=3, lo_from=0)
    assert bool(((p0[0] == 0) & (p0[1] != 0)).any())


@pytest.mark.parametrize("taps,cin,cout,amax", [(t, ci, co, AMAX) for t, ci, _, co in DENSE_LAYERS.values()] +
                         [(27, ci, co, AMAX) for ci, _, co in SPARSE_PAIRS] + [(1, 64, 64, AMAX), (9, 64, 256, 3)])
def test_column_bounds_at_every_shape(taps, cin, cout, amax):
    """The structural bound holds per column at every listed shape: the big accumulator below 2^11 in integers, the
    small one below 2^11 in quarters, so big + small/2048 fits 24 bits."""
    w = grid_weights(taps, cin, cout, seed=taps * 1000 + cin + cout, amax=amax)
    big, small = column_bound(w, amax)
    assert big <= BUDGET < 2 ** 11 and small < 2 ** 11
    assert big + small / LO_SCALE < 2 ** 10
    nnz = (w != 0).sum((0, 1))
    assert int(nnz.max()) == min(taps * cin, BUDGET // amax)


def test_reference_is_exact_and_order_free():
    """On the grid the fp64 reference equals an exact rational evaluation (integers scaled by 2^13) in any order,
    and its value and epilogue are fp32 values."""
    p = grid_planes((2, 5, 6, 64), 64, seed=4, lo_from=0)
    w = grid_weights(9, 64, 8, seed=5)
    v = conv_ref(p, 64, w)
    # the same sum in integers: with stored lo = wl / 4 and al / 4, v * 2^13 = 8192 a_hi w_hi + a_hi wl + al w_hi
    hi, lo = split16(w)
    ah = p[0].double().round().long()
    al = (p[1].double() * 4).round().long()
    wh, wl = hi.double().round().long(), (lo.double() * 4).round().long()
    assert torch.equal(ah.double(), p[0].double()) and torch.equal(wl.double(), lo.double() * 4)
    xp = torch.nn.functional.pad(torch.stack([ah, al]), (0, 0, 1, 1, 1, 1))
    acc = torch.zeros(2, 5, 6, 8, dtype=torch.long)
    for t in range(9):
        ky, kx = divmod(t, 3)
        a, l_ = xp[0, :, ky:ky + 5, kx:kx + 6], xp[1, :, ky:ky + 5, kx:kx + 6]
        acc += a @ (wh[t] * 8192) + a @ wl[t] + l_ @ wh[t]
    assert torch.equal(v, acc.double() / 2 ** 13)
    scale, shift = grid_bn(8, 6, "cpu")
    epilogue(v, scale, shift, True)


# ------------------------------------------------------------------------------------------------ GPU: dense conv
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _bn(opt, cout, seed, dev):
    relu, has_scale, has_shift = opt
    scale, shift = grid_bn(cout, seed, dev)
    return relu, (scale if has_scale else None), (shift if has_shift else None)


def _dense(x, w, opt, cout, seed, dev, v=None):
    """Run ops.conv2d_split (both outputs) and compare with the exact reference; returns the outputs."""
    from sassd_b200 import ops
    relu, scale, shift = _bn(opt, cout, seed, dev)
    sp, f32 = ops.conv2d_split(x, w, scale, shift, relu, cout, out_split=True, out_f32=True)
    if v is None:
        v = conv_ref(x.planes, x.channels, w)
    ref = epilogue(v, scale, shift, relu)
    assert sp.planes.shape[-1] == (cout + 63) // 64 * 64
    assert_split_out(sp.planes, ref, cout, "split output")
    assert_f32_out(f32, ref, cout, "fp32 output")
    return sp, f32


@pytest.mark.gpu
@pytest.mark.parametrize("W", [16, 20])
@pytest.mark.parametrize("H", [8, 9, 21])
@pytest.mark.parametrize("layer", sorted(DENSE_LAYERS))
def test_dense_conv_exact_partial_tiles(dev, layer, H, W):
    """Every layer shape on maps with whole and partial tiles, under every epilogue option, bit for bit."""
    from sassd_b200 import ops
    taps, cin, cs, cout = DENSE_LAYERS[layer]
    x = ops.SplitMap(grid_planes((2, H, W, cs), cin, seed=H * 100 + W, device=dev, lo_from=0), cin)
    w = grid_weights(taps, cin, cout, seed=cin + cout + taps).to(dev)
    v = conv_ref(x.planes, cin, w)
    for k, opt in enumerate(OPTIONS):
        _dense(x, w, opt, cout, k, dev, v)


@pytest.mark.gpu
@pytest.mark.parametrize("layer", ["3x3_320_256", "3x3_256_28"])
def test_dense_conv_exact_detector_grid(dev, layer):
    """The detector's 200 x 176 grid at batch 1, 2, 16 and 17 (4400 tiles are ordered in shared memory, 17 frames are
    walked round-robin); the frames are the first B of one 17-frame map, so one reference serves all four."""
    from sassd_b200 import ops
    taps, cin, cs, cout = DENSE_LAYERS[layer]
    planes = grid_planes((17, 200, 176, cs), cin, seed=17, device=dev, lo_from=0)
    w = grid_weights(taps, cin, cout, seed=77).to(dev)
    v = conv_ref(planes, cin, w)
    for B in (1, 2, 16, 17):
        _dense(ops.SplitMap(planes[:, :B].contiguous(), cin), w, OPTIONS[B % 4], cout, B, dev, v[:B])
    del v
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ GPU: tile skipping
def _scatter_input(dev, B, H, W, C, per_frame, seed):
    """A scattered map from grid features: (SplitMap from sparse_to_bev_split, the planes expected of it).  Features
    carry a lo part only beside |hi| = 2, pointing away from zero, so a signed permutation with a shift in {-1, 0, 1}
    keeps them on the grid."""
    from sassd_b200 import ops
    rs = np.random.RandomState(seed)
    cells = []
    for b in range(B):
        flat = rs.choice(H * W, per_frame, replace=False)
        cells += [(b, int(f // W), int(f % W)) for f in flat]
    coors = torch.zeros((len(cells), 4), dtype=torch.int32)
    coors[:, 0] = torch.tensor([c[0] for c in cells])
    coors[:, 2] = torch.tensor([c[1] for c in cells])
    coors[:, 3] = torch.tensor([c[2] for c in cells])
    rows = grid_planes((len(cells), C), C, seed=seed, device=dev, lo_from=2)
    rows[1] = rows[1].abs() * rows[0].sign()      # lo away from zero: +-a + shift never lands just below 1 in magnitude
    feat = planes_value(rows).contiguous()
    d_rows = torch.tensor([len(cells)], dtype=torch.int32, device=dev)
    x = ops.sparse_to_bev_split(feat, coors.to(dev), d_rows, C, 1, H, W, B)
    want = torch.zeros_like(x.planes)
    c = coors.long().to(dev)
    want[:, c[:, 0], c[:, 2], c[:, 3]] = rows
    assert torch.equal(x.planes, want), "sparse_to_bev_split scattered other planes"
    return x, want


def _perm_layer(C, seed, dev):
    """A 3x3 layer with only its centre tap: out[c] = +-in[perm(c)] + shift[c], shift in {-1, 0, 1}."""
    g = torch.Generator().manual_seed(seed)
    perm = torch.randperm(C, generator=g)
    sign = torch.randint(0, 2, (C,), generator=g).float() * 2 - 1
    w = torch.zeros(9, C, C)
    w[4, perm, torch.arange(C)] = sign
    shift = torch.randint(-1, 2, (C,), generator=g).float()
    return w.to(dev), shift.to(dev)


@pytest.mark.gpu
@pytest.mark.parametrize("order", [0, 1])
@pytest.mark.parametrize("B", [1, 16, 17])
def test_tile_skipping_exact(dev, B, order):
    """Constant and background tiles store exactly what computing them gives.  A reach-1 layer on a scattered map
    (its constant is act(shift)); then a centre-tap permutation (output still on the grid) and a reach-2 layer with
    constant interior tiles and background-copied border tiles."""
    from sassd_b200 import ops
    assert ops.TILE_OCCUPANCY
    H, W, C = 200, 176, 64
    order0, ops.CONV2D_TILE_ORDER = ops.CONV2D_TILE_ORDER, order
    try:
        x0, e0 = _scatter_input(dev, B, H, W, C, 40, seed=B)
        wa = grid_weights(9, C, 256, seed=11).to(dev)
        sa, sha = grid_bn(256, 12, dev)
        ya, _ = ops.conv2d_split(x0, wa, sa, sha, True, 256)
        assert ya.reach == 1
        assert torch.equal(ops.conv_constant(None, C, wa, sa, sha, True, 256), sha.clamp_min(0))
        assert_split_out(ya.planes, epilogue(conv_ref(e0, C, wa), sa, sha, True), 256, "reach-1 layer")
        del ya
        wp, shp = _perm_layer(C, 13, dev)
        yp, _ = ops.conv2d_split(x0, wp, None, shp, True, C)
        rp = epilogue(conv_ref(e0, C, wp), None, shp, True)
        assert_split_out(yp.planes, rp, C, "permutation layer")
        ep = torch.stack(split16(rp.float()))
        assert float(ep[0].float().abs().max()) <= 3 and bool((ep[0].float().frac() == 0).all())
        wq = grid_weights(9, C, 256, seed=14, amax=3).to(dev)
        sq, shq = grid_bn(256, 15, dev)
        yq, fq = ops.conv2d_split(yp, wq, sq, shq, True, 256, out_split=True, out_f32=True)
        assert yq.reach == 2 and yq.tile_dist is not None
        rq = epilogue(conv_ref(ep, C, wq), sq, shq, True)
        assert_split_out(yq.planes, rq, 256, "reach-2 layer")
        assert_f32_out(fq, rq, 256, "reach-2 layer")
    finally:
        ops.CONV2D_TILE_ORDER = order0
    kinds = tile_kinds(x0.tile_dist.view(B, H // TH, W // TW).cpu().numpy()[0], 2)
    assert {0, 1, 2} <= set(np.unique(kinds).tolist()), "the map lacks computed, constant or background tiles"


# ------------------------------------------------------------------------------------------------ GPU: sparse conv
_TABLES = {}


def _lidar_tables(B, dev):
    """Neighbour tables of synthetic LiDAR frames (rulebook_subm on the voxels, rulebook_conv to the next level)."""
    if B not in _TABLES:
        from oracle import ref_pipeline as O
        from sassd_b200 import ops, spconv
        from sassd_b200.synth import synth_cloud
        cl = []
        for b in range(B):
            _, c, _ = O.points_to_voxel(synth_cloud(b, fov_deg=20.0, az_step_deg=0.3456), [0.05, 0.05, 0.1],
                                        [0, -40., -3., 70.4, 40., 1.], 5, 20000)
            cl.append(np.pad(c, ((0, 0), (1, 0)), constant_values=b))
        coords = torch.from_numpy(np.concatenate(cl, 0).astype(np.int32)).to(dev)
        shape = [40, 1600, 1408]
        x = spconv.SparseConvTensor(torch.zeros((coords.shape[0], 4), device=dev), coords, shape, B)
        nbr, tm = ops.rulebook_subm(x._indices, x.d_rows, shape, x.hash_index())
        n = coords.shape[0]
        cap = 2 * n
        _, dn, nbr2, _, tm2 = ops.rulebook_conv(x._indices, x.d_rows, B, shape, x.hash_index(), cap, x.status)
        x.check_status()
        _TABLES[B] = {"subm": (nbr, tm, n, n, x.d_rows, n), "conv": (nbr2, tm2, n, cap, dn, int(dn.item()))}
    return _TABLES[B]


def _hand_table(rows_cap, in_rows, n_rows, seed, absent=0.75, full_every=7, density=0.3, keep_all=False):
    """A hand-built neighbour table [rows_cap, 27] with taps absent from whole tiles, and its tile masks."""
    rs = np.random.RandomState(seed)
    nb = np.where(rs.rand(rows_cap, 27) < density, rs.randint(0, in_rows, (rows_cap, 27)), -1).astype(np.int32)
    nt = (rows_cap + 127) // 128
    gone = rs.rand(nt, 27) < (0.0 if keep_all else absent)
    if full_every:
        gone[::full_every] = False
    nb[np.repeat(gone, 128, axis=0)[:rows_cap]] = -1
    return nb, _tile_masks(nb, n_rows)


def _sparse_runs(dev, planes, w, cout, rows_cap, nbr, tm, d_rows, n, opt, seed, configs):
    """ops.spconv_split under each (tap skipping, chunk deal) config; every result equals the exact reference."""
    from sassd_b200 import ops
    relu, scale, shift = _bn(opt, cout, seed, dev)
    ref = epilogue(rows_ref(planes, w.shape[1], w, nbr, n), scale, shift, relu)
    saved = ops.SPCONV_TAP_SKIP, ops.SPCONV_TAP_SPLIT
    outs = {}
    try:
        for skip, split in configs:
            ops.SPCONV_TAP_SKIP, ops.SPCONV_TAP_SPLIT = skip, split
            out, of = ops.spconv_split(planes, w, scale, shift, relu, cout, rows_cap, nbr=nbr, d_rows=d_rows,
                                       want_f32=True, tile_mask=tm)
            what = "skip=%d deal=%d" % (skip, split)
            assert_split_out(out[:, :n], ref, cout, what)
            assert_f32_out(of[:n], ref, cout, what)
            outs[(skip, split)] = (out[:, :n], of[:n])
    finally:
        ops.SPCONV_TAP_SKIP, ops.SPCONV_TAP_SPLIT = saved
    return outs, ref


_ALL_CONFIGS = [(True, True), (True, False), (False, True), (False, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("table", ["subm", "conv"])
@pytest.mark.parametrize("B", [1, 16])
@pytest.mark.parametrize("pair", SPARSE_PAIRS, ids=["%d(%d)-%d" % p for p in SPARSE_PAIRS])
def test_sparse_conv_exact_lidar_tables(dev, pair, B, table):
    """Every backbone channel pair on the rulebooks of synthetic LiDAR frames, with tile masks and chunk deal on and
    off: each result equals the reference, so the dealt one equals the undealt one bit for bit."""
    cin, cs, cout = pair
    nbr, tm, in_rows, rows_cap, d_rows, n = _lidar_tables(B, dev)[table]
    planes = grid_planes((in_rows, cs), cin, seed=cin * 10 + cout + B, device=dev, lo_from=0)
    w = grid_weights(27, cin, cout, seed=cin * 100 + cout).to(dev)
    _sparse_runs(dev, planes, w, cout, rows_cap, nbr, tm, d_rows, n, OPTIONS[(cin + cout) % 4], cin, _ALL_CONFIGS)


@pytest.mark.gpu
def test_sparse_conv_exact_1x1(dev):
    from sassd_b200 import ops
    rows_cap, n = 5 * 128 - 3, 4 * 128 + 7
    planes = grid_planes((rows_cap, 64), 64, seed=5, device=dev, lo_from=0)
    w = grid_weights(1, 64, 64, seed=6).to(dev)
    d_rows = torch.tensor([n], dtype=torch.int32, device=dev)
    for k, opt in enumerate(OPTIONS):
        relu, scale, shift = _bn(opt, 64, k, dev)
        out, of = ops.spconv_split(planes, w, scale, shift, relu, 64, rows_cap, d_rows=d_rows, want_f32=True)
        ref = epilogue(rows_ref(planes, 64, w, None, n), scale, shift, relu)
        assert_split_out(out[:, :n], ref, 64, "1x1")
        assert_f32_out(of[:n], ref, 64, "1x1")


def _grid_ctas():
    return min(torch.cuda.get_device_properties(0).multi_processor_count, 148)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["1", "G-1", "G", "G+1", "one_tile"])
def test_sparse_chunk_deal_exact(dev, which):
    """The chunk deal at 1, G-1, G and G+1 tiles and one tile over many CTAs, on hand-built tables with absent taps:
    dealt and undealt results both equal the reference."""
    G = _grid_ctas()
    ntiles = {"1": 1, "G-1": G - 1, "G": G, "G+1": G + 1, "one_tile": 1}[which]
    rows_cap = ntiles * 128 - (8 if which == "one_tile" else 5)
    n = rows_cap
    nb, masks = _hand_table(rows_cap, rows_cap, n, seed=ntiles, keep_all=which == "one_tile")
    counts = [len(active_chunks(int(m), 1, 27)) for m in masks]
    assert takes_deal(counts, min(ntiles * 27, G)) == (ntiles <= G), "the table does not exercise the deal"
    planes = grid_planes((rows_cap, 64), 64, seed=ntiles + 1, device=dev, lo_from=0)
    w = grid_weights(27, 64, 64, seed=ntiles + 2).to(dev)
    d_rows = torch.tensor([n], dtype=torch.int32, device=dev)
    _sparse_runs(dev, planes, w, 64, rows_cap, torch.from_numpy(nb).to(dev), torch.from_numpy(masks).to(dev), d_rows,
                 n, OPTIONS[0], 3, [(True, True), (True, False)])


# ------------------------------------------------------------------------------------------------ GPU: gathered GEMM
def _gconv(inp, w, scale, shift, relu, cout, mode, precision, taps, nbr=None, d_rows=None, B=0, H=0, W=0):
    from sassd_b200 import ops
    rows = inp.numel() // inp.shape[-1]
    out = torch.full((rows, cout), float("nan"), device=inp.device)
    m = {"table": ops.GCONV_TABLE, "conv2d": ops.GCONV_CONV2D, "rows": ops.GCONV_ROWS}[mode]
    ops.gconv(inp, w, scale, shift, out, mode=m, taps=taps, cin=inp.shape[-1], cout=cout, relu=relu, nbr=nbr,
              d_rows=d_rows, rows_cap=rows, batch=B, H=H, W=W, precision=precision)
    return out


def _gconv_case(dev, mode, coarse):
    """Operands of one gconv mode: (planes, weights, taps, extra kwargs, reference before the epilogue)."""
    seed = {"table": 1, "conv2d": 2, "rows": 3}[mode] + (10 if coarse else 0)
    amax = 1 if coarse else AMAX
    if mode == "conv2d":
        B, H, W, cin, cout, taps = 2, 21, 20, 128, 72, 9
        planes = grid_planes((B, H, W, cin), cin, seed, dev, coarse=coarse)
        w = grid_weights(taps, cin, cout, seed, amax=amax, coarse=coarse).to(dev)
        return planes, w, cout, dict(taps=taps, B=B, H=H, W=W), conv_ref(planes, cin, w).view(-1, cout)
    rows, cin, cout = 3 * 128 - 11, 64, 64
    planes = grid_planes((rows, cin), cin, seed, dev, coarse=coarse)
    if mode == "rows":
        w = grid_weights(1, cin, cout, seed, amax=amax, coarse=coarse).to(dev)
        d_rows = torch.tensor([rows], dtype=torch.int32, device=dev)
        return planes, w, cout, dict(taps=1, d_rows=d_rows), rows_ref(planes, cin, w, None, rows)
    nb, _ = _hand_table(rows, rows, rows, seed, absent=0.3)
    nbr = torch.from_numpy(nb).to(dev)
    w = grid_weights(27, cin, cout, seed, amax=amax, coarse=coarse).to(dev)
    d_rows = torch.tensor([rows], dtype=torch.int32, device=dev)
    return planes, w, cout, dict(taps=27, nbr=nbr, d_rows=d_rows), rows_ref(planes, cin, w, nbr, rows)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["table", "conv2d", "rows"])
def test_gconv_coarse_grid_all_precisions(dev, mode):
    """On fp16-exact operands with lo = 0, FFMA, 3xTF32 and 3xFP16 give the reference's bits."""
    from sassd_b200 import ops
    planes, w, cout, kw, v = _gconv_case(dev, mode, coarse=True)
    scale, shift = grid_bn(cout, 4, dev)
    ref = epilogue(v, scale, shift, True)
    inp = planes_value(planes).contiguous()
    for prec in (ops.PREC_FP32, ops.PREC_TF32X3, ops.PREC_F16X3):
        assert_f32_out(_gconv(inp, w, scale, shift, True, cout, mode, prec, **kw), ref, cout, "gconv prec %d" % prec)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["table", "conv2d", "rows"])
def test_gconv_split_grid_matches_split_kernels(dev, mode):
    """On the split grid 3xTF32 and 3xFP16 give the reference's bits, and so do the TMA conv (conv2d mode) and the
    split-row conv (table and rows modes) on the same operands."""
    from sassd_b200 import ops
    planes, w, cout, kw, v = _gconv_case(dev, mode, coarse=False)
    scale, shift = grid_bn(cout, 5, dev)
    ref = epilogue(v, scale, shift, False)
    inp = planes_value(planes).contiguous()
    for prec in (ops.PREC_TF32X3, ops.PREC_F16X3):
        assert_f32_out(_gconv(inp, w, scale, shift, False, cout, mode, prec, **kw), ref, cout, "gconv prec %d" % prec)
    if mode == "conv2d":
        x = ops.SplitMap(planes, planes.shape[-1])
        _, f32 = ops.conv2d_split(x, w, scale, shift, False, cout, out_split=False, out_f32=True)
        assert_f32_out(f32.view(-1, f32.shape[-1]), ref, cout, "TMA conv")
    else:
        rows = planes.shape[1]
        _, of = ops.spconv_split(planes, w, scale, shift, False, cout, rows, nbr=kw.get("nbr"),
                                 d_rows=kw["d_rows"], want_f32=True)
        assert_f32_out(of, ref, cout, "split-row conv")


# ------------------------------------------------------------------------------------------------ GPU: sensitivity
def _nudge(w, col, tap, seed):
    """w with one nonzero weight of column `col` moved by 2^-13 (its stored lo by 1/4): (w', channel, step)."""
    rs = np.random.RandomState(seed)
    cands = torch.nonzero(w[tap, :, col] != 0).view(-1).cpu().numpy()
    assert len(cands), "fixture: no nonzero weight at that tap and column"
    c = int(rs.choice(cands))
    i = float(torch.round(w[tap, c, col]))
    j = round((float(w[tap, c, col]) - i) * 2 ** 13)
    step = 1 if j <= 0 else -1
    w2 = w.clone()
    w2[tap, c, col] = i + (j + step) * 2.0 ** -13
    hi, lo = split16(w2[tap, c, col].view(1).float())
    assert float(hi) == i and float(lo) == (j + step) / 4
    return w2, c, step


@pytest.mark.gpu
def test_one_weight_lo_step_moves_one_dense_column(dev):
    """One stored w_lo entry moved by 1/4 at (corner tap, channel of the second chunk, column of the second unit):
    that column moves by exactly a_hi * 2^-13 * scale, with a_hi the input the tap reads; every other bit stays."""
    from sassd_b200 import ops
    B, H, W, C, cout, tap, col = 2, 21, 20, 256, 256, 0, 200
    x = ops.SplitMap(grid_planes((B, H, W, C), C, seed=21, device=dev, lo_from=0), C)
    w = grid_weights(9, C, cout, seed=22).to(dev)
    scale, shift = grid_bn(cout, 23, dev)
    w2, c, step = _nudge(w, col, tap, 24)
    sp1, f1 = ops.conv2d_split(x, w, scale, shift, False, cout, out_split=True, out_f32=True)
    sp2, f2 = ops.conv2d_split(x, w2, scale, shift, False, cout, out_split=True, out_f32=True)
    ky, kx = divmod(tap, 3)
    a = torch.nn.functional.pad(x.planes[0, ..., c].double(), (1, 1, 1, 1))[:, ky:ky + H, kx:kx + W]
    want = a * step * 2.0 ** -13 * float(scale[col])
    assert bool((want != 0).any())
    assert torch.equal(f2[..., col].double() - f1[..., col].double(), want)
    others = torch.arange(cout, device=dev) != col
    assert torch.equal(f1[..., others], f2[..., others])
    assert torch.equal(sp1.planes[..., others], sp2.planes[..., others])
    assert_f32_out(f1, epilogue(conv_ref(x.planes, C, w), scale, shift, False), cout, "before the nudge")


@pytest.mark.gpu
def test_one_weight_lo_step_moves_one_sparse_column(dev):
    """The same through the split-row conv's table: rows without a neighbour at that tap keep their bits."""
    from sassd_b200 import ops
    rows, C, cout, tap, col = 3 * 128 - 7, 64, 64, 26, 37
    nb, masks = _hand_table(rows, rows, rows, seed=31, absent=0.3)
    nbr = torch.from_numpy(nb).to(dev)
    planes = grid_planes((rows, C), C, seed=32, device=dev, lo_from=0)
    w = grid_weights(27, C, cout, seed=33).to(dev)
    scale, shift = grid_bn(cout, 34, dev)
    w2, c, step = _nudge(w, col, tap, 35)
    d_rows = torch.tensor([rows], dtype=torch.int32, device=dev)
    tm = torch.from_numpy(masks).to(dev)
    o1, f1 = ops.spconv_split(planes, w, scale, shift, False, cout, rows, nbr=nbr, d_rows=d_rows, want_f32=True,
                              tile_mask=tm)
    o2, f2 = ops.spconv_split(planes, w2, scale, shift, False, cout, rows, nbr=nbr, d_rows=d_rows, want_f32=True,
                              tile_mask=tm)
    src = nbr[:, tap].long()
    a = torch.where(src >= 0, planes[0, src.clamp_min(0), c].double(), torch.zeros((), dtype=torch.float64, device=dev))
    want = a * step * 2.0 ** -13 * float(scale[col])
    assert bool((want != 0).any()) and bool((want == 0).any())
    assert torch.equal(f2[:, col].double() - f1[:, col].double(), want)
    others = torch.arange(cout, device=dev) != col
    assert torch.equal(f1[:, others], f2[:, others]) and torch.equal(o1[..., others], o2[..., others])


# ------------------------------------------------------------------------------------------------ GPU: a full small sum
def _saturated(planes, w, ncols=4):
    """Planes hi = 2, lo = 3/4 in every valid channel and ncols columns of BUDGET // AMAX - 1 weights 1 + 2^-13: each
    term adds 1.25 to the small accumulator, which reaches 561.25 - a quarter above 512, where fp16 holds only halves
    (the column bound still holds: 2 * 449 <= BUDGET)."""
    planes[0][planes[0] != 0] = 2
    planes[1][planes[0] != 0] = 0.75
    g = torch.Generator().manual_seed(3)
    taps, cin, _ = w.shape
    nnz = BUDGET // AMAX - 1
    for n in range(ncols):
        col = torch.zeros(taps * cin)
        col[torch.randperm(taps * cin, generator=g)[:nnz]] = 1 + 2.0 ** -13
        w[:, :, n] = col.view(taps, cin).to(w.device)
    return planes, w


@pytest.mark.gpu
def test_small_accumulator_keeps_quarters_past_512_dense(dev):
    from sassd_b200 import ops
    planes = grid_planes((1, 9, 20, 320), 320, seed=61, device=dev, lo_from=0)
    planes[0, ..., :320] = 1
    planes, w = _saturated(planes, grid_weights(9, 320, 256, seed=62).to(dev))
    x = ops.SplitMap(planes, 320)
    v = conv_ref(planes, 320, w)
    assert float(v[0, 4, 8, 0]) == 898 + 561.25 / LO_SCALE
    _dense(x, w, OPTIONS[1], 256, 63, dev, v)


@pytest.mark.gpu
def test_small_accumulator_keeps_quarters_past_512_sparse(dev):
    rows = 2 * 128 - 9
    nb, masks = _hand_table(rows, rows, rows, seed=71, density=1.0, keep_all=True)
    planes = grid_planes((rows, 64), 64, seed=72, device=dev, lo_from=0)
    planes[0, :, :64] = 1
    planes, w = _saturated(planes, grid_weights(27, 64, 64, seed=73).to(dev))
    d_rows = torch.tensor([rows], dtype=torch.int32, device=dev)
    _sparse_runs(dev, planes, w, 64, rows, torch.from_numpy(nb).to(dev), torch.from_numpy(masks).to(dev), d_rows,
                 rows, OPTIONS[1], 74, [(True, True), (True, False)])


# ------------------------------------------------------------------------------------------------ GPU: ABI write guards
@pytest.mark.gpu
@pytest.mark.parametrize("cout", [20, 28])
def test_conv2d_abi_writes_zero_channels_into_nan_buffers(dev, cout):
    """sassd_conv2d_f16x3_occ_bg with out_split_ch = 64 > cout into buffers full of NaN, with computed, constant and
    background tiles: channels [cout, 64) of every pixel read zero (the header's promise), the rest is exact."""
    from sassd_b200 import ops
    B, H, W, C = 2, 56, 80, 64
    x0, e0 = _scatter_input(dev, B, H, W, C, 2, seed=41)
    wp, shp = _perm_layer(C, 42, dev)
    yp, _ = ops.conv2d_split(x0, wp, None, shp, True, C)
    ep = torch.stack(split16(epilogue(conv_ref(e0, C, wp), None, shp, True).float()))
    w = grid_weights(9, C, cout, seed=43, amax=3).to(dev)
    scale, shift = grid_bn(cout, 44, dev)
    reach = yp.reach + 1
    cvec = ops.conv_constant(yp.const, C, w, scale, shift, True, cout)
    bg_sp, bg_f = ops.conv_background(yp, w, scale, shift, True, cout, True, True)
    stride = (cout + 3) // 4 * 4
    osp = torch.full((2, B, H, W, 64), float("nan"), dtype=torch.float16, device=dev)
    of = torch.full((B, H, W, stride), float("nan"), device=dev)
    d = ops.Conv2dDesc()
    d.batch, d.H, d.W, d.cin, d.cin_stored = B, H, W, C, C
    d.cout, d.taps, d.relu, d.out_f32_stride, d.out_split_ch = cout, 9, 1, stride, 64
    wpk = ops.tc_pack_cached(w, ops.PREC_F16X3)
    ops._call("sassd_conv2d_f16x3_occ_bg", None, ctypes.byref(d), ops._ptr(yp.planes), ops._ptr(wpk), ops._ptr(scale),
              ops._ptr(shift), ops._ptr(of), ops._ptr(osp), ops._ptr(yp.tile_dist), reach, ops._ptr(cvec),
              ops._ptr(bg_sp.planes), ops._ptr(bg_f), ops._ptr(None), ops._stream())
    torch.cuda.synchronize()
    kinds = np.concatenate([tile_kinds(dd, reach).ravel()
                            for dd in yp.tile_dist.view(B, H // TH, W // TW).cpu().numpy()])
    assert {0, 1, 2} <= set(np.unique(kinds).tolist()), "the map lacks computed, constant or background tiles"
    assert bool((bg_sp.planes[..., cout:] == 0).all()), "the background map's stored channels past cout"
    ref = epilogue(conv_ref(ep, C, w), scale, shift, True)
    assert_split_out(osp, ref, cout, "ABI call")
    assert_f32_out(of, ref, cout, "ABI call")


@pytest.mark.gpu
@pytest.mark.parametrize("deal", [True, False])
@pytest.mark.parametrize("out_ch", [32, 64])
def test_spconv_abi_writes_zero_channels_and_keeps_rows(dev, out_ch, deal):
    """sassd_spconv_f16x3 with cout 16 and out_ch > 16 into buffers full of NaN: channels [16, out_ch) of the live rows
    read zero, the rows at and past *d_rows keep their NaN, and the live rows are exact (one tile, dealt over many
    CTAs with the workspace)."""
    from sassd_b200 import ops
    rows_cap, n, C, cout = 2 * 128, 120, 64, 16
    nb, masks = _hand_table(rows_cap, rows_cap, n, seed=51, keep_all=True)
    nbr, tm = torch.from_numpy(nb).to(dev), torch.from_numpy(masks).to(dev)
    planes = grid_planes((rows_cap, C), C, seed=52, device=dev, lo_from=0)
    w = grid_weights(27, C, cout, seed=53).to(dev)
    scale, shift = grid_bn(cout, 54, dev)
    d_rows = torch.tensor([n], dtype=torch.int32, device=dev)
    out = torch.full((2, rows_cap, out_ch), float("nan"), dtype=torch.float16, device=dev)
    of = torch.full((rows_cap, cout), float("nan"), device=dev)
    d = ops.SpconvDesc()
    d.cin, d.cout, d.taps, d.rows_cap, d.in_rows_cap = C, cout, 27, rows_cap, rows_cap
    d.relu, d.out_ch, d.out_f32_stride = 1, out_ch, cout
    wpk = ops.spconv_pack_cached(w, C)
    ws = torch.zeros(ops._L().sassd_spconv_workspace_bytes(), dtype=torch.uint8, device=dev) if deal else None
    ops._call("sassd_spconv_f16x3", None, ctypes.byref(d), ops._ptr(planes), ops._ptr(wpk), ops._ptr(scale),
              ops._ptr(shift), ops._ptr(nbr), ops._ptr(tm), ops._ptr(d_rows), ops._ptr(out), ops._ptr(of),
              ops._ptr(ws), 0 if ws is None else ws.numel(), ops._ptr(None), ops._stream())
    torch.cuda.synchronize()
    assert bool(torch.isnan(out[:, n:]).all()) and bool(torch.isnan(of[n:]).all()), "rows past *d_rows were written"
    ref = epilogue(rows_ref(planes, C, w, nbr, n), scale, shift, True)
    assert_split_out(out[:, :n], ref, cout, "ABI call")
    assert_f32_out(of[:n], ref, cout, "ABI call")
