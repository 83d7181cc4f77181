"""The 3xFP16 convolutions across the whole fp16 range.

Every tensor-core conv stores its activations as the split hi = half(x), lo = half((x - hi) * 2048) and reads them as
hi + lo / 2048.  The other tests feed O(1) data and scale their tolerance by the largest output; here:

* the split's own error on a log sweep and at its edge values (CPU);
* every store of split planes (the constant tile, the BN = 128 staged epilogue, the BN <= 64 register epilogue, the
  sparse-to-BEV scatter, the sparse conv's epilogue, fp32 rows to split) is numpy's split of its fp32 value, bit for
  bit, on outputs from 2^-40 to 2^15 and exactly on the edge values;
* the result against fp64 per element with a condition-aware bound, and two operand changes the bound must catch;
* the range contract: a finite value at or above 65520 sets SASSD_FLAG_F16_RANGE at every site and the step raises;
* NaN through the convs: NaN exactly where the receptive field holds it, everything else unchanged.

Error of the split (x fp32, hi = half_rn(x), r = x - hi exact in fp32, lo = half_rn(2048 r)):

* 2^-14 <= |x| < 65520: hi is a normal half, |r| <= ulp16(x) / 2 = 2^(e-11) for |x| in [2^e, 2^(e+1)).  2048 r is a
  real of magnitude <= 2^e; its half rounding errs by at most 2^-11 of it when it is normal (|2048 r| >= 2^-14), so
  the reconstruction errs by |r| 2^-11 <= 2^(e-22) - with |x| >= 2^e that is 2^-22 |x|, and a closer count (|r| <= 2^(e-11)
  with 2048 r landing below the half's next power of two) gives 2^-23 |x| for |x| >= 2^-3, where 2048 r >= 2^-14
  whenever r != 0 (checked on 2M values).  Below 2^-3, 2048 r can be a half subnormal (spacing 2^-24): the absolute
  error is then 2^-25 / 2048 = 2^-36, which stays below 2^-22 |x| down to |x| = 2^-14.
* |x| < 2^-14: hi is subnormal or zero with spacing 2^-24, |r| <= 2^-25, 2048 r <= 2^-14 rounds with spacing 2^-24:
  error <= 2^-25 / 2048 = 2^-36 absolute.
* |x| >= 65520 rounds to inf: hi = +-inf, lo = -+inf, and the next conv's big + small / 2048 is NaN."""
import numpy as np
import pytest
import torch

from tests.test_tc_exact import DENSE_LAYERS, SPARSE_PAIRS, split16_np

LO = 2048.0
F16_RANGE = 512
EDGES = np.array([2.0 ** -25, 2.0 ** -24, 2.0 ** -14, 65504.0, 65519.99, -65519.99, 0.0, 1.0, -3.0], np.float32)
OVER = np.array([65520.0, -65520.0, 1e5], np.float32)
# per-element accuracy bound: TOL_REL * sum |a| |w| |scale| + SPLIT_FLOOR * (sum |a| + sum |w|) |scale| + TOL_ABS.
# TOL_REL as the max-scaled tests use; SPLIT_FLOOR is the split's absolute error below 2^-14 (an operand there keeps
# fewer than 22 bits, see the module docstring), which the relative term cannot cover.
TOL_REL, SPLIT_FLOOR, TOL_ABS = 2e-5, 2.0 ** -36, 2.0 ** -30


def recon(hi, lo):
    return hi.astype(np.float64) + lo.astype(np.float64) / LO


def split_bound(x):
    """The bound of the module docstring for |x| < 65520."""
    a = np.abs(x.astype(np.float64))
    return np.where(a >= 2.0 ** -3, 2.0 ** -23 * a, np.where(a >= 2.0 ** -14, 2.0 ** -22 * a, 2.0 ** -36))


# ------------------------------------------------------------------------------------------------ CPU: the split
def test_split_error_bounds_on_a_log_sweep():
    rs = np.random.RandomState(0)
    mag = np.exp2(rs.uniform(-40, np.log2(65519.99), 2_000_000)).astype(np.float32)
    x = np.concatenate([mag, -mag, np.float32([65519.99, -65519.99])])
    x = x[np.abs(x) < 65520]
    hi, lo = split16_np(x)
    assert np.isfinite(hi).all() and np.isfinite(lo).all()
    err = np.abs(x.astype(np.float64) - recon(hi, lo))
    bound = split_bound(x)
    assert (err <= bound).all(), "split error above the bound at %s" % x[err > bound][:4]
    # each range is populated and its bound is tight to within a factor of 4 (a loose bound would hide a broken split)
    a = np.abs(x)
    for lo_e, hi_e in ((-3, 16.1), (-14, -3), (-40, -14)):
        sel = (a >= 2.0 ** lo_e) & (a < 2.0 ** hi_e)
        assert sel.sum() > 1000 and (err[sel] / bound[sel]).max() > 0.25


def test_split_edge_values():
    def one(v):
        hi, lo = split16_np(np.float32([v]))
        return hi[0], lo[0]
    hi, lo = one(2.0 ** -25)                      # half of the least subnormal: hi ties to 0, lo carries it all
    assert hi == 0 and lo == np.float16(2.0 ** -14) and recon(hi, lo) == 2.0 ** -25
    assert one(2.0 ** -24) == (np.float16(2.0 ** -24), 0) and one(2.0 ** -14) == (np.float16(2.0 ** -14), 0)
    assert one(65504.0) == (np.float16(65504), 0)
    hi, lo = one(65519.99)
    assert hi == np.float16(65504) and np.isfinite(lo) and abs(recon(hi, lo) - float(np.float32(65519.99))) <= 2.0 ** -8
    hi, lo = one(65520.0)
    assert hi == np.inf and lo == -np.inf and np.isnan(hi.astype(np.float64) + lo.astype(np.float64) / LO)
    hi, lo = one(-65520.0)
    assert hi == -np.inf and lo == np.inf
    hi, lo = one(-0.0)
    assert hi == 0 and np.signbit(hi) and lo == 0 and not np.signbit(lo)
    hi, lo = one(0.0)
    assert hi == 0 and not np.signbit(hi) and lo == 0 and not np.signbit(lo)
    hi, lo = one(np.inf)                          # inf - inf: an infinite input splits into (inf, NaN)
    assert hi == np.inf and np.isnan(lo)
    hi, lo = one(np.nan)
    assert np.isnan(hi) and np.isnan(lo)


def test_status_names_f16_range_and_points_to_fp32():
    from sassd_b200 import lib
    assert lib.FLAGS[F16_RANGE] == "F16_RANGE" and lib.F16_RANGE == F16_RANGE
    with pytest.raises(lib.SassdError, match="F16_RANGE.*PREC_FP32"):
        lib.raise_on_status(F16_RANGE | 2)
    with pytest.raises(lib.SassdError, match="ROWS_CAP"):
        lib.raise_on_status(2)


def test_weight_packs_refuse_out_of_range_weights():
    from sassd_b200 import ops
    w = torch.zeros(9, 64, 32)
    ops.check_f16_weight(w, "layer")
    w[3, 5, 7] = 65519.99
    ops.check_f16_weight(w, "layer")
    w[3, 5, 7] = float(np.nextafter(np.float32(65520.0), np.float32(0)))    # the largest fp32 below the edge
    ops.check_f16_weight(w, "layer")
    w[3, 5, 7] = 65520.0
    with pytest.raises(ValueError, match="conv2d_tma.*65520"):
        ops.check_f16_weight(w, "conv2d_tma[taps=9 64->32]")
    w[3, 5, 7] = -1e5
    with pytest.raises(ValueError):
        ops.check_f16_weight(w, "x")


# ------------------------------------------------------------------------------------------------ GPU fixtures
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _status(dev):
    return torch.zeros((1,), dtype=torch.int32, device=dev)


def _flag(status):
    return bool(int(status.item()) & F16_RANGE)


def _assert_split_of(planes, f32, cout, what):
    """Split planes [2, ..., Cs]: channels < cout are numpy's split of the fp32 values bit for bit, the rest zero."""
    f = f32[..., :cout].contiguous().cpu().numpy()
    hi, lo = split16_np(f)
    for k, want in enumerate((hi, lo)):
        got = planes[k, ..., :cout].cpu().numpy()
        differ = (got.view(np.uint16) != want.view(np.uint16)) & ~(np.isnan(got) & np.isnan(want))   # any NaN bits
        if differ.any():
            bad = np.argwhere(differ)[:4]
            raise AssertionError("%s: %s plane differs at %s: fp32 %s, got %s, want %s" % (
                what, ("hi", "lo")[k], bad.tolist(), [f[tuple(i)] for i in bad], [got[tuple(i)] for i in bad],
                [want[tuple(i)] for i in bad]))
    assert bool((planes[..., cout:] == 0).all()), "%s: stored channels past cout are not zero" % what


def _range_bn(cout, dev, edges):
    """Per-channel epilogue: power-of-two scales 2^-40 .. 2^12 on most channels (outputs of O(1) convs up to ~2^15); on
    every 7th channel scale 0 and a shift from ``edges``, so that its outputs are exactly that value."""
    scale = torch.tensor([2.0 ** (-40 + (c * 11) % 53) for c in range(cout)], dtype=torch.float32)
    shift = torch.zeros(cout)
    for k, c in enumerate(range(3, cout, 7)):
        scale[c] = 0.0
        shift[c] = float(edges[k % len(edges)])
    return scale.to(dev), shift.to(dev)


def _rand_split_map(dev, B, H, W, cin, seed, scale=1.0):
    from sassd_b200 import ops
    g = torch.Generator(device=dev).manual_seed(seed)
    return ops.SplitMap.from_float(torch.randn((B, H, W, cin), generator=g, device=dev) * scale)


def _rand_weight(dev, taps, cin, cout, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    return (torch.randn((taps, cin, cout), generator=g, device=dev) / np.sqrt(taps * cin)).contiguous()


def _finite_below(f):
    return bool((f.abs() < 65520).all())


# ------------------------------------------------------------------------------------------------ GPU: split stores
@pytest.mark.gpu
@pytest.mark.parametrize("cout", [256, 96, 72, 64, 28, 20])
def test_dense_epilogue_stores_the_split_of_its_fp32_output(dev, cout):
    """BN = 128 staged epilogue (cout 256, 96, 72) and BN <= 64 register epilogue (64, 28, 20): with out_f32 and
    out_split together, the planes are numpy's split of the fp32 outputs on every pixel and channel, from 2^-40 to the
    edge of the range; a value past the edge flags F16_RANGE, a value at 65519.99 does not."""
    from sassd_b200 import ops
    taps = 9 if cout in (256, 28) else 1
    x = _rand_split_map(dev, 2, 19, 37, 256, seed=cout)
    w = _rand_weight(dev, taps, 256, cout, seed=cout + 1)
    for relu in (False, True):
        scale, shift = _range_bn(cout, dev, EDGES)
        x.status = st = _status(dev)
        sp, f32 = ops.conv2d_split(x, w, scale, shift, relu, cout, out_split=True, out_f32=True)
        assert _finite_below(f32) and float(f32[..., :cout].abs().max()) > 2.0 ** 11
        assert float(f32[f32 != 0].abs().min()) < 2.0 ** -30
        _assert_split_of(sp.planes, f32, cout, "cout %d relu %d" % (cout, relu))
        assert not _flag(st), "a finite value below 65520 flagged F16_RANGE"
        if not relu:
            assert bool((f32[..., 3] == float(EDGES[0])).all()) and bool((f32[..., 3 + 7 * 4] == 65519.99).all()) \
                if cout > 31 else bool((f32[..., 3] == float(EDGES[0])).all())
        scale, shift = _range_bn(cout, dev, OVER)
        x.status = st = _status(dev)
        sp, f32 = ops.conv2d_split(x, w, scale, shift, relu, cout, out_split=True, out_f32=True)
        _assert_split_of(sp.planes, f32, cout, "cout %d relu %d past the edge" % (cout, relu))
        finite_over = bool(((f32[..., :cout].abs() >= 65520) & torch.isfinite(f32[..., :cout])).any())
        assert finite_over and _flag(st), "a finite value past 65520 did not flag F16_RANGE"
        # the fp32-only store does not flag: nothing is split
        x.status = st = _status(dev)
        ops.conv2d_split(x, w, scale, shift, relu, cout, out_split=False, out_f32=True)
        assert not _flag(st)
    x.status = None


def _scatter(dev, B, H, W, C, per_frame, seed, values=None):
    """Rows scattered into a BEV map: (feat [rows, C], coors [rows, 4], d_rows)."""
    rs = np.random.RandomState(seed)
    cells = []
    for b in range(B):
        for f in rs.choice(H * W, per_frame, replace=False):
            cells.append((b, 0, int(f // W), int(f % W)))
    coors = torch.tensor(cells, dtype=torch.int32, device=dev)
    if values is None:
        mag = np.exp2(rs.uniform(-40, 15, (len(cells), C))) * np.sign(rs.randn(len(cells), C))
        values = mag.astype(np.float32)
    feat = torch.from_numpy(np.asarray(values, np.float32)).to(dev).contiguous()
    return feat, coors, torch.tensor([len(cells)], dtype=torch.int32, device=dev)


@pytest.mark.gpu
@pytest.mark.parametrize("cout", [256, 64])
def test_constant_and_background_tiles_store_the_split_of_their_value(dev, cout):
    """With tile skipping on a scattered map, the constant tiles (store_constant_unit when only split planes are
    stored), the background tiles and the computed tiles all hold numpy's split of the fp32 output of the same layer
    run with both outputs, bit for bit; the constant vector lands exactly on the edge values (scale 0 channels).  A
    constant past the edge flags F16_RANGE from the constant stores alone."""
    from sassd_b200 import ops
    assert ops.TILE_OCCUPANCY
    B, H, W, C = 2, 200, 176, 64
    feat, coors, d_rows = _scatter(dev, B, H, W, C, 30, seed=cout)
    feat = feat.clamp(-8, 8)
    x0 = ops.sparse_to_bev_split(feat, coors, d_rows, C, 1, H, W, B)
    w = _rand_weight(dev, 9, C, cout, seed=5)
    for edges, over in ((EDGES, False), (OVER, True)):
        scale, shift = _range_bn(cout, dev, edges)
        shift = torch.where(scale == 0, shift, torch.full_like(shift, 0.5))
        x0.status = st1 = _status(dev)
        y1, _ = ops.conv2d_split(x0, w, scale, shift, False, cout, out_split=True, out_f32=False)
        x0.status = st2 = _status(dev)
        y2, f2 = ops.conv2d_split(x0, w, scale, shift, False, cout, out_split=True, out_f32=True)
        _assert_split_of(y2.planes, f2, cout, "both outputs")
        _assert_split_of(y1.planes, f2, cout, "split output only (constant tile stores)")
        assert _flag(st1) == over and _flag(st2) == over
        # a second layer at reach 2: background-copied border tiles
        if not over:
            w2 = _rand_weight(dev, 9, cout, 64, seed=6)
            s2 = torch.full((64,), 0.25, device=dev)
            y1.status = st = _status(dev)
            z1, _ = ops.conv2d_split(y1, w2, s2, None, True, 64)
            z2, g2 = ops.conv2d_split(y1, w2, s2, None, True, 64, out_split=True, out_f32=True)
            assert z1.reach == 2
            _assert_split_of(z1.planes, g2, 64, "reach-2 layer")
            _assert_split_of(z2.planes, g2, 64, "reach-2 layer, both outputs")
            assert not _flag(st)


@pytest.mark.gpu
def test_sparse_to_bev_and_rows_to_split(dev):
    """sassd_sparse_to_bev_split and sassd_features_to_split store numpy's split of their fp32 inputs bit for bit on
    values from 2^-40 to 2^15 and the edge values; 65520, -65520 and 1e5 flag F16_RANGE, inf and NaN do not."""
    from sassd_b200 import ops
    B, H, W, C = 2, 40, 48, 64
    feat, coors, d_rows = _scatter(dev, B, H, W, C, 300, seed=3)
    feat[:len(EDGES), 0] = torch.from_numpy(EDGES).to(dev)
    for extra, flagged in ((None, False), (65519.99, False), (65520.0, True), (-65520.0, True), (1e5, True),
                           (float("inf"), False), (float("-inf"), False), (float("nan"), False)):
        f = feat.clone()
        if extra is not None:
            f[7, 5] = extra
        st = _status(dev)
        x = ops.sparse_to_bev_split(f, coors, d_rows, C, 1, H, W, B, status=st)
        want = torch.zeros((B, H, W, C), device=dev)
        c = coors.long()
        want[c[:, 0], c[:, 2], c[:, 3]] = f
        _assert_split_of(x.planes, want, C, "sparse_to_bev_split %s" % extra)
        assert _flag(st) == flagged, "sparse_to_bev_split %s" % extra
        for cin in (C, 20):
            st = _status(dev)
            rows = f[:, :cin].contiguous()
            sp = ops.features_to_split(rows, d_rows, status=st)
            _assert_split_of(sp, rows, cin, "features_to_split cin %d %s" % (cin, extra))
            assert _flag(st) == flagged, "features_to_split %s" % extra


def _lidar(B, dev):
    from tests.test_tc_exact import _lidar_tables
    return _lidar_tables(B, dev)


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["subm", "conv", "1x1"])
def test_sparse_epilogue_stores_the_split_of_its_fp32_output(dev, kind):
    """The sparse conv's epilogue: at 27 taps with the chunk deal on and off, and at 1x1, its planes are numpy's split
    of its fp32 rows, bit for bit, from 2^-40 to the edge; past the edge F16_RANGE."""
    from sassd_b200 import ops
    t = _lidar(1, dev)["subm" if kind == "1x1" else kind]
    nbr, tm, in_rows, cap, d_rows, n = t
    cin, cout = 32, 64
    g = torch.Generator(device=dev).manual_seed(4)
    planes = ops.features_to_split(torch.randn((in_rows, cin), generator=g, device=dev))
    taps = 1 if kind == "1x1" else 27
    w = _rand_weight(dev, taps, cin, cout, seed=9)
    saved = ops.SPCONV_TAP_SPLIT
    try:
        for deal in ((False,) if kind == "1x1" else (False, True)):
            ops.SPCONV_TAP_SPLIT = deal
            for edges, over in ((EDGES, False), (OVER, True)):
                scale, shift = _range_bn(cout, dev, edges)
                st = _status(dev)
                out, of = ops.spconv_split(planes, w, scale, shift, False, cout, cap if taps > 1 else in_rows,
                                           nbr=nbr if taps > 1 else None, d_rows=d_rows, want_f32=True,
                                           tile_mask=tm if taps > 1 else None, status=st)
                _assert_split_of(out[:, :n], of[:n], cout, "%s deal %d" % (kind, deal))
                assert _flag(st) == over
    finally:
        ops.SPCONV_TAP_SPLIT = saved


# ------------------------------------------------------------------------------------------------ GPU: accuracy
def _conv64(x, w, cond=False):
    """fp64 3x3 (pad 1) or 1x1 NHWC conv of x [B,H,W,C] with w [taps,C,cout]; cond: the bound's two sums,
    (|x| (*) |w|, |x| (*) 1 + 1 (*) |w| over the taps that read the image)."""
    if cond:
        ax, aw = x.double().abs(), w.double().abs()
        return _conv64(ax, aw), _conv64(ax, torch.ones_like(aw)) + _conv64(torch.ones_like(ax), aw)
    x, w = x.double(), w.double()
    if w.shape[0] == 1:
        return x @ w[0]
    B, H, W, _ = x.shape
    xp = torch.nn.functional.pad(x, (0, 0, 1, 1, 1, 1))
    v = 0
    for t in range(9):
        ky, kx = divmod(t, 3)
        v = v + xp[:, ky:ky + H, kx:kx + W] @ w[t]
    return v


def _check_bound(got, ref, cond, scale, what):
    """|got - ref| <= TOL_REL * cond[0] * |scale| + SPLIT_FLOOR * cond[1] * |scale| + TOL_ABS per element, cond =
    (sum |a| |w|, sum |a| + sum |w|); returns the worst ratio."""
    tol = (TOL_REL * cond[0] + SPLIT_FLOOR * cond[1]) * scale.double().abs() + TOL_ABS
    err = (got.double() - ref).abs()
    ratio = float((err / tol).max())
    if ratio > 1:
        i = tuple(int(v) for v in torch.nonzero(err > tol)[0])
        raise AssertionError("%s: error %.3g above the bound %.3g at %s (ref %.6g, got %.6g, %d elements over)" % (
            what, float(err[i]), float(tol[i]), i, float(ref[i]), float(got[i]), int((err > tol).sum())))
    return ratio


def _span_input(dev, B, H, W, cin, seed, per_pixel):
    """fp32 input: 64-channel blocks scaled 2^-20 .. 2^12, or (per_pixel) one magnitude 2^-20 .. 2^12 per pixel."""
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn((B, H, W, cin), generator=g, device=dev)
    if per_pixel:
        e = torch.randint(-20, 13, (B, H, W, 1), generator=g, device=dev).float()
    else:
        e = torch.linspace(-20, 12, (cin + 63) // 64, device=dev).round().repeat_interleave(64)[:cin]
    return (x * torch.exp2(e)).contiguous()


def _span_weight(dev, taps, cin, cout, seed):
    """Weights whose output columns span 2^-16 .. 2^0."""
    w = _rand_weight(dev, taps, cin, cout, seed)
    return (w * torch.exp2(torch.linspace(-16, 0, cout, device=dev).round())).contiguous()


def _dense_accuracy(dev, x, w, cout, relu=True, planes=None, scale=None):
    from sassd_b200 import ops
    sm = ops.SplitMap.from_float(x)
    if planes is not None:
        sm.planes = planes
    if scale is None:
        scale = torch.exp2(torch.randint(-2, 3, (cout,), device=dev).float())
    _, f32 = ops.conv2d_split(sm, w, scale, None, relu, cout, out_split=False, out_f32=True)
    ref = _conv64(x, w) * scale.double()
    if relu:
        ref = ref.clamp_min(0)
    return f32[..., :cout], ref, _conv64(x, w, cond=True), scale


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 16])
@pytest.mark.parametrize("layer", sorted(DENSE_LAYERS))
def test_dense_accuracy_per_element(dev, layer, B):
    """Every dense layer shape, on the 200 x 176 grid and on a map with partial tiles, within TOL_REL * sum |a| |w|
    |scale| + TOL_ABS of fp64 per element, on inputs whose channel blocks or pixels span 2^-20 .. 2^12 and weights
    whose columns span 2^-16 .. 2^0."""
    taps, cin, _, cout = DENSE_LAYERS[layer]
    shapes = [(200, 176), (21, 37)] if B == 1 else [(200, 176)]
    for H, W in shapes:
        for per_pixel in (False, True):
            x = _span_input(dev, B, H, W, cin, seed=H + per_pixel, per_pixel=per_pixel)
            w = _span_weight(dev, taps, cin, cout, seed=cout)
            got, ref, cond, scale = _dense_accuracy(dev, x, w, cout)
            _check_bound(got, ref, cond, scale, "%s B=%d %dx%d per_pixel=%d" % (layer, B, H, W, per_pixel))
            del got, ref, cond
    torch.cuda.empty_cache()


def _coherent(dev, shape, seed, span=None):
    """Positive fp32 values m (1 + 3 * 2^-13) with m an fp16 value: every split keeps lo = 0.75 m, so a lost lo path
    errs coherently by 3 * 2^-13 of what it drops (random signs would cancel it below the bound)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    m = (torch.rand(shape, generator=g, device=dev) + 0.5).half().float()
    if span is not None:
        m = m * span
    return (m * (1 + 3 * 2.0 ** -13)).contiguous()


@pytest.mark.gpu
def test_bound_catches_a_lost_low_order_path(dev):
    """The per-element bound fails, with no kernel change, when the lo plane of one 64-channel input block is zeroed
    at the small pixels of a map whose pixels span 2^-13 .. 2^12 or when the lo half of one weight column is zeroed (the 2^-13 column; both
    kept in fp16's normal range, where the split holds 22 bits);
    the same operands pass intact.  A bound scaled by the map's maximum accepts both."""
    from sassd_b200 import ops
    B, H, W, cin, cout = 1, 24, 40, 256, 64
    pix = torch.exp2(torch.randint(-13, 13, (B, H, W, 1), device=dev).float())
    x = _coherent(dev, (B, H, W, cin), 1, pix)
    cols = torch.exp2(torch.linspace(-13, 0, cout, device=dev).round())
    # a 1x1 conv: with every product positive the tensor cores' truncating accumulation errs coherently too, by
    # 2.1e-5 of the sum over the 2304 terms of a 3x3 256-channel conv (measured on an H100), ~1/9 of that over 256
    w = _coherent(dev, (1, cin, cout), 2, cols)
    got, ref, cond, scale = _dense_accuracy(dev, x, w, cout, relu=False)
    assert _check_bound(got, ref, cond, scale, "intact operands") < 0.5
    # (1) the lo plane of input block 1 zeroed at the small-magnitude pixels (<= 2^-6)
    planes = ops.SplitMap.from_float(x).planes.clone()
    block = planes[1, ..., 64:128]
    block[pix[..., 0] <= 2.0 ** -6] = 0
    got1, *_ = _dense_accuracy(dev, x, w, cout, relu=False, planes=planes, scale=scale)
    with pytest.raises(AssertionError, match="above the bound"):
        _check_bound(got1, ref, cond, scale, "lo plane of one input block zeroed")
    assert float((got1.double() - ref).abs().max()) <= 2e-5 * float(ref.abs().max()), "the max-scaled bound catches it"
    # (2) the lo half of the smallest weight column zeroed: a weight whose split is hi only
    w2 = w.clone()
    w2[..., 0] = w2[..., 0].half().float()
    got2, *_ = _dense_accuracy(dev, x, w2, cout, relu=False, scale=scale)
    with pytest.raises(AssertionError, match="above the bound"):
        _check_bound(got2, ref, cond, scale, "lo half of one weight column zeroed")
    assert float((got2.double() - ref).abs().max()) <= 2e-5 * float(ref.abs().max()), "the max-scaled bound catches it"


@pytest.mark.gpu
@pytest.mark.parametrize("pair", SPARSE_PAIRS, ids=lambda p: "%d_%d_%d" % p)
def test_sparse_accuracy_per_element(dev, pair):
    """Every sparse channel pair on LiDAR rulebooks (submanifold and strided), chunk deal on, within the bound."""
    from sassd_b200 import ops
    cin, cs, cout = pair
    for kind in ("subm", "conv"):
        nbr, tm, in_rows, cap, d_rows, n = _lidar(1, dev)[kind]
        x = _span_input(dev, 1, 1, in_rows, cin, seed=cin, per_pixel=True).view(in_rows, cin)
        xs = torch.zeros((in_rows, cs), device=dev)
        xs[:, :cin] = x
        planes = ops.features_to_split(xs)
        w = _span_weight(dev, 27, cin, cout, seed=cout)
        scale = torch.exp2(torch.randint(-2, 3, (cout,), device=dev).float())
        _, of = ops.spconv_split(planes, w, scale, None, True, cout, cap, nbr=nbr, d_rows=d_rows, want_f32=True,
                                 tile_mask=tm)
        nb = nbr[:n].long()
        ref = torch.zeros((n, cout), dtype=torch.float64, device=dev)
        c0, c1 = torch.zeros_like(ref), torch.zeros_like(ref)
        for t in range(27):
            o = torch.nonzero(nb[:, t] >= 0).view(-1)
            a, wt = x[nb[o, t]].double(), w[t].double()
            ref.index_add_(0, o, a @ wt)
            c0.index_add_(0, o, a.abs() @ wt.abs())
            c1.index_add_(0, o, a.abs().sum(1, keepdim=True) + wt.abs().sum(0))
        cond = (c0, c1)
        ref = (ref * scale.double()).clamp_min(0)
        _check_bound(of[:n, :cout], ref, cond, scale, "sparse %s %s" % (pair, kind))


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [0, 1, 2], ids=["fp32", "tf32x3", "f16x3"])
def test_gconv_accuracy_and_range_flag(dev, precision):
    """sassd_gconv (CONV2D and TABLE modes) at all three precisions within the bound; at F16X3 an input past the edge
    flags F16_RANGE from the on-the-fly split, 65519.99, inf and NaN do not; the other precisions never flag."""
    from sassd_b200 import ops
    B, H, W, cin, cout = 2, 21, 37, 64, 96
    x = _span_input(dev, B, H, W, cin, seed=7, per_pixel=True)
    w = _span_weight(dev, 9, cin, cout, seed=8)
    scale = torch.exp2(torch.randint(-2, 3, (cout,), device=dev).float())
    out = torch.empty((B, H, W, cout), device=dev)
    st = _status(dev)
    ops.gconv(x.view(-1, cin), w, scale, None, out.view(-1, cout), mode=ops.GCONV_CONV2D, taps=9, cin=cin, cout=cout,
              relu=True, rows_cap=B * H * W, batch=B, H=H, W=W, precision=precision, status=st)
    _check_bound(out, (_conv64(x, w) * scale.double()).clamp_min(0), _conv64(x, w, cond=True), scale,
                 "gconv precision %d" % precision)
    assert not _flag(st)
    for v, flagged in ((65519.99, False), (65520.0, True), (-1e5, True), (float("inf"), False), (float("nan"), False)):
        xv = x.clone()
        xv[1, 3, 4, 10] = v
        st = _status(dev)
        ops.gconv(xv.view(-1, cin), w, scale, None, out.view(-1, cout), mode=ops.GCONV_CONV2D, taps=9, cin=cin,
                  cout=cout, relu=True, rows_cap=B * H * W, batch=B, H=H, W=W, precision=precision, status=st)
        assert _flag(st) == (flagged and precision == 2), "gconv precision %d input %s" % (precision, v)


# ------------------------------------------------------------------------------------------------ GPU: NaN
def _nan_cases(dev, taps, cin, cout, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn((2, 19, 37, cin), generator=g, device=dev)
    x[0, 4, 7] = -x[0, 4, 7].abs()          # negative and signed-zero inputs keep their bits
    x[1, 0, 0, :8] = -0.0
    x[1, 0, 1, :8] = 0.0
    w = _rand_weight(dev, taps, cin, cout, seed + 1)
    return x, w


def _nan_expect(shape, taps, pix):
    """Pixels whose receptive field holds input pixel pix = (b, y, x)."""
    B, H, W = shape
    m = torch.zeros((B, H, W), dtype=torch.bool)
    b, y, x = pix
    r = 1 if taps == 9 else 0
    m[b, max(y - r, 0):y + r + 1, max(x - r, 0):x + r + 1] = True
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("cout", [256, 64, 28])
@pytest.mark.parametrize("taps", [9, 1])
def test_nan_input_pixel_spreads_to_its_receptive_field_only(dev, taps, cout):
    """A NaN in one input pixel: NaN on every output channel of exactly the pixels whose receptive field holds it, at
    all three precisions and with and without ReLU; every other output keeps its bits, and the padding channels of the
    split output stay exactly zero.  The F16X3 dense conv (conv2d_tma) and sassd_gconv at FP32 / TF32X3 / F16X3."""
    from sassd_b200 import ops
    cin = 64
    x, w = _nan_cases(dev, taps, cin, cout, seed=taps + cout)
    pix = (1, 9, 17)
    xn = x.clone()
    xn[pix][5] = float("nan")
    expect = _nan_expect((2, 19, 37), taps, pix).to(dev)
    scale = torch.rand(cout, device=dev) + 0.5
    shift = torch.randn(cout, device=dev)
    for relu in (False, True):
        runs = {}
        for name in ("tma", 0, 1, 2):
            outs = []
            for inp in (x, xn):
                if name == "tma":
                    sp, f = ops.conv2d_split(ops.SplitMap.from_float(inp), w, scale, shift, relu, cout, out_split=True,
                                             out_f32=True)
                    assert bool((sp.planes[..., cout:] == 0).all()), "padding channels of the split output"
                    assert bool((f[..., cout:] == 0).all()), "padding columns of the fp32 output"
                    _assert_split_of(sp.planes, f, cout, "NaN run")
                    f = f[..., :cout]
                else:
                    f = torch.empty((2, 19, 37, cout), device=dev)
                    ops.gconv(inp.view(-1, cin), w, scale, shift, f.view(-1, cout), mode=ops.GCONV_CONV2D, taps=taps,
                              cin=cin, cout=cout, relu=relu, rows_cap=2 * 19 * 37, batch=2, H=19, W=37, precision=name)
                outs.append(f)
            clean, dirty = outs
            what = "%s relu %d" % (name, relu)
            assert not bool(torch.isnan(clean).any()), what
            assert torch.equal(torch.isnan(dirty), expect[..., None].expand_as(dirty)), "%s: NaN pattern" % what
            assert torch.equal(dirty[~expect].view(torch.int32), clean[~expect].view(torch.int32)), what
            runs[name] = clean
        # negative inputs, +0 and -0: ReLU outputs of the NaN-keeping kernel are those of fmaxf (no -0, no negative)
        if relu:
            for name, f in runs.items():
                assert bool((f >= 0).all()) and not bool(torch.signbit(f).any()), name


@pytest.mark.gpu
@pytest.mark.parametrize("cout", [256, 28])
def test_nan_weight_poisons_its_output_channel_only(dev, cout):
    """One NaN weight: its output channel is NaN at every pixel (the zero padding times NaN is NaN, as in torch's
    conv2d), every other channel keeps its bits, padding channels stay zero; dense conv and gconv at all precisions."""
    from sassd_b200 import ops
    cin = 64
    x, w = _nan_cases(dev, 9, cin, cout, seed=cout)
    wn = w.clone()
    wn[4, 7, 3] = float("nan")
    for relu in (False, True):
        for name in ("tma", 0, 1, 2):
            outs = []
            for ww in (w, wn):
                if name == "tma":
                    sp, f = ops.conv2d_split(ops.SplitMap.from_float(x), ww, None, None, relu, cout, out_split=True,
                                             out_f32=True)
                    assert bool((sp.planes[..., cout:] == 0).all()) and bool((f[..., cout:] == 0).all())
                    f = f[..., :cout]
                else:
                    f = torch.empty((2, 19, 37, cout), device=dev)
                    ops.gconv(x.view(-1, cin), ww, None, None, f.view(-1, cout), mode=ops.GCONV_CONV2D, taps=9,
                              cin=cin, cout=cout, relu=relu, rows_cap=2 * 19 * 37, batch=2, H=19, W=37, precision=name)
                outs.append(f)
            clean, dirty = outs
            assert bool(torch.isnan(dirty[..., 3]).all()), "%s relu %d" % (name, relu)
            keep = torch.ones(cout, dtype=torch.bool, device=dev)
            keep[3] = False
            assert not bool(torch.isnan(dirty[..., keep]).any())
            assert torch.equal(dirty[..., keep].view(torch.int32), clean[..., keep].view(torch.int32))


@pytest.mark.gpu
@pytest.mark.parametrize("cout", [64, 16])
def test_sparse_nan_row_spreads_to_its_neighbours_only(dev, cout):
    """A NaN in one input row of the sparse conv: NaN on every output channel of exactly the rows that list it in
    their neighbour table, with and without ReLU and the chunk deal; the other rows keep their bits and the stored
    channels past cout stay zero (their zero weights times NaN would otherwise be NaN)."""
    from sassd_b200 import ops
    nbr, tm, in_rows, cap, d_rows, n = _lidar(1, dev)["subm"]
    cin = 32
    g = torch.Generator(device=dev).manual_seed(cout)
    x = torch.randn((in_rows, cin), generator=g, device=dev)
    w = _rand_weight(dev, 27, cin, cout, seed=3)
    bad = int(n // 3)
    xn = x.clone()
    xn[bad, 2] = float("nan")
    expect = (nbr[:n].long() == bad).any(1)
    assert 1 < int(expect.sum()) <= 27
    saved = ops.SPCONV_TAP_SPLIT
    try:
        for deal in (False, True):
            ops.SPCONV_TAP_SPLIT = deal
            for relu in (False, True):
                outs = []
                for inp in (x, xn):
                    out, of = ops.spconv_split(ops.features_to_split(inp), w, None, None, relu, cout, cap, nbr=nbr,
                                               d_rows=d_rows, want_f32=True, tile_mask=tm)
                    stored = out.shape[-1]
                    assert bool((out[:, :n, cout:] == 0).all()) and bool((of[:n, cout:] == 0).all()), \
                        "padding channels (stored %d, cout %d)" % (stored, cout)
                    outs.append(of[:n, :cout])
                clean, dirty = outs
                assert not bool(torch.isnan(clean).any())
                assert torch.equal(torch.isnan(dirty), expect[:, None].expand_as(dirty))
                assert torch.equal(dirty[~expect].view(torch.int32), clean[~expect].view(torch.int32))
    finally:
        ops.SPCONV_TAP_SPLIT = saved


# ------------------------------------------------------------------------------------------------ GPU: the step
OCFG = dict(voxel_size=[0.05, 0.05, 0.1], pc_range=[0, -40., -3., 70.4, 40., 1.], max_points=5, max_voxels=20000,
            sparse_shape=[40, 1600, 1408],
            anchor_cfgs=[dict(sizes=[1.6, 3.9, 1.56], anchor_strides=[0.4, 0.4, 1.0],
                              anchor_offsets=[0.2, -39.8, -1.78], rotations=[0, 1.57])],
            grid_offsets=(0., 40.), featmap_stride=.4, score_thr=0.3, iou_thr=0.1)
# (BN layer, weight and bias multiplier, expected to overflow)
# (2^14 is not enough on this cloud: the oracle measures 4.0e4 at its largest; 2^16 is)
CONSTRUCTIONS = [("neck.fcn.bn3", 2.0 ** 16, True), ("neck.backbone.conv2.4", 2.0 ** 16, True),
                 ("neck.fcn.bn3", 2.0 ** 8, False)]


def _cloud():
    from sassd_b200.synth import synth_cloud
    return synth_cloud(1, fov_deg=20.0, az_step_deg=0.3456)


def _constructed(layer, mult):
    from sassd_b200 import checkpoint
    sd = checkpoint.make_synthetic_state_dict(0, 1)
    for s in (".weight", ".bias"):
        sd[layer + s] = sd[layer + s] * mult
    return sd


@pytest.mark.parametrize("layer,mult,over", CONSTRUCTIONS)
def test_constructions_land_where_intended(layer, mult, over):
    """On the CPU oracle: the largest positive BatchNorm output (what the ReLU stores) of the constructed checkpoint
    is above 65520 for an "over" construction and below it everywhere for an "under" one."""
    from oracle import ref_pipeline as O
    sd = _constructed(layer, mult)
    top = {}
    orig = O.bn_eval

    def bn_eval(x, sd_, prefix, eps=1e-3):
        y = orig(x, sd_, prefix, eps)
        top[prefix] = max(top.get(prefix, 0.0), float(y.max()))
        return y
    O.bn_eval = bn_eval
    try:
        O.forward_test(sd, [_cloud()], OCFG)
    finally:
        O.bn_eval = orig
    assert layer in top
    if over:
        assert top[layer] > 65520.0, top
    else:
        assert max(top.values()) < 65520.0, top


def _model(sd, dev="cuda:0"):
    from sassd_b200 import checkpoint
    from tests.checkpoint_weights import build
    m = build(dev)
    checkpoint.load_state_dict_into(m, sd)
    return m


def _same_out(a, b, what):
    for da, db in zip(a, b):
        assert (da["boxes_lidar"] is None) == (db["boxes_lidar"] is None), what
        if da["boxes_lidar"] is not None:
            assert np.array_equal(da["boxes_lidar"], db["boxes_lidar"]), what
            assert np.array_equal(da["scores"], db["scores"]), what


@pytest.mark.gpu
@pytest.mark.parametrize("layer,mult", [(c[0], c[1]) for c in CONSTRUCTIONS if c[2]])
def test_overflowing_checkpoint_raises_in_every_mode(dev, layer, mult):
    """The over construction raises SassdError naming F16_RANGE eagerly, captured, through detect_stream and in a
    CheckpointSweep beside seed 0; at PREC_FP32 the same model completes with finite head maps."""
    from sassd_b200 import checkpoint, lib, ops
    from sassd_b200.detectors import CheckpointSweep
    pts = [_cloud()]
    m = _model(_constructed(layer, mult))
    with pytest.raises(lib.SassdError, match="F16_RANGE"):
        m.forward_points(pts)
    m.enable_cuda_graph(1, 32768)
    with pytest.raises(lib.SassdError, match="F16_RANGE"):
        m.forward_points(pts)
    m.disable_cuda_graph()
    with pytest.raises(lib.SassdError, match="F16_RANGE"):
        list(m.detect_stream([pts], 1, 32768, depth=2))
    m0 = _model(checkpoint.make_synthetic_state_dict(0, 1))
    alone = m0.forward_points(pts)
    with pytest.raises(lib.SassdError, match="F16_RANGE"):
        CheckpointSweep([m0, m]).forward_points(pts)
    _same_out(m0.forward_points(pts), alone, "seed 0 after the sweep")
    m.set_precision(ops.PREC_FP32)
    out, aux = m.forward_points(pts, return_aux=True)
    assert bool(torch.isfinite(aux["head"]).all())
    del m, m0
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_in_range_checkpoint_sets_no_flag_and_matches_fp32(dev):
    """The under construction (activations up to ~2^8 times seed 0's) sets no flag, and its f16x3 neck output is
    within the per-element bound's relative constant of the FP32 path's."""
    from sassd_b200 import ops
    layer, mult, _ = CONSTRUCTIONS[2]
    pts = [_cloud()]
    m = _model(_constructed(layer, mult))
    p = torch.from_numpy(pts[0]).to(dev).contiguous()
    off = torch.tensor([0, p.shape[0]], dtype=torch.int32, device=dev)
    _, _, st, aux = m.forward_device(p, off, 1, p.shape[0])    # the boosted scores may fill DET_CAP: read the bit
    assert not _flag(st)
    x16 = aux["x"].float() if isinstance(aux["x"], ops.SplitMap) else aux["x"]
    m.set_precision(ops.PREC_FP32)
    _, _, _, aux32 = m.forward_device(p, off, 1, p.shape[0])
    x32 = aux32["x"][..., :x16.shape[-1]]
    scale = float(x32.abs().max())
    assert scale > 64.0, "the construction does not reach the magnitudes it is meant to"
    assert float((x16 - x32).abs().max()) <= 1e-4 * scale
