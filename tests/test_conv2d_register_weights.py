"""The dense BEV conv's BN = 128 kernel (every layer with cout > 64): weights in wgmma register fragments
(sassd_conv2d_pack), pixels from shared memory, the epilogue transposed through shared memory.

The pack layout against a numpy restatement; the outputs against an fp64 restatement within the bound of
test_gpu_parity.py::test_tensor_core_conv_matches_fp64, bit for bit on operands whose split products sum exactly
(test_tc_exact.py's grids), and with tile skipping and backgrounds equal to the fully computed map."""
import ctypes

import numpy as np
import pytest
import torch

from tests.test_tc_exact import (assert_f32_out, assert_split_out, conv_ref, epilogue, grid_bn, grid_planes,
                                 grid_weights, split16_np)

# (taps, cin, cout): cin 64 / 256 / 320, cout 96 / 128 / 256, 3x3 and 1x1
SHAPES = [(9, 64, 96), (9, 256, 128), (9, 256, 256), (9, 320, 256), (1, 256, 256), (1, 64, 128), (1, 320, 96)]
# (batch, H, W): the detector's grid and a map with partial edge tiles (13 = 8 + 5 rows, 21 = 16 + 5 columns)
MAPS = [(1, 200, 176), (2, 13, 21), (16, 13, 21)]
# (out_split, out_f32, relu)
OUTPUTS = [(True, False, True), (False, True, False), (True, True, True), (True, True, False)]


def pack_np(w, cout):
    """numpy restatement of sassd_conv2d_pack for cout > 64: uint32 words [q][s][mb][t][hi a0..a3, lo a0..a3]."""
    taps, cin, _ = w.shape
    kchunks, ncols = (cin + 63) // 64, 3 if taps == 9 else 1
    nblk = 2 if cout <= 128 else 4
    wp = np.zeros((taps, kchunks * 64, nblk * 64), np.float32)
    wp[:, :cin, :cout] = w
    hi, lo = split16_np(wp)
    out = np.zeros((taps * kchunks, 4, nblk, 128, 8), np.uint32)
    t = np.arange(128)
    lane = t % 32
    for q in range(taps * kchunks):
        row, kc, col = q % ncols, (q // ncols) % kchunks, q // (ncols * kchunks)
        tap = row * ncols + col
        for s in range(4):
            for mb in range(nblk):
                for a in range(4):
                    n = 64 * mb + 16 * (t // 32) + lane // 4 + 8 * (a & 1)
                    k = kc * 64 + 16 * s + 2 * (lane % 4) + 8 * (a >> 1)
                    for part, plane in enumerate((hi, lo)):
                        lo16 = plane[tap, k, n].view(np.uint16).astype(np.uint32)
                        hi16 = plane[tap, k + 1, n].view(np.uint16).astype(np.uint32)
                        out[q, s, mb, :, 4 * part + a] = lo16 | (hi16 << 16)
    return out.reshape(-1)


def test_pack_bytes():
    from sassd_b200 import lib
    L = lib.load()
    assert L.sassd_conv2d_pack_bytes(9, 256, 256) == 9 * 4 * 4 * 4 * 128 * 32
    assert L.sassd_conv2d_pack_bytes(9, 320, 96) == 9 * 5 * 4 * 2 * 128 * 32
    assert L.sassd_conv2d_pack_bytes(1, 28, 28) == L.sassd_gconv_pack_bytes(1, 28, 28, 2)
    assert L.sassd_conv2d_pack_bytes(3, 64, 128) == 0 and L.sassd_conv2d_pack_bytes(9, 64, 257) == 0


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("taps,cin,cout", [(9, 320, 256), (9, 64, 96), (1, 256, 128), (1, 100, 200)])
def test_pack_layout_matches_numpy(dev, taps, cin, cout):
    from sassd_b200 import ops
    g = torch.Generator().manual_seed(taps + cin + cout)
    w = torch.randn(taps, cin, cout, generator=g) * 0.3
    got = ops.conv2d_pack_cached(w.to(dev)).cpu().numpy().view(np.uint32)
    assert np.array_equal(got, pack_np(w.numpy(), cout))


def _run(x, w, cout, relu, out_split, out_f32, scale, shift):
    from sassd_b200 import ops
    return ops.conv2d_split(x, w, scale, shift, relu, cout, out_split=out_split, out_f32=out_f32)


@pytest.mark.gpu
@pytest.mark.parametrize("mp", MAPS)
@pytest.mark.parametrize("shape", SHAPES)
def test_conv_matches_fp64(dev, shape, mp):
    """Random operands against fp64: within 4x the FFMA kernel's error (or 4e-6 of the output's range), under every
    output / ReLU combination; the split planes are the split of the fp32 output."""
    from sassd_b200 import ops
    taps, cin, cout = shape
    B, H, W = mp
    g = torch.Generator(device=dev).manual_seed(taps * 7 + cin + cout + B)
    x = torch.randn(B, H, W, cin, device=dev, generator=g)
    w = torch.randn(taps, cin, cout, device=dev, generator=g) * 0.05
    scale = torch.rand(cout, device=dev, generator=g) + 0.5
    shift = torch.randn(cout, device=dev, generator=g) * 0.1
    xs = ops.SplitMap.from_float(x)
    xv = xs.float()
    k = 3 if taps == 9 else 1
    wk = w.double().view(k, k, cin, cout).permute(3, 2, 0, 1)
    ref = torch.nn.functional.conv2d(xv.double().permute(0, 3, 1, 2), wk, padding=k // 2).permute(0, 2, 3, 1)
    ref = ref * scale.double() + shift.double()
    ffma = torch.zeros(B * H * W, (cout + 3) // 4 * 4, device=dev)
    ops.gconv(xv.reshape(-1, cin), w, scale, shift, ffma, mode=ops.GCONV_CONV2D, taps=taps, cin=cin, cout=cout,
              relu=False, rows_cap=B * H * W, batch=B, H=H, W=W, precision=ops.PREC_FP32)
    e_ffma = (ffma[:, :cout].double() - ref.reshape(-1, cout)).abs().max().item()
    tol = max(4 * e_ffma, 4e-6 * ref.abs().max().item())
    for out_split, out_f32, relu in OUTPUTS:
        r = ref.clamp_min(0) if relu else ref
        sp, f32 = _run(xs, w, cout, relu, out_split, out_f32, scale, shift)
        if out_f32:
            assert f32.shape[-1] == (cout + 3) // 4 * 4
            err = (f32[..., :cout].double() - r).abs().max().item()
            assert err <= tol, (err, tol)
            assert bool((f32[..., cout:] == 0).all())
        if out_split:
            err = (sp.float().double() - r).abs().max().item()
            assert err <= tol, (err, tol)
            assert bool((sp.planes[..., cout:] == 0).all())
            if out_f32:
                hi = f32[..., :cout].half()
                assert torch.equal(sp.planes[0, ..., :cout], hi)
                assert torch.equal(sp.planes[1, ..., :cout], ((f32[..., :cout] - hi.float()) * 2048).half())


@pytest.mark.gpu
@pytest.mark.parametrize("mp", [(1, 200, 176), (2, 13, 21), (16, 13, 21)])
@pytest.mark.parametrize("shape", SHAPES)
def test_conv_exact_on_exact_sums(dev, shape, mp):
    """On test_tc_exact's grids every split product and partial sum is exact in fp32: the outputs equal the fp64
    restatement bit for bit."""
    from sassd_b200 import ops
    taps, cin, cout = shape
    B, H, W = mp
    cs = (cin + 63) // 64 * 64
    x = ops.SplitMap(grid_planes((B, H, W, cs), cin, seed=B * 100 + H + W, device=dev, lo_from=0), cin)
    w = grid_weights(taps, cin, cout, seed=taps + cin + cout).to(dev)
    scale, shift = grid_bn(cout, cout, dev)
    v = conv_ref(x.planes, cin, w)
    for out_split, out_f32, relu in OUTPUTS:
        ref = epilogue(v, scale, shift, relu)
        sp, f32 = _run(x, w, cout, relu, out_split, out_f32, scale, shift)
        if out_split:
            assert_split_out(sp.planes, ref, cout, "split output")
        if out_f32:
            assert_f32_out(f32, ref, cout, "fp32 output")


@pytest.mark.gpu
@pytest.mark.parametrize("order", [0, 1])
@pytest.mark.parametrize("B", [1, 2, 16])
def test_tile_skipping_and_backgrounds_match_computing_every_tile(dev, B, order):
    """A scattered map through 64->128 (reach 1: constant tiles) and 128->256 (reach 2: constant interior tiles,
    background border tiles), with tile skipping on and off: the same bits."""
    from sassd_b200 import ops
    H, W, C = 200, 176, 64
    rs = np.random.RandomState(B)
    coors = np.zeros((40 * B, 4), np.int32)
    for b in range(B):
        flat = rs.choice(H * W, 40, replace=False)
        coors[40 * b:40 * (b + 1), 0], coors[40 * b:40 * (b + 1), 2], coors[40 * b:40 * (b + 1), 3] = b, flat // W, flat % W
    feat = torch.from_numpy(rs.randn(40 * B, C).astype(np.float32)).to(dev)
    d_rows = torch.tensor([40 * B], dtype=torch.int32, device=dev)
    g = torch.Generator(device=dev).manual_seed(B)
    wa, wb = (torch.randn(9, ci, co, device=dev, generator=g) * 0.05 for ci, co in ((C, 128), (128, 256)))
    sa, sb = (torch.rand(co, device=dev, generator=g) + 0.5 for co in (128, 256))
    ha, hb = (torch.randn(co, device=dev, generator=g) * 0.1 for co in (128, 256))
    outs = []
    occ0, order0 = ops.TILE_OCCUPANCY, ops.CONV2D_TILE_ORDER
    try:
        for occ in (True, False):
            ops.TILE_OCCUPANCY, ops.CONV2D_TILE_ORDER = occ, order
            x = ops.sparse_to_bev_split(feat, torch.from_numpy(coors).to(dev), d_rows, C, 1, H, W, B)
            ya, _ = ops.conv2d_split(x, wa, sa, ha, True, 128)
            yb, fb = ops.conv2d_split(ya, wb, sb, hb, True, 256, out_split=True, out_f32=True)
            if occ:
                assert yb.reach == 2 and yb.tile_dist is not None and yb.background is not None
            outs.append((ya.planes, yb.planes, fb))
    finally:
        ops.TILE_OCCUPANCY, ops.CONV2D_TILE_ORDER = occ0, order0
    for a, b in zip(*outs):
        assert torch.equal(a, b)
