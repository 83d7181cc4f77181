"""The operand feed of the dense BEV conv (csrc/conv2d_tma.cu): a unit walks (tap column, 64-channel chunk) outer and
the vertical taps inner, all three reading one halo box of TILE_H + 2 rows.  These tests reach the cases that feed
has to get right: halos that cross the top or bottom edge or a partial last tile row, 1x1 and 3x3 taps, the layer
widths of the detector, the skipping chain with few or no computed tiles, at 16 frames of the detector's grid (the
largest map the kernel orders in shared memory) and above, the tile counters and a captured CUDA graph."""
import numpy as np
import pytest
import torch

from tests.test_background_tiles import tile_kinds
from tests.test_constant_region_rule import TH, TW


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout", [(256, 256), (320, 256), (256, 28), (256, 20)])
@pytest.mark.parametrize("taps", [1, 9])
@pytest.mark.parametrize("H", [8, 9, 21, 200])
@pytest.mark.parametrize("W", [16, 20, 176])
def test_conv_matches_fp64(dev, H, W, taps, cin, cout):
    """Split-plane and fp32 outputs against an fp64 conv, with tests/tools/tc_check.py's tolerance."""
    from sassd_b200 import ops
    g = torch.Generator(device=dev).manual_seed(H * 1000 + W + taps + cin + cout)
    B = 2
    x = torch.randn(B, H, W, cin, device=dev, generator=g)
    w = torch.randn(taps, cin, cout, device=dev, generator=g) * 0.05
    scale = torch.rand(cout, device=dev, generator=g) + 0.5
    shift = torch.randn(cout, device=dev, generator=g) * 0.1
    sp, f32 = ops.conv2d_split(ops.SplitMap.from_float(x), w, scale, shift, True, cout, out_split=True, out_f32=True)
    k = 3 if taps == 9 else 1
    ref = torch.nn.functional.conv2d(x.double().permute(0, 3, 1, 2), w.double().view(k, k, cin, cout).permute(3, 2, 0, 1),
                                     padding=k // 2).permute(0, 2, 3, 1)
    ref = (ref * scale.double() + shift.double()).clamp_min(0)
    tol = 2e-5 * max(ref.abs().max().item(), 1.0)
    assert (f32[..., :cout].double() - ref).abs().max().item() < tol
    assert (sp.float().double() - ref).abs().max().item() < tol


def _map(dev, B, H, W, C, cells, seed=3):
    """A split BEV map scattered from the active cells `cells` [(frame, y, x)]."""
    from sassd_b200 import ops
    g = torch.Generator().manual_seed(seed)
    cap = torch.zeros((max(len(cells), 1), 4), dtype=torch.int32)
    for i, (b, y, x) in enumerate(cells):
        cap[i, 0], cap[i, 2], cap[i, 3] = b, y, x
    feat = torch.randn(cap.shape[0], C, generator=g).to(dev)
    d_rows = torch.tensor([len(cells)], dtype=torch.int32, device=dev)
    return ops.sparse_to_bev_split(feat, cap.to(dev), d_rows, C, 1, H, W, B)


# 256 output channels: two 128-channel units per tile
_LAYERS = [(9, 64, 256), (9, 256, 256), (9, 256, 256)]


def _params(dev, seed):
    g = torch.Generator().manual_seed(seed)
    return [((torch.randn(t, ci, co, generator=g) * (1.2 / (t * ci) ** 0.5)).to(dev),
             (torch.rand(co, generator=g) + 0.5).to(dev), (torch.randn(co, generator=g) * 0.3).to(dev))
            for t, ci, co in _LAYERS]


def _chain(x, params):
    from sassd_b200 import ops
    outs = []
    for (t, ci, co), (w, sc, sh) in zip(_LAYERS, params):
        x, _ = ops.conv2d_split(x, w, sc, sh, True, co)
        outs.append(x)
    return outs


def _tile_center(j, i):
    return j * TH + TH // 2, i * TW + TW // 2


# Cells at tile centres are more than 3 pixels from every other tile: each marks exactly one tile computed at every
# layer of the chain (reach 1..3).
_CASES = {
    "one": (1, 56, 80, [(0,) + _tile_center(3, 2)]),
    "odd": (2, 56, 80, [(0,) + _tile_center(3, 2), (1,) + _tile_center(1, 1), (1,) + _tile_center(5, 3)]),
    "none": (2, 56, 80, []),
    # 16 frames of the detector's grid: 4400 tiles, the most the kernel keeps a tile order for in shared memory
    "b16": (16, 200, 176, [(b,) + _tile_center((3 * b) % 25, (5 * b) % 11) for b in range(15)] +
            [(b, 20 + 7 * b, 30 + 9 * b) for b in range(15)]),
    # 24 frames: 6600 tiles, walked without that order
    "b24": (24, 200, 176, [(b,) + _tile_center((3 * b) % 25, (5 * b) % 11) for b in range(23)] +
            [(b, 20 + 7 * b, 30 + 6 * b) for b in range(23)]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("order", [0, 1])
@pytest.mark.parametrize("case", sorted(_CASES))
def test_skipping_chain_bit_identical(dev, case, order):
    """Constant and background tiles, few or no computed tiles: the skipping chain equals every tile computed."""
    from sassd_b200 import ops
    B, H, W, cells = _CASES[case]
    params = _params(dev, 5)
    order0, ops.CONV2D_TILE_ORDER = ops.CONV2D_TILE_ORDER, order
    try:
        skip = _chain(_map(dev, B, H, W, 64, cells), params)
        ops.TILE_OCCUPANCY = False
        plain = _chain(_map(dev, B, H, W, 64, cells), params)
    finally:
        ops.TILE_OCCUPANCY = True
        ops.CONV2D_TILE_ORDER = order0
    torch.cuda.synchronize()
    assert [x.reach for x in skip] == [1, 2, 3] and plain[0].tile_dist is None
    for i, (a, b) in enumerate(zip(skip, plain)):
        assert torch.equal(a.planes, b.planes), "layer %d differs" % i
    if case == "one":
        dist = skip[0].tile_dist.view(-1).cpu().numpy()
        assert all(int((dist <= r).sum()) == 1 for r in (1, 2, 3))


class _Lazy(dict):
    def __init__(self, dev):
        super().__init__()
        self.dev = dev

    def get(self, label, default=None):
        if label not in self:
            self[label] = torch.zeros(2, dtype=torch.int32, device=self.dev)
        return self[label]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["odd", "b16", "b24"])
def test_counters_equal_the_host_count(dev, case):
    """The kernel counts each computed tile once (not once per 128-channel unit): the tiles within `reach`."""
    from sassd_b200 import ops
    B, H, W, cells = _CASES[case]
    params = _params(dev, 7)
    x0 = _map(dev, B, H, W, 64, cells)
    _chain(x0, params)                       # constants and backgrounds are built here, uncounted
    ops.CONV2D_COUNTERS = _Lazy(dev)
    try:
        outs = _chain(x0, params)
        torch.cuda.synchronize()
        counts = {k: [int(v) for v in c.cpu()] for k, c in ops.CONV2D_COUNTERS.items()}
    finally:
        ops.CONV2D_COUNTERS = None
    dist = x0.tile_dist.cpu().numpy()
    # the two 256 -> 256 layers share a label: their counts add up
    want = {}
    for (t, ci, co), x in zip(_LAYERS, outs):
        label = "conv2d_tma[taps=%d %d->%d]" % (t, ci, co)
        c, n = want.get(label, (0, 0))
        want[label] = (c + int((dist <= x.reach).sum()), n + dist.size)
    assert counts == {k: list(v) for k, v in want.items()}
    per_frame = dist.reshape(B, (H + TH - 1) // TH, (W + TW - 1) // TW)
    assert sum(int((tile_kinds(d, 3) == 2).sum()) for d in per_frame) > 0


@pytest.mark.gpu
@pytest.mark.parametrize("order", [0, 1])
def test_graph_replay_equals_eager(dev, order):
    """The chain captured in a CUDA graph and replayed gives the eager launch's outputs bit for bit."""
    from sassd_b200 import ops
    B, H, W, cells = _CASES["odd"]
    params = _params(dev, 9)
    order0, ops.CONV2D_TILE_ORDER = ops.CONV2D_TILE_ORDER, order
    try:
        x0 = _map(dev, B, H, W, 64, cells)
        eager = [x.planes.clone() for x in _chain(x0, params)]      # also warms packs, constants and backgrounds
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                captured = _chain(x0, params)
        torch.cuda.current_stream().wait_stream(s)
        for x in captured:
            x.planes.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
    finally:
        ops.CONV2D_TILE_ORDER = order0
    for i, (a, x) in enumerate(zip(eager, captured)):
        assert torch.equal(a, x.planes), "layer %d differs" % i
