"""Background tiles of the dense neck (DESIGN.md section 4): from the second conv on, a tile on the image border whose
distance to the nearest active cell exceeds `reach` sees only inactive cells and the zero padding, so its output is the
layer's output on an empty scene.  sassd_conv2d_f16x3_occ_bg copies such tiles from a per-layer background map instead
of computing them.  The CPU test restates the rule in fp64; the GPU tests hold the kernel to the full computation."""
import numpy as np
import pytest
import torch

from tests.test_constant_region_rule import TH, TW, skipping_valid, tile_distances


def tile_kinds(dist, reach):
    """Restates csrc/conv2d_tma.cu:tile_skip_flag with a background: 0 computed, 1 constant, 2 background."""
    kind = np.where(dist > reach, 1, 0)
    if reach >= 2:
        border = np.zeros(dist.shape, bool)
        border[0, :] = border[-1, :] = border[:, 0] = border[:, -1] = True
        kind[border & (dist > reach)] = 2
    return kind


def test_far_border_tiles_equal_the_chain_on_an_empty_map():
    H, W, C = 72, 112, 6
    torch.manual_seed(1)
    rs = np.random.RandomState(1)
    active = {(int(rs.randint(20, 50)), int(rs.randint(30, 80))) for _ in range(25)} | {(0, 0), (H - 1, 60)}
    x = torch.zeros(1, C, H, W, dtype=torch.float64)
    for y, xx in active:
        x[0, :, y, xx] = torch.randn(C, dtype=torch.float64)
    empty = torch.zeros_like(x)
    dist = tile_distances(sorted(active), H, W)
    layers = [(3, C, 8), (3, 8, 8), (3, 8, 8), (1, 8, 8), (3, 8, 5), (3, 5, 5), (3, 5, 5)]
    reach, copied = 0, 0
    for k, ci, co in layers:
        w = torch.randn(co, ci, k, k, dtype=torch.float64) * 0.4
        b = torch.randn(co, dtype=torch.float64) * 0.5 + 0.3
        x = torch.relu(torch.nn.functional.conv2d(x, w, b, padding=k // 2))
        empty = torch.relu(torch.nn.functional.conv2d(empty, w, b, padding=k // 2))
        reach += 1 if k == 3 else 0
        assert skipping_valid(H, W, reach)
        kind = tile_kinds(dist, reach)
        for j, i in zip(*np.nonzero(kind == 2)):
            win = (slice(None), slice(None), slice(j * TH, (j + 1) * TH), slice(i * TW, (i + 1) * TW))
            assert torch.allclose(x[win], empty[win], rtol=0, atol=1e-12), "reach %d tile (%d,%d)" % (reach, j, i)
            copied += 1
        # the border does differ from the layer constant: these tiles could not store it instead
        if reach >= 2:
            assert not torch.allclose(empty[0, :, 0, 0], empty[0, :, H // 2, W // 2])
    assert copied > 100


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _scattered_map(dev, B, H, W, C, seed):
    """A split BEV map whose active cells sit in one corner of every frame but the last (empty) one."""
    from sassd_b200 import ops
    g = torch.Generator().manual_seed(seed)
    n = 30
    coors = torch.zeros((n, 4), dtype=torch.int32)
    coors[:, 0] = torch.randint(0, max(B - 1, 1), (n,), generator=g)
    coors[:, 2] = torch.randint(0, 10, (n,), generator=g)
    coors[:, 3] = torch.randint(0, 18, (n,), generator=g)
    key = (coors[:, 0].long() * H + coors[:, 2].long()) * W + coors[:, 3].long()
    rows = coors[torch.from_numpy(np.unique(key.numpy(), return_index=True)[1])]
    cap = torch.zeros((64, 4), dtype=torch.int32)
    cap[: rows.shape[0]] = rows
    feat = torch.randn(64, C, generator=g).to(dev)
    d_rows = torch.tensor([rows.shape[0]], dtype=torch.int32, device=dev)
    return ops.sparse_to_bev_split(feat, cap.to(dev), d_rows, C, 1, H, W, B)


# 64 -> 256 -> 256 runs two 128-channel units per tile; 28 output channels: 32-wide units into 64 stored channels;
# the last layer also writes fp32
_LAYERS = [(9, 64, 64), (9, 64, 256), (9, 256, 256), (1, 256, 64), (9, 64, 28)]


def _params(dev, seed):
    g = torch.Generator().manual_seed(seed)
    return [((torch.randn(t, ci, co, generator=g) * (1.2 / (t * ci) ** 0.5)).to(dev),
             (torch.rand(co, generator=g) + 0.5).to(dev), (torch.randn(co, generator=g) * 0.3).to(dev))
            for t, ci, co in _LAYERS]


def _run_chain(dev, B, H, W, params, use_tiles):
    from sassd_b200 import ops
    ops.TILE_OCCUPANCY = use_tiles
    try:
        x = _scattered_map(dev, B, H, W, 64, 3)
        outs = []
        for i, ((t, ci, co), (w, sc, sh)) in enumerate(zip(_LAYERS, params)):
            last = i == len(_LAYERS) - 1
            x, f = ops.conv2d_split(x, w, sc, sh, True, co, out_split=True, out_f32=last)
            outs.append((x.planes.clone(), None if f is None else f.clone(), x.reach, x.background))
        torch.cuda.synchronize()
        return outs
    finally:
        ops.TILE_OCCUPANCY = True


@pytest.mark.gpu
@pytest.mark.parametrize("B,order", [(2, 0), (2, 1), (27, 0)])     # 27 frames: more tiles than the kernel orders
def test_background_tiles_chain_bit_identical(dev, B, order):
    """Skipping chain (constant and background tiles) == every tile computed, bit for bit, at every layer - also
    after the weights are reloaded in place, which must build new backgrounds."""
    from sassd_b200 import ops
    H, W = 56, 80
    params = _params(dev, 11)
    order0, ops.CONV2D_TILE_ORDER = ops.CONV2D_TILE_ORDER, order
    try:
        for reload in (False, True):
            if reload:
                for (w, sc, sh), (w2, sc2, sh2) in zip(params, _params(dev, 12)):
                    w.copy_(w2); sc.copy_(sc2); sh.copy_(sh2)
            skip, plain = _run_chain(dev, B, H, W, params, True), _run_chain(dev, B, H, W, params, False)
            assert [o[2] for o in skip] == [1, 2, 3, 3, 4]
            assert all(o[3] is not None for o in skip)
            for i, (a, b) in enumerate(zip(skip, plain)):
                assert torch.equal(a[0], b[0]), "split planes differ at layer %d (reload %s)" % (i, reload)
                assert (a[1] is None) == (b[1] is None)
                assert a[1] is None or torch.equal(a[1], b[1]), "fp32 map differs at layer %d" % i
            if not reload:
                before = skip[-1][3]
        assert skip[-1][3] is not before and not torch.equal(skip[-1][3].planes, before.planes)
    finally:
        ops.CONV2D_TILE_ORDER = order0


@pytest.mark.gpu
def test_counters_count_only_tiles_within_reach(dev):
    """The kernel counts the tiles it computes: exactly those within `reach` of an active cell once far border tiles
    copy the background."""
    from sassd_b200 import ops
    B, H, W = 2, 56, 80
    params = _params(dev, 21)
    x0 = _scattered_map(dev, B, H, W, 64, 5)
    dist = x0.tile_dist.cpu().numpy()

    class _Lazy(dict):
        def get(self, label, default=None):
            if label not in self:
                self[label] = torch.zeros(2, dtype=torch.int32, device=dev)
            return self[label]

    def chain():
        x, reach = x0, {}
        for (t, ci, co), (w, sc, sh) in zip(_LAYERS[:3], params[:3]):
            x, _ = ops.conv2d_split(x, w, sc, sh, True, co)
            reach["conv2d_tma[taps=%d %d->%d]" % (t, ci, co)] = x.reach
        return reach
    chain()                                  # constants and backgrounds are built here, uncounted
    ops.CONV2D_COUNTERS = _Lazy()
    try:
        reach = chain()
        torch.cuda.synchronize()
        counts = {k: [int(v) for v in c.cpu()] for k, c in ops.CONV2D_COUNTERS.items()}
    finally:
        ops.CONV2D_COUNTERS = None
    assert sorted(counts) == sorted(reach)
    per_frame = dist.reshape(B, (H + TH - 1) // TH, (W + TW - 1) // TW)
    for label, (computed, total) in counts.items():
        assert total == dist.size
        assert computed == int((dist <= reach[label]).sum()), label
    assert sum(int((tile_kinds(d, 3) == 2).sum()) for d in per_frame) > 0     # background tiles at reach 3
