"""The BEV neck's per-tile ready counters (ops.tile_ready_arena, sassd_conv2d_desc.in_ready / out_ready): conv1-conv7
start each tile once the tiles it reads of the previous map are stored instead of waiting for the whole previous layer.
That changes when a unit runs, never what it sums, so every BEV map and the head map are compared bit for bit with the
counters on and off: eager with programmatic launches, and the captured latency graph at batch 1 and 16 replayed with
frames A, B, A (the counters are zeroed per step, never by a kernel)."""
import collections
import ctypes

import pytest
import torch

from tests.test_frame_independence import MAXPTS, _assert_same, _frames, _slot
from tests.test_gpu_parity import _make_model

TH, TW = 8, 16                  # SASSD_CONV2D_TILE_H / _W


def _waited_tiles(ty, tx, taps, tiles_y, tiles_x):
    """The input tiles the kernel's TMA lane waits for before a unit of tile (ty, tx) loads (wait_input_tiles)."""
    h = 1 if taps == 9 else 0
    return {(y, x) for y in range(max(ty - h, 0), min(ty + h, tiles_y - 1) + 1)
            for x in range(max(tx - h, 0), min(tx + h, tiles_x - 1) + 1)}


@pytest.mark.parametrize("taps", [9, 1])
@pytest.mark.parametrize("H,W", [(200, 176), (50, 70), (8, 16), (9, 17)])
def test_waited_tiles_cover_every_box_pixel(taps, H, W):
    """Every in-image pixel the unit's halo boxes read (per tap column dx one box of TILE_H + 2 halo rows and TILE_W
    columns at (y0 - halo, x0 + dx)) lies in a waited tile, edge and partial tiles included; out-of-image pixels are
    TMA's zero fill and need no tile."""
    tiles_y, tiles_x = (H + TH - 1) // TH, (W + TW - 1) // TW
    halo = 1 if taps == 9 else 0
    for ty in range(tiles_y):
        for tx in range(tiles_x):
            waited = _waited_tiles(ty, tx, taps, tiles_y, tiles_x)
            y0, x0 = ty * TH, tx * TW
            ys = [y for y in range(y0 - halo, y0 + TH + halo) if 0 <= y < H]
            xs = {x for dx in range(-halo, halo + 1) for x in range(x0 + dx, x0 + dx + TW) if 0 <= x < W}
            need = {(y // TH, x // TW) for y in ys for x in xs}
            assert need <= waited, "tile (%d, %d) of %dx%d, %d taps: unwaited %s" % (ty, tx, H, W, taps,
                                                                                sorted(need - waited))
            assert len(waited) <= (2 * halo + 1) ** 2


# ------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def model(dev):
    return _make_model(dev)[0]


@pytest.fixture(scope="module")
def frames():
    return _frames()


# "edge" computes tiles on every border of the map; "empty" and "outside" frames have no voxels
BATCHES = {1: (["edge"], ["dense"]),
           16: (["dense", "empty", "edge", "wide", "outside", "sparse", "one", "crowded"] * 2, ["empty", "maxpts"] * 8)}


def _maps(aux, B):
    """Frame by frame: the split planes of conv7's output and of conv6, and the head map, on the host."""
    return [{n: _slot(aux[n], b).cpu().numpy() for n in ("x", "conv6", "head")} for b in range(B)]


def _counting_arena(monkeypatch):
    """ops.tile_ready_arena, recording whether it handed out counters."""
    from sassd_b200 import ops
    real, used = ops.tile_ready_arena, []

    def arena(x, maps):
        r = real(x, maps)
        used.append(r is not None)
        return r
    monkeypatch.setattr(ops, "tile_ready_arena", arena)
    return used


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 16])
def test_tile_flags_keep_every_bev_map_bit_for_bit(model, frames, monkeypatch, B):
    """Counters off, then on (at batch 16 forced on: by default only batch 1 uses them), empty frames beside full
    ones."""
    from sassd_b200 import ops
    lib = ops._lib.load()
    monkeypatch.setattr(ops, "TILE_FLAGS_MAX_BATCH", 16)
    a, b = BATCHES[B]
    seq = [a, b, a]
    used = _counting_arena(monkeypatch)
    ref = {}
    for flags in (False, True):
        monkeypatch.setattr(ops, "CONV2D_TILE_FLAGS", flags)
        # eager, launched as programmatic dependents (the counters need PDL)
        prev = lib.sassd_set_pdl(1)
        try:
            for s in seq[:2]:
                used.clear()
                _, aux = model.forward_points([frames[n] for n in s], return_aux=True)
                assert used == [flags]
                got = _maps(aux, B)
                if not flags:
                    ref[tuple(s)] = got
                for b, n in enumerate(s):
                    _assert_same(got[b], ref[tuple(s)][b], "eager B=%d flags=%s: %s at slot %d" % (B, flags, n, b))
        finally:
            lib.sassd_set_pdl(prev)
        # the captured latency graph, replayed A, B, A
        used.clear()
        g = model.enable_cuda_graph(B, MAXPTS)
        try:
            assert used and all(u == flags for u in used)
            for i, s in enumerate(seq):
                model.forward_points([frames[n] for n in s])
                got = _maps(g.aux, B)
                for b, n in enumerate(s):
                    _assert_same(got[b], ref[tuple(s)][b], "graph B=%d flags=%s step %d: %s at slot %d" % (
                        B, flags, i, n, b))
        finally:
            model.disable_cuda_graph()


@pytest.mark.gpu
def test_tile_flags_with_cold_caches(model, frames, monkeypatch):
    """The first call after the layer caches are emptied (weight packs, constant vectors, backgrounds, the neck's
    weights and folded BatchNorm) queues their work between the convs: each conv whose preparation launched anything
    waits for it instead of polling the counters, and the maps are the same bits as with the counters off."""
    from sassd_b200 import ops
    lib = ops._lib.load()
    fcn = model.neck.fcn
    pts = [frames["edge"]]

    def cold():
        monkeypatch.setattr(ops, "_TC_PACKS", {})
        monkeypatch.setattr(ops, "_CONV_CONSTS", {})
        monkeypatch.setattr(ops, "_BACKGROUNDS", collections.OrderedDict())
        monkeypatch.setattr(fcn, "_packed", {})
        for i in range(8):
            monkeypatch.delattr(getattr(fcn, "bn%d" % i), "_sassd_fold", raising=False)

    used = _counting_arena(monkeypatch)
    prev = lib.sassd_set_pdl(1)
    try:
        got = {}
        for flags in (False, True):
            monkeypatch.setattr(ops, "CONV2D_TILE_FLAGS", flags)
            cold()
            fills = ops._CONV2D_FILLS
            used.clear()
            _, aux = model.forward_points(pts, return_aux=True)
            assert used == [flags] and ops._CONV2D_FILLS > fills
            got[flags] = _maps(aux, 1)[0]
    finally:
        lib.sassd_set_pdl(prev)
    _assert_same(got[True], got[False], "cold caches, counters on vs off")


@pytest.mark.gpu
def test_tile_flags_need_pdl_and_a_status_word(dev):
    """The counters are handed out only where they can work and pay: launches programmatic, a status word to report a
    timed-out wait in, at most TILE_FLAGS_MAX_BATCH frames; the C entry point refuses them for cout <= 64, for stored
    channels past the units' (a zero tail, whose stores are not counted) and for in_ready without a status word."""
    from sassd_b200 import ops
    lib = ops._lib.load()
    st = torch.zeros((1,), dtype=torch.int32, device=dev)
    x = ops.SplitMap(torch.zeros((2, 2, 24, 40, 64), dtype=torch.float16, device=dev), 64, status=st)
    prev = lib.sassd_set_pdl(0)
    try:
        assert ops.tile_ready_arena(x, 3) is None
        lib.sassd_set_pdl(1)
        assert ops.tile_ready_arena(ops.SplitMap(x.planes, 64), 3) is None
        assert ops.TILE_FLAGS_MAX_BATCH == 1 and ops.tile_ready_arena(x, 3) is None      # two frames
        ops.TILE_FLAGS_MAX_BATCH = 2
        try:
            arena = ops.tile_ready_arena(x, 3)
        finally:
            ops.TILE_FLAGS_MAX_BATCH = 1
        assert len(arena) == 3 and all(a.shape == (2 * 3 * 3 + 1,) and not a.any() for a in arena)
    finally:
        lib.sassd_set_pdl(prev)
    w = torch.zeros((9, 64, 32), device=dev)
    with pytest.raises(ops._lib.SassdError):
        ops.conv2d_split(x, w, None, None, True, 32, out_ready=arena[0])
    # real buffers of the right sizes: the calls must fail on the counters alone
    wp = ops.conv2d_pack_cached(torch.zeros((9, 64, 128), device=dev))
    out = torch.zeros((2, 2, 24, 40, 192), dtype=torch.float16, device=dev)

    def call(cout, out_ch, in_ready, out_ready, status):
        d = ops.Conv2dDesc()
        d.batch, d.H, d.W, d.cin, d.cin_stored, d.cout, d.taps, d.relu = 2, 24, 40, 64, 64, cout, 9, 1
        d.out_split_ch = out_ch
        d.in_ready = None if in_ready is None else ops._ptr(in_ready).value
        d.out_ready = None if out_ready is None else ops._ptr(out_ready).value
        return lib.sassd_conv2d_f16x3_occ_bg_status(ctypes.byref(d), ops._ptr(x.planes), ops._ptr(wp), None, None,
                                                    None, ops._ptr(out), None, 0, None, None, None, None,
                                                    ops._ptr(status), ops._stream())
    assert call(128, 128, arena[0], None, None) == -1                    # in_ready without a status word
    assert call(128, 192, None, arena[1], st) == -1                      # channels 128..191 would be a zero tail
    assert call(128, 192, arena[0], arena[1], st) == -1
    torch.cuda.synchronize()
    assert int(st.item()) == 0 and not any(a.any() for a in arena)
