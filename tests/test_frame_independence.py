"""A frame's outputs are a function of that frame alone: not of its slot in the batch, the other frames beside it,
the kind of step (eager, the captured latency graph, a detect_stream slot) or what the same captured graph ran before.

Round-off tolerances (tests/test_gpu_parity.py) can hide leakage between frames - a halo read from the neighbouring
frame, a capacity computed over the batch, a counter or hash slot left by the previous replay - so the same frame in
different surroundings is compared bit for bit.  Two scheduling decisions of the split-row sparse conv
(csrc/spconv_split.cu) are made over the concatenated rows of all frames and change a row's fp32 summation order:

  * the chunk deal (ops.SPCONV_TAP_SPLIT): a layer with at most as many 128-row tiles as CTAs may cut tiles between
    CTAs and sum the pieces' fp32 partials; whether it deals, and where it cuts, depends on every frame's rows;
  * the tap rotation (ops.SPCONV_TAP_ROTATE): each tile walks its K chunks from a chunk that depends on the tile's
    index, i.e. on how many rows the frames before it have.

With both off no stage of the step makes a decision that depends on other frames, and every per-frame quantity is
bit-identical (test 1).  The same frames in the same step kind are bit-identical whatever ran before (test 2).  With
the defaults a frame's backbone output may differ only by fp32 summation order, bounded in test 3.
"""
import numpy as np
import pytest
import torch

from sassd_b200.synth import synth_cloud
from tests.test_detector_set import SHAPES, _calibs
from tests.test_front_end_edges import RG, VS, b23_coords, crowded_cloud, cut_cloud, edge_cloud, nonfinite_cloud
from tests.test_gpu_parity import _compare_frame, _make_model
from tests.test_sparse_chunk_deal import _grid, _tile_masks, active_chunks, deal, takes_deal

f32 = np.float32
GRID = (40, 1600, 1408)           # z, y, x cells of the detector's voxel grid
MAXPTS = 40000                    # max_points_per_frame of the captured graphs in test 2
CONFIGS = [("car_cfg.py", 1, "f16x3"), ("car_cfg.py", 1, "fp32"), ("multi_cfg.py", 3, "f16x3"),
           ("multi_cfg.py", 3, "fp32")]


def _centres(cells):
    """Points at the centres of voxel cells (z, y, x) of the detector's grid."""
    c = np.asarray(cells, np.float64)
    pts = np.stack([RG[0] + (c[:, 2] + 0.5) * VS[0], RG[1] + (c[:, 1] + 0.5) * VS[1], RG[2] + (c[:, 0] + 0.5) * VS[2],
                    np.full(len(c), 0.5)], 1)
    return pts.astype(f32)


def _grid_edge_frame():
    """Voxels on the corners, edges and faces of the 1408 x 1600 x 40 grid (BEV halos and anchors reach the map border)
    beside edge_cloud's points one ulp either side of the range and cell faces."""
    Z, Y, X = (g - 1 for g in GRID)
    corners = [(z, y, x) for z in (0, Z) for y in (0, Y) for x in (0, X)]
    edges = [(z, y, x) for z in (0, 20, Z) for y in (0, 1, 800, Y - 1, Y) for x in (0, 1, 704, X - 1, X)]
    faces = [(z, y, x) for z in range(0, 40, 3) for y in (0, Y) for x in range(0, 1408, 97)]
    faces += [(z, y, x) for z in range(0, 40, 3) for y in range(0, 1600, 101) for x in (0, X)]
    return np.concatenate([_centres(np.unique(np.array(corners + edges + faces), axis=0)), edge_cloud()], 0)


def _frames():
    """Every kind of frame, by name."""
    dense = synth_cloud(12, fov_deg=180.0)
    assert dense.shape[0] > MAXPTS
    far = synth_cloud(5)
    far[:, 0] = -far[:, 0]                     # x < 0: every point outside the range, 0 voxels
    return {
        "dense": synth_cloud(0), "dense9": synth_cloud(9), "sparse": synth_cloud(11, fov_deg=28.0, az_step_deg=0.6912),
        "wide": synth_cloud(3, fov_deg=45.0),
        "cut": dense,                          # a full sweep: exactly max_voxels = 20000 voxels
        "maxpts": dense[:MAXPTS].copy(),       # exactly the captured graphs' max_points_per_frame
        "empty": np.zeros((0, 4), f32), "one": np.array([[20.0, 1.5, -1.0, 0.4]], f32), "outside": far,
        "edge": _grid_edge_frame(), "crowded": crowded_cloud("shuffled")[0], "cutopen": cut_cloud(8192),
        "nonfinite": nonfinite_cloud()[0],
    }


TARGETS = ["dense", "edge", "cut"]            # the frames compared alone and in batches
SLOTS = [0, 7, 15]


def _batch16(frames, k):
    """Batch k (0..2) of 16: TARGETS at SLOTS (rotated by k) and every other kind of frame around them, in an order
    that also changes with k."""
    others = [n for n in frames if n not in TARGETS]
    others = others[k:] + others[:k]
    names = [None] * 16
    for j, s in enumerate(SLOTS):
        names[s] = TARGETS[(j + k) % 3]
    it = iter(others * 2)
    return [n if n is not None else next(it) for n in names]


def _b23_frames():
    """test_front_end_edges.b23_coords' 23 frames as voxel-centre clouds (frame 0 holds cell (0,0,0), frame 22 the far
    corner): the keys of the last frame's level-0 hash exceed 2e9."""
    c = b23_coords()
    return [_centres(c[c[:, 0] == b, 1:]) for b in range(23)]


# ------------------------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def models(dev):
    """Each (config, precision) model is built once per module."""
    cache = {}

    def get(cfg, ncls, prec):
        if (cfg, prec) not in cache:
            cache[(cfg, prec)] = _make_model(dev, num_class=ncls, cfg_name=cfg, prec=prec)[0]
        return cache[(cfg, prec)]
    return get


@pytest.fixture(scope="module")
def frames():
    return _frames()


@pytest.fixture(scope="module")
def metas(frames, golden_dir):
    """One img_meta per frame name (the same calibration, image shape and sample index wherever the frame sits)."""
    calibs = _calibs(golden_dir)
    names = list(frames) + ["b23_%d" % b for b in range(23)]
    return {n: dict(calib=calibs[i % 2], img_shape=SHAPES[i % 3], sample_idx=100 + i) for i, n in enumerate(names)}


@pytest.fixture
def deal_off(monkeypatch):
    """The sparse convs' batch-dependent schedule choices off: no chunk deal, every tile walks its chunks from 0."""
    from sassd_b200 import ops
    monkeypatch.setattr(ops, "SPCONV_TAP_SPLIT", False)
    monkeypatch.setattr(ops, "SPCONV_TAP_ROTATE", False)


# ------------------------------------------------------------------------------------------------- per-frame outputs
def _slot(t, b):
    """Frame b of a BEV map: the fp16 split planes of an ops.SplitMap, else the fp32 NHWC map."""
    return t.planes[:, b] if hasattr(t, "planes") else t[b]


def _per_frame(ret, b):
    """Every per-frame quantity of forward_points(..., metas=, point_outputs=True, return_aux=True) for frame b, as
    host arrays cut to the frame's rows or slot."""
    annos, pts, aux = ret
    fr = aux["frame_rows"].cpu().numpy()
    sp = aux["sparse"]
    idx = sp.indices
    rows = (idx[:, 0] == b).nonzero().view(-1)
    k = int(aux["d_k"][b])
    nd = int(aux["ndet"][b])
    out = dict(coors=aux["coors"][fr[b]:fr[b + 1], 1:], mask=aux["mask"][b], sparse_idx=idx[rows, 1:],
               sparse=sp.features[rows], x=_slot(aux["x"], b), conv6=_slot(aux["conv6"], b), head=aux["head"][b],
               d_k=aux["d_k"][b], guided=aux["guided"][b, :k], labels=aux["guided_labels"][b, :k],
               index=aux["guided_index"][b, :k], ps_scores=aux["ps_scores"][b, :k], det=aux["det"][b, :nd])
    out = {n: v.cpu().numpy() for n, v in out.items()}
    for n, v in annos[b].items():
        out["kitti_" + n] = np.asarray(v)
    for n, v in pts[b].items():
        out["points_" + n] = v
    return out


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view(np.uint8) if a.dtype.kind in "fciub" else a


def _assert_same(got, exp, tag):
    assert got.keys() == exp.keys(), tag
    for n in exp:
        g, e = got[n], exp[n]
        assert g.shape == e.shape, "%s: %s shape %s vs %s" % (tag, n, g.shape, e.shape)
        if not np.array_equal(_bits(g), _bits(e)):
            bad = np.argwhere(_bits(g).reshape(g.shape + (-1,)) != _bits(e).reshape(e.shape + (-1,)))
            raise AssertionError("%s: %s differs at %d places, first %s" % (tag, n, len(bad), bad[:3].tolist()))


def _step(model, frames, names, metas):
    return model.forward_points([frames[n] for n in names], metas=[metas[n] for n in names], point_outputs=True,
                                return_aux=True)


# ------------------------------------------------------------------------------------------------- test 1
@pytest.mark.gpu
@pytest.mark.parametrize("cfg,ncls,prec", CONFIGS)
def test_frame_alone_equals_frame_in_any_batch(models, frames, metas, deal_off, cfg, ncls, prec):
    """Deal and tap rotation off: every per-frame quantity of a frame run alone (eager, batch 1) equals, bit for bit,
    the same frame at slots 0, 7 and 15 of batches of 16 beside every other kind of frame, and at slot 22 of a batch of
    23 (the largest the level-0 hash keys).  Bit for bit because no stage then makes a decision over other frames:
    the voxelizer, the hashes and the rulebooks key cells by frame; the sparse convs sum each row's taps in one fixed
    order; the BEV scatter, the dense convs' tiles, their constant-region distances and the anchor masks are per frame;
    decoding, PSWarp, rescoring, NMS and the KITTI formatter run per frame with per-frame capacities."""
    model = models(cfg, ncls, prec)
    alone = {n: _per_frame(_step(model, frames, [n], metas), 0) for n in TARGETS}
    assert alone["cut"]["coors"].shape[0] == 20000 and alone["dense"]["det"].shape[0] > 0
    for k in range(3):
        names = _batch16(frames, k)
        ret = _step(model, frames, names, metas)
        for s in SLOTS:
            _assert_same(_per_frame(ret, s), alone[names[s]], "%s %s: %s at slot %d of %s" % (cfg, prec, names[s], s,
                                                                                               names))
    b23 = _b23_frames()
    fr23 = dict(frames, **{"b23_%d" % b: f for b, f in enumerate(b23)})
    names = ["b23_%d" % b for b in range(22)] + ["edge"]
    ret = _step(model, fr23, names, metas)
    _assert_same(_per_frame(ret, 22), alone["edge"], "%s %s: edge at slot 22 of 23" % (cfg, prec))
    # frame 22 of the b23 batch alone vs in its batch: the far-corner keys above 2e9
    _assert_same(_per_frame(ret, 21), _per_frame(_step(model, fr23, ["b23_21"], metas), 0), "b23_21 at slot 21")


# ------------------------------------------------------------------------------------------------- test 2
def _host(res, pts=None):
    """A step's host results as one flat dict of arrays (detection dicts or KITTI annos, then point outputs)."""
    out = {}
    for b, r in enumerate(res):
        for n, v in r.items():
            out["%d_%s" % (b, n)] = np.asarray(v) if v is not None else np.zeros(0)
    for b, p in enumerate(pts or []):
        for n, v in p.items():
            out["%d_points_%s" % (b, n)] = v
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("dealt", [True, False], ids=["deal_on", "deal_off"])
def test_step_kinds_and_history_give_the_same_bits(models, frames, metas, monkeypatch, dealt):
    """Eager, the captured latency graph (batch 1 and 16: PDL on, computed tiles first), detect_stream slots at batch 16
    (PDL off, round-robin tiles, two in flight) and the KITTI-formatting + point-outputs graph give the same bits for
    the same frames, replayed as A, then a denser batch B, A, an all-empty batch, A: no hash table, deal counter, row
    count or capacity is left over from the step before.  Bit for bit because every step kind makes the same
    decisions on the same frames: the deal and the tap rotation see the same rows, and the dense convs' tile order
    and PDL change when a tile runs, not what it sums.  With the deal on (the default) and off."""
    from sassd_b200 import ops
    if not dealt:
        monkeypatch.setattr(ops, "SPCONV_TAP_SPLIT", False)
    model = models("car_cfg.py", 1, "f16x3")
    small = [n for n in frames if n != "cut"]                     # everything that fits MAXPTS
    seqs = {1: [["dense"], ["maxpts"], ["dense"], ["empty"], ["dense"]],
            16: [small + small[:16 - len(small)], ["maxpts", "wide"] * 8, None, ["empty"] * 16, None]}
    for B, seq in seqs.items():
        seq[2] = seq[4] = seq[0]
        assert all(len(s) == B for s in seq)
        eager = {}
        for s in seq:
            key = tuple(s)
            if key not in eager:
                pts = [frames[n] for n in s]
                annos, points = model.forward_points(pts, metas=[metas[n] for n in s], point_outputs=True)
                eager[key] = (_host(model.forward_points(pts)), _host(annos, points))
        model.enable_cuda_graph(B, MAXPTS)
        try:
            for i, s in enumerate(seq):
                pts = [frames[n] for n in s]
                _assert_same(_host(model.forward_points(pts)), eager[tuple(s)][0], "graph B=%d step %d" % (B, i))
                annos, points = model.forward_points(pts, metas=[metas[n] for n in s], point_outputs=True)
                _assert_same(_host(annos, points), eager[tuple(s)][1], "KITTI + points graph B=%d step %d" % (B, i))
        finally:
            model.disable_cuda_graph()
        if B == 16:
            got = list(model.detect_stream([[frames[n] for n in s] for s in seq], 16, MAXPTS, depth=2, concurrent=True))
            for i, (s, g) in enumerate(zip(seq, got)):
                _assert_same(_host(g), eager[tuple(s)][0], "detect_stream step %d" % i)


# ------------------------------------------------------------------------------------------------- test 3
def _sum_bound(scale, absdot, out):
    """|a - b| for two fp32 evaluations of one output row of the layer that sum the same products in different orders.

    The accumulator of a row adds, per 64-wide K chunk, 64 products hi*hi (and 128 cross products hi*lo + lo*hi into
    the small accumulator, weighted 1/2048), over at most 27 chunks, plus at most 27 partial sums of the pieces of a
    cut tile: N = 2 * 27 * 64 + 27 + 2 additions.  Each may err by 2u of its result (u = 2^-24, a truncating tensor-core
    accumulation allowed), so each evaluation is within N * 2u * sum|x||w| of the exact sum of the products (first
    order), and the two within twice that.  The products' magnitudes sum to at most (1 + 2^-10) sum|x||w| (hi/lo split
    of both operands), rounded up to 1.01.  The epilogue scale * acc + shift (one fmaf, rounded once in each run) adds
    2u |out|; ReLU does not widen a difference."""
    u = 2.0 ** -24
    N = 2 * 27 * 64 + 27 + 2
    return np.abs(scale)[None, :] * (2 * N * 2 * u * 1.01) * absdot + 2 * u * np.abs(out)


@pytest.mark.gpu
def test_chunk_deal_and_tap_rotation_bounded_at_one_layer(dev, monkeypatch):
    """One 64 -> 64 spconv_split layer on identical inputs: 40 tiles, every 6th with all 27 taps, so the deal is taken;
    the same rows padded past 132 tiles (more tiles than CTAs: never dealt); and the deal off.  Rows of tiles the deal
    does not cut are bit-identical in all three (a whole tile is summed by one CTA in the same chunk order); rows of cut
    tiles, and every row with the tap rotation off against on, are within _sum_bound of each other."""
    from sassd_b200 import ops
    rs = np.random.RandomState(41)
    taps, cin, cout = 27, 64, 64
    n, n_pad = 40 * 128 - 9, 140 * 128
    x = rs.randn(n_pad, cin).astype(f32)
    w = (rs.randn(taps, cin, cout) * 0.1).astype(f32)
    scale = (rs.rand(cout) + 0.5).astype(f32)
    shift = (rs.randn(cout) * 0.1).astype(f32)
    nb = np.where(rs.rand(n_pad, taps) < 0.3, rs.randint(0, n, (n_pad, taps)), -1).astype(np.int32)
    gone = rs.rand(n_pad // 128, taps) < 0.75
    gone[::6] = False
    nb[np.repeat(gone, 128, axis=0)] = -1
    nb[n:40 * 128] = -1
    t = lambda a: torch.from_numpy(a).to(dev)
    planes = ops.features_to_split(t(x))
    W, sc, sh = t(w), t(scale), t(shift)

    def run(rows, split, rotate):
        monkeypatch.setattr(ops, "SPCONV_TAP_SPLIT", split)
        monkeypatch.setattr(ops, "SPCONV_TAP_ROTATE", rotate)
        nbr = t(np.ascontiguousarray(nb[:rows]))
        tm = t(_tile_masks(nb[:rows], rows))
        _, of = ops.spconv_split(planes, W, sc, sh, True, cout, rows, nbr=nbr,
                                 d_rows=torch.tensor([rows], dtype=torch.int32, device=dev), want_f32=True, tile_mask=tm)
        torch.cuda.synchronize()
        return of[:n, :cout].cpu().numpy()

    dealt = run(n, True, True)
    padded = run(n_pad, True, True)
    whole = run(n, False, True)
    fixed = run(n, False, False)
    masks = _tile_masks(nb[:n], n)
    counts = [len(active_chunks(int(m), 1, 27)) for m in masks]
    G = min(40 * 27, _grid())
    assert takes_deal(counts, G) and not takes_deal(counts * 4, G)
    ctas, _ = deal(counts, G)
    cut = sorted({it[0] for items in ctas for it in items if it[3] is not None})
    assert 0 < len(cut) < 40
    row_cut = np.zeros(n, bool)
    for tile in cut:
        row_cut[tile * 128:(tile + 1) * 128] = True
    assert np.array_equal(padded, whole), "undealt runs differ"
    assert np.array_equal(dealt[~row_cut], whole[~row_cut]), "rows of uncut tiles differ"
    xd, wd = np.abs(x.astype(np.float64)), np.abs(w.astype(np.float64))
    absdot = np.zeros((n, cout))
    for k in range(taps):
        o = np.nonzero(nb[:n, k] >= 0)[0]
        absdot[o] += xd[nb[o, k]] @ wd[k]
    bound = _sum_bound(scale.astype(np.float64), absdot, whole)
    assert np.all(np.abs(dealt - whole.astype(np.float64)) <= bound), "cut tiles beyond the summation bound"
    assert np.all(np.abs(fixed.astype(np.float64) - whole) <= bound), "tap rotation beyond the summation bound"


@pytest.mark.gpu
def test_frame_in_batch_with_the_default_deal(models, frames, metas):
    """The defaults (deal and tap rotation on): integer stages bit for bit, and the detections of a frame alone and in
    a batch of 16 within the oracle comparison's tolerances (tests/test_gpu_parity.py: matched as sets, scores to
    PS_CHAIN_ATOL, boxes to BOX_ATOL) - the backbone's rows may differ by the summation order bounded above."""
    model = models("car_cfg.py", 1, "f16x3")
    alone = {n: _step(model, frames, [n], metas) for n in TARGETS}
    names = _batch16(frames, 1)
    ret = _step(model, frames, names, metas)
    compared = 0
    for s in SLOTS:
        got, exp = _per_frame(ret, s), _per_frame(alone[names[s]], 0)
        for q in ("coors", "mask", "sparse_idx"):
            assert np.array_equal(got[q], exp[q]), "%s: %s at slot %d" % (q, names[s], s)
        det = lambda p: dict(boxes_lidar=p["det"][:, :7], scores=p["det"][:, 7]) if len(p["det"]) else \
            dict(boxes_lidar=None, scores=None)
        e = det(exp)
        compared += _compare_frame(det(got), (e["boxes_lidar"], e["scores"], None), "%s at slot %d" % (names[s], s))
    assert compared > 0


# ------------------------------------------------------------------------------------------------- test 4
@pytest.mark.gpu
def test_batch_24_refused_before_any_launch(models, frames, metas, deal_off):
    """24 frames exceed the level-0 hash's 31-bit keys: forward_points raises SassdError naming the limit before it
    launches a kernel, and the next call at batch 23 returns exactly what it returned before the refusal."""
    from sassd_b200 import ops
    from sassd_b200.lib import SassdError
    model = models("car_cfg.py", 1, "f16x3")
    b23 = _b23_frames()
    fr = {"b23_%d" % b: f for b, f in enumerate(b23)}
    names = list(fr)
    before = _step(model, fr, names, metas)
    launches = ops.LAUNCHES
    with pytest.raises(SassdError, match="hash limit of 23 frames"):
        model.forward_points(b23 + [frames["one"]])
    assert ops.LAUNCHES == launches, "kernels were launched before the refusal"
    after = _step(model, fr, names, metas)
    for b in (0, 11, 22):
        _assert_same(_per_frame(after, b), _per_frame(before, b), "b23 frame %d after the refusal" % b)
