"""The chunk deal of the split-row sparse conv (sa-ssd_b200/csrc/spconv_split.cu): a layer with at most as many
128-row tiles as CTAs deals its tiles' active K chunks evenly over the CTAs, and the pieces of a tile cut between CTAs
are reduced by whichever CTA counts last, in a fixed order.

CPU: a Python model of the deal arithmetic (the same integer formulas as the kernel).  GPU: ops.spconv_split on
hand-built neighbour tables and tile masks against an fp64 reference, at tile counts on both sides of the grid size."""
import numpy as np
import pytest

MAX_CTAS = 148          # sps::MAX_CTAS: the grid bound
DEAL_MIN_GAIN = 14      # sps::DEAL_MIN_GAIN: chunks the deal must save on the longest chain


def active_chunks(mask, tpg, nchunks):
    """Chunks the kernel runs for a tile with tap mask `mask` (a tile without any pair runs chunk 0)."""
    if mask == 0:
        mask = 1
    group = (1 << tpg) - 1
    return [g for g in range(nchunks) if (mask >> (g * tpg)) & group]


def takes_deal(counts, G):
    """The kernel's choice for a layer of len(counts) tiles: deal when it shortens the longest chain enough."""
    return len(counts) <= G and max(counts) - -(-sum(counts) // G) >= DEAL_MIN_GAIN


def deal(counts, G):
    """Per CTA, the items (tile, lo, hi) it runs - ranks [lo, hi) of the tile's active chunks - and for the pieces of
    shared tiles (first CTA, number of pieces, piece index, slot written, slots read), as the kernel derives them."""
    pre = np.concatenate([[0], np.cumsum(counts)]).astype(int)
    ntiles, S = len(counts), int(pre[-1])
    D = min(G, S)

    def tile_of(k):
        return int(np.searchsorted(pre[:ntiles], k, side="right") - 1)

    def owner_of(k):
        return ((k + 1) * D - 1) // S

    ctas = []
    for c in range(G):
        s0, s1 = (c * S // D, (c + 1) * S // D) if c < D else (0, 0)
        items = []
        if s1 > s0:
            t0 = tile_of(s0)
            for ii, t in enumerate(range(t0, tile_of(s1 - 1) + 1)):
                b, e = int(pre[t]), int(pre[t + 1])
                lo, hi = max(s0 - b, 0), min(s1, e) - b
                red = None
                if lo > 0 or hi < e - b:
                    first = owner_of(b)
                    nparts = owner_of(e - 1) - first + 1
                    read = [2 * (first + j) + (1 if j == 0 and (first + j) * S // D < b else 0) for j in range(nparts)]
                    red = dict(first=first, nparts=nparts, part=c - first, slot=2 * c + (1 if ii > 0 else 0),
                               read=read)
                items.append((t, lo, hi, red))
        ctas.append(items)
    return ctas, S


def _cases():
    rs = np.random.RandomState(0)
    out = [([27], 132), ([3], 132), ([1], 1), ([27] * 132, 132), ([5, 1, 27, 2], 3), ([1] * 7, 132)]
    for _ in range(300):
        G = int(rs.choice([1, 2, 3, 7, 64, 114, 132, 148]))
        ntiles = int(rs.randint(1, G + 1))
        out.append((list(rs.randint(1, 28, ntiles)), G))
    return out


@pytest.mark.parametrize("counts,G", _cases()[:6])
def test_deal_model_examples(counts, G):
    _check_deal(counts, G)


def test_deal_model_random():
    for counts, G in _cases()[6:]:
        _check_deal(counts, G)


def _check_deal(counts, G):
    ctas, S = deal(counts, G)
    seen = {}
    per_cta = []
    for c, items in enumerate(ctas):
        n = sum(hi - lo for _, lo, hi, _ in items)
        per_cta.append(n)
        partial = [i for i, (t, lo, hi, red) in enumerate(items) if red is not None]
        assert len(partial) <= 2, "CTA %d holds %d partial tiles" % (c, len(partial))
        assert all(i in (0, len(items) - 1) for i in partial), "a partial tile inside a CTA's range"
        for t, lo, hi, red in items:
            assert 0 <= lo < hi <= counts[t]
            for r in range(lo, hi):
                assert (t, r) not in seen, "chunk %d of tile %d dealt twice" % (r, t)
                seen[(t, r)] = c
    assert len(seen) == S == sum(counts), "every active chunk is dealt exactly once"
    assert max(per_cta) <= -(-S // G) and min(per_cta[:min(G, S)]) >= S // G, "even deal"
    # the pieces of each shared tile: as many as the owner formula says, pieces in CTA order, unique slots that the
    # finishing piece can find from the tile alone
    pieces = {}
    for c, items in enumerate(ctas):
        for t, lo, hi, red in items:
            if red is not None:
                pieces.setdefault(t, []).append((c, lo, red))
    slots = set()
    for t, ps in pieces.items():
        ps.sort()
        nparts = ps[0][2]["nparts"]
        assert nparts == len(ps) >= 2
        assert [p[1] for p in ps] == sorted(p[1] for p in ps)
        read = ps[0][2]["read"]
        for j, (c, lo, red) in enumerate(ps):
            assert red["part"] == j and red["first"] == ps[0][0] and red["nparts"] == nparts and red["read"] == read
            assert read[j] == red["slot"], "tile %d: piece %d written to slot %d, read from %d" % (t, j, red["slot"],
                                                                                                  read[j])
            assert red["slot"] not in slots
            slots.add(red["slot"])
            assert red["slot"] < 2 * MAX_CTAS


# ------------------------------------------------------------------------------------------------------------- GPU
def _grid():
    import torch
    return min(torch.cuda.get_device_properties(0).multi_processor_count, MAX_CTAS)


def _tile_masks(nb, n_rows):
    """What the rulebook kernels record: per 128-row tile, the taps that occur among its first n_rows rows."""
    M, taps = nb.shape
    nt = (M + 127) // 128
    pad = np.full((nt * 128, taps), -1, np.int64)
    pad[:n_rows] = nb[:n_rows]
    present = (pad.reshape(nt, 128, taps) >= 0).any(1)
    return (present * (1 << np.arange(taps))[None, :]).sum(1).astype(np.int32)


def _run(rows_cap, n_rows, cin, cout, seed, absent=0.4, density=0.3, empty_tiles=(), keep_taps=None, full_every=0):
    """One ruled conv (27 taps) on rows_cap output rows of which n_rows are live; returns the outputs of two launches,
    the fp64 reference, the counters of the first launch, the host rule's (executed chunks, tiles) and whether the
    layer takes the deal.  full_every: every full_every-th tile keeps all 27 taps (a long chain among short ones, as
    in a frame's 64-channel layers)."""
    import torch
    from sassd_b200 import ops
    dev = torch.device("cuda:0")
    rs = np.random.RandomState(seed)
    taps = 27
    x = torch.from_numpy(rs.randn(rows_cap, cin).astype(np.float32)).to(dev)
    w = torch.from_numpy((rs.randn(taps, cin, cout) * 0.1).astype(np.float32)).to(dev)
    scale = torch.from_numpy((rs.rand(cout) + 0.5).astype(np.float32)).to(dev)
    shift = torch.from_numpy((rs.randn(cout) * 0.1).astype(np.float32)).to(dev)
    nb = np.where(rs.rand(rows_cap, taps) < density, rs.randint(0, rows_cap, (rows_cap, taps)), -1).astype(np.int32)
    nt = (rows_cap + 127) // 128
    gone = rs.rand(nt, taps) < absent
    if keep_taps is not None:
        gone[:, :] = True
        gone[:, list(keep_taps)] = False
    if full_every:
        gone[::full_every, :] = False
    for t in empty_tiles:
        gone[t, :] = True
    nb[np.repeat(gone, 128, axis=0)[:rows_cap]] = -1
    masks = _tile_masks(nb, n_rows)
    nbr = torch.from_numpy(nb).to(dev)
    tm = torch.from_numpy(masks).to(dev)
    d_rows = torch.tensor([n_rows], dtype=torch.int32, device=dev)
    planes = ops.features_to_split(x)
    outs = []
    counters = torch.zeros(2, dtype=torch.int32, device=dev)
    saved = ops.SPCONV_COUNTERS
    try:
        for i in range(2):
            ops.SPCONV_COUNTERS = counters if i == 0 else None
            out, of = ops.spconv_split(planes, w, scale, shift, True, cout, rows_cap, nbr=nbr, d_rows=d_rows,
                                       want_f32=True, tile_mask=tm)
            outs.append((out.clone(), of.clone()))
    finally:
        ops.SPCONV_COUNTERS = saved
    torch.cuda.synchronize()
    xd, wd = x.double().cpu(), w.double().cpu()
    ref = torch.zeros(rows_cap, cout, dtype=torch.float64)
    nbl = nbr.cpu().long()
    for t in range(taps):
        o = torch.nonzero(nbl[:, t] >= 0).view(-1)
        ref.index_add_(0, o, xd[nbl[o, t]] @ wd[t])
    ref = (ref * scale.double().cpu() + shift.double().cpu()).clamp_min(0)
    ntiles = (n_rows + 127) // 128
    tpg = 64 // cin
    nchunks = (taps + tpg - 1) // tpg
    counts = [len(active_chunks(int(masks[t]), tpg, nchunks)) for t in range(ntiles)]
    grid = min(nt * nchunks, _grid())          # the kernel's grid: no more CTAs than the layer's chunks
    return outs, ref, counters.cpu().tolist(), (sum(counts), ntiles), takes_deal(counts, grid)


def _check(rows_cap, n_rows, cin, cout, seed, dealt, **kw):
    import torch
    from sassd_b200 import ops
    outs, ref, counters, host, takes = _run(rows_cap, n_rows, cin, cout, seed, **kw)
    assert takes == dealt, "the inputs do not exercise the path they are meant for"
    (out, of), (out2, of2) = outs
    n = n_rows
    sc = max(ref[:n].abs().max().item(), 1.0)
    e1 = (of[:n, :cout].double().cpu() - ref[:n]).abs().max().item()
    e2 = (ops.split_rows_float(out, cout)[:n].double().cpu() - ref[:n]).abs().max().item()
    # the tolerance of tests/tools/tc_check.py's split stage
    assert e1 < 2e-5 * sc and e2 < 2e-5 * sc, "err f32 %.3g split %.3g (|ref| %.3g)" % (e1, e2, sc)
    assert torch.equal(of[:n], of2[:n]) and torch.equal(out[:, :n], out2[:, :n]), "two launches differ"
    assert counters == list(host), "kernel counters %s, host rule %s" % (counters, host)


@pytest.mark.gpu
@pytest.mark.parametrize("which", ["1", "G/2", "G-1", "G", "G+1", "3G"])
def test_chunk_deal_tile_counts(which):
    G = _grid()
    ntiles = {"1": 1, "G/2": G // 2, "G-1": G - 1, "G": G, "G+1": G + 1, "3G": 3 * G}[which]
    cin = 64 if ntiles <= G else 16          # keeps the fp64 reference of the 3G case small
    rows = ntiles * 128 - 5
    _check(rows, rows, cin, 64 if cin == 64 else 32, seed=ntiles, dealt=ntiles <= G, absent=0.75, full_every=7)


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout", [(8, 16), (16, 16), (16, 32), (32, 32), (32, 64), (64, 16), (64, 32), (64, 64)])
def test_chunk_deal_channels(cin, cout):
    # 20 tiles of which 14 live (d_rows < rows_cap), one of them without any pair.  Narrow inputs have at most 4 / 7 / 14
    # chunks per tile: too few for the deal to pay, they run one CTA per tile.
    _check(20 * 128, 14 * 128 - 37, cin, cout, seed=cin * 100 + cout, dealt=cin == 64, absent=0.75, full_every=5,
           empty_tiles=(3,))


@pytest.mark.gpu
def test_chunk_deal_one_tile_over_many_ctas():
    # one 64-channel tile: its 27 chunks go to 27 CTAs, each a piece of the same tile
    _check(128, 120, 64, 64, seed=7, dealt=True, absent=0.0)


@pytest.mark.gpu
def test_chunk_deal_more_ctas_than_chunks():
    # one tile with 16 active taps: 16 CTAs share it, the rest of the grid has nothing to do
    _check(128, 128, 64, 64, seed=8, dealt=True, keep_taps=range(16))


@pytest.mark.gpu
def test_chunk_deal_tile_without_pairs():
    # only empty tiles: each runs its one all-zero chunk and writes act(shift)
    _check(3 * 128, 3 * 128 - 1, 32, 32, seed=9, dealt=False, empty_tiles=(0, 1, 2))


@pytest.mark.gpu
def test_chunk_deal_matches_one_cta_per_tile():
    """The dealt layer against the same layer with one CTA per tile (no workspace): equal up to the partial-sum
    order."""
    import torch
    from sassd_b200 import ops
    saved = ops.SPCONV_TAP_SPLIT
    try:
        ops.SPCONV_TAP_SPLIT = False
        outs_tile, ref, counters_tile, host, _ = _run(40 * 128, 40 * 128 - 9, 64, 64, seed=11, absent=0.75,
                                                      full_every=6)
        ops.SPCONV_TAP_SPLIT = True
        outs_deal, _, counters_deal, _, takes = _run(40 * 128, 40 * 128 - 9, 64, 64, seed=11, absent=0.75,
                                                     full_every=6)
        assert takes
    finally:
        ops.SPCONV_TAP_SPLIT = saved
    n = 40 * 128 - 9
    sc = max(ref[:n].abs().max().item(), 1.0)
    d = (outs_tile[0][1][:n] - outs_deal[0][1][:n]).abs().max().item()
    assert d < 2e-5 * sc
    assert counters_tile == counters_deal == list(host)
    assert torch.isfinite(outs_deal[0][1][:n]).all()
