"""The detection tail on head outputs outside the calibrated range.

Seed 0's synthetic weights keep every activation below ~8, so the tail's other tests only see finite, moderate boxes.
A checkpoint early in a training run does not: a box-size regression above ~88 makes expf overflow, a large x / y
regression puts PSWarp's sample points billions of pixels off the map, and a NaN anywhere in the head map reaches
every stage behind it.  Here each kernel of the tail is driven through the C ABI (ops.*) at those values and held to
the plain reference of the same operation (oracle/ref_pipeline.py, oracle/nms.c, the reference NMS kernel when
oracle/_ref/ has it), with torch's CPU fp32 semantics: NaN > thr is false, sigmoid(+-inf) is 1 / 0, exp overflows to
inf, torch.max lets the first NaN win both the value and the index.  Outputs are pre-filled with 0x7F bytes, their
capacities carry a guard band that must stay untouched, and a second call is bit-identical.  The last cases run the
whole step on constructed checkpoints whose guided boxes lie past 2^31 pixels or have infinite sizes.

PSWarp's contract beyond the reference (F.grid_sample is undefined there): a tap off the map adds exactly 0 however
far off it is; a non-finite sample coordinate makes its part, and so the box's score, NaN, and the rescoring
threshold then drops the box.
"""
import ctypes
import functools
import warnings

import numpy as np
import pytest
import torch

from oracle import ref_pipeline as O
from tests.test_detection_tail import (C_PS, EPS32, H, OFF_X, OFF_Y, REF_LIB, SSCALE, W, _ordered, _pswarp_ref64,
                                       _sig64, _ulp, _ulps)

GUIDED_THR, SCORE_THR, IOU_THR = 0.1, 0.3, 0.1
NMS_CAP = 4096
SENT = 0x7F7F7F7F                  # sentinel word of every pre-filled output
GUARD = 16                         # rows of every output past what the kernel may write
F32 = np.float32
FMAX = float(np.finfo(F32).max)
INF, NAN = float("inf"), float("nan")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _filled(shape, dtype, dev):
    """A CUDA tensor every byte of which is 0x7F."""
    t = torch.empty(shape, dtype=dtype, device=dev)
    t.view(torch.uint8).fill_(0x7F)
    return t


def _untouched(t):
    return bool(np.all(t.cpu().contiguous().view(torch.uint8).numpy() == 0x7F))


def _bits(t):
    return t.cpu().contiguous().view(torch.uint8).numpy().tobytes()


def _nan_equal_ordered(a, b):
    """equal as fp32 values, sign of zero included, NaN equal to NaN (any payload)"""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    na, nb = np.isnan(a), np.isnan(b)
    return np.array_equal(na, nb) and np.array_equal(_ordered(np.where(na, 0, a)), _ordered(np.where(nb, 0, b)))


# ====================================================================== 0. the semantics the oracle stands for
def test_torch_cpu_semantics_the_tail_follows():
    """What the reference computes on torch's CPU at these values, and so what the kernels must do."""
    v, i = torch.max(torch.tensor([[0.5, NAN, 0.7, NAN], [NAN, 0.9, NAN, 0.2], [0.2, 0.2, 0.1, 0.1]]), dim=-1)
    assert torch.isnan(v[:2]).all() and i.tolist() == [1, 0, 0]           # the first NaN wins; ties: the first max
    _, i = torch.max(torch.tensor([[NAN, 1.0], [1.0, NAN], [NAN, NAN], [1.0, 1.0]]), dim=-1)
    assert i.tolist() == [0, 1, 0, 0]
    s = torch.sigmoid(torch.tensor([INF, -INF, 1e4, -1e4, 20.0, NAN]))
    assert s[:5].tolist() == [1.0, 0.0, 1.0, 0.0, 1.0] and torch.isnan(s[5])
    assert not bool(torch.tensor(NAN) > SCORE_THR)
    e = torch.exp(torch.tensor([88.72283, 88.7229, 1e4]))
    assert torch.isfinite(e[0]) and torch.isinf(e[1:]).all()


# ====================================================================== 1. polygon bound of the rotated overlap
def _overlap_pairs(n, seed):
    """BEV box pairs [n,5] x 2 that stress the polygon: extents log-uniform from 1e-6 to 1e39 (1e39 is inf in fp32),
    exact zero, inf and NaN; centres near-coincident or a few extents apart; yaws up to 1e6 and exact copies."""
    rs = np.random.RandomState(seed)

    def boxes(ext_scale):
        with np.errstate(over="ignore", invalid="ignore"):
            ext = (10.0 ** rs.uniform(-6, 39, (n, 2))).astype(F32) * ext_scale
            c = rs.normal(0, 1, (n, 2)) * rs.choice([0.0, 1e-4, 1.0, 10.0, 1e6], (n, 1))
            ext[rs.uniform(size=(n, 2)) < 0.03] = 0.0
            ext[rs.uniform(size=(n, 2)) < 0.03] = INF
            ext[rs.uniform(size=(n, 2)) < 0.01] = NAN
            yaw = rs.choice([0.0, np.pi / 2, -np.pi / 2, np.pi, 1e6], n) + rs.normal(0, 1, n) * rs.choice(
                [0.0, 1e-6, 1.0], n)
            lo = (c - ext / 2).astype(F32)
            hi = (c + ext / 2).astype(F32)
        return np.concatenate([lo, hi, yaw[:, None]], 1).astype(F32)

    a, b = boxes(1.0), boxes(rs.choice([1.0, 1.0001, 0.5], (n, 1)))
    same = rs.uniform(size=n) < 0.1
    b[same] = a[same]
    near = rs.uniform(size=n) < 0.2                                  # b = a slightly turned and shifted
    b[near] = a[near]
    b[near, 4] = (a[near, 4] + rs.normal(0, 1e-3, near.sum())).astype(F32)
    return a, b


def test_rotated_overlap_polygon_stays_within_16_points():
    """box_overlap keeps 16 polygon points, as the reference does; no pair here needs more (the most seen is exactly 16)."""
    worst = 0
    for seed in range(4):
        a, b = _overlap_pairs(250000, seed)
        cnt = O.overlap_points(a, b)
        worst = max(worst, int(cnt.max()))
        assert cnt.max() <= 16, "pair %d needs %d polygon points" % (int(cnt.argmax()), int(cnt.max()))
    assert worst >= 8                                                  # the draw reaches past octagons
    print("rotated overlap: at most %d polygon points" % worst)


# ====================================================================== 2. PSWarp (sassd_pswarp)
def _kernel_pixel(x32, n):
    """The kernel's pixel coordinate from a sample position in pixels: normalise by n - 1, then grid_sample's
    align_corners un-normalisation, each step one correctly rounded fp32 operation."""
    with np.errstate(over="ignore", invalid="ignore"):
        x = np.asarray(x32, F32)
        g = (x / F32(n - 1)) * F32(2) - F32(1)
        return ((g + F32(1)) / F32(2)) * F32(n - 1)


def _f32_at(o):
    """the fp32 value at ordered index o (inverse of _ordered)"""
    i = np.int64(o)
    return np.array([i if i >= 0 else (-i) | -0x80000000], np.int64).astype(np.int32).view(F32)[0]


def _reach(target, n, side):
    """An fp32 sample position whose kernel pixel coordinate is ``target`` (side 0), or the nearest one the kernel's
    normalisation can produce below it (side -1) or above it (side +1); non-finite targets are their own position.
    The pixel coordinate is a non-decreasing function of the position, so a bisection over the fp32 values finds
    it; returns (position, pixel)."""
    t = F32(target)
    if not np.isfinite(t):
        return t, t
    lo, hi = int(_ordered(F32(-FMAX))[()]), int(_ordered(F32(FMAX))[()])
    strict = side > 0
    while lo < hi:                                   # the first position whose pixel is >= t (> t when strict)
        mid = (lo + hi) // 2
        v = _kernel_pixel(_f32_at(mid), n)
        if (v > t) if strict else (v >= t):
            hi = mid
        else:
            lo = mid + 1
    x = _f32_at(lo - 1 if side < 0 else lo)
    return x, _kernel_pixel(x, n)


def _edge_targets(n):
    """(pixel, side): just below, at and just above -1, 0, n-1 and 2^31 (where a cast to int saturates), 1e30, just
    below FLT_MAX, +-inf and NaN.  The normalisation's rounding leaves gaps between the pixels it can produce (about
    1e-5 near -1, 256 near 2^31), so "just below / above" is the nearest pixel it produces on that side and "at" is
    the first one at or above."""
    return [(-1.0, -1), (-1.0, 0), (0.0, -1), (0.0, 0), (n - 1.0, -1), (n - 1.0, 0), (n - 1.0, 1), (2.0 ** 31, -1),
            (2.0 ** 31, 0), (1e30, 0), (FMAX, -1), (INF, 0), (-INF, 0), (NAN, 0)]


def _pswarp_call(dev, feat, boxes, d_k, off_x, off_y, sscale):
    """sassd_pswarp on a pre-filled score buffer with a guard band; returns the scores [B, k_cap] and checks that
    rows past d_k are untouched and that a second call is bit-identical."""
    from sassd_b200 import ops
    B, Hf, Wf, C = feat.shape
    k_cap = boxes.shape[1]
    f, bx = torch.from_numpy(feat).to(dev), torch.from_numpy(boxes).to(dev)
    dk = torch.tensor(d_k, dtype=torch.int32, device=dev)
    outs = []
    for _ in range(2):
        s = _filled((B, k_cap), torch.float32, dev)
        ops._call("sassd_pswarp", None, ops._ptr(f), C, B, Hf, Wf, ops._ptr(bx), ops._ptr(dk), k_cap,
                  ctypes.c_float(off_x), ctypes.c_float(off_y), ctypes.c_float(sscale), ops._ptr(s), ops._stream())
        torch.cuda.synchronize()
        for b in range(B):
            assert _untouched(s[b, d_k[b]:]), "frame %d: rows past d_k written" % b
        outs.append(s)
    assert _bits(outs[0]) == _bits(outs[1]), "second call differs"
    return outs[0].cpu().numpy()


def _expected_scores(feat_hwc, ix, iy):
    """fp64 score [N] and S [N] (tests/test_detection_tail.py's restatement) at the kernel's pixel positions [28,N]:
    NaN where any part's position is non-finite."""
    fin = np.isfinite(ix) & np.isfinite(iy)
    with np.errstate(invalid="ignore", over="ignore"):
        ref, S = _pswarp_ref64(feat_hwc.astype(np.float64), np.where(fin, ix, -1e9), np.where(fin, iy, -1e9))
    bad = ~fin.all(0)
    return np.where(bad, np.nan, ref), np.where(bad, 0.0, S), bad


@pytest.mark.gpu
def test_pswarp_sample_points_at_every_range_edge(dev):
    """Zero-size boxes (all 28 parts on one point; spatial scale 1, offsets 0, so the position is the box centre)
    at x / y = -1 - ulp, -1, -ulp, 0, n-1 - ulp, n-1, n-1 + ulp, 2^31 - 128, 2^31, 1e30, FLT_MAX, +-inf and NaN in the
    kernel's pixel coordinate, each axis alone (the other at a pixel centre or in between) and every combination:
    finite points within the fp64 bound, taps off the map exactly 0, a non-finite coordinate NaN."""
    rs = np.random.RandomState(11)
    feat = rs.normal(0, 1, (1, H, W, 28)).astype(F32)
    ex = [_reach(t, W, side) for t, side in _edge_targets(W)]
    ey = [_reach(t, H, side) for t, side in _edge_targets(H)]
    # the construction reaches what it claims to: on the stated side of each target and within 2e-5 + 2e-7 |t| of it
    for (t, side), (_, v) in zip(_edge_targets(W) + _edge_targets(H), ex + ey):
        if np.isfinite(t):
            d = float(v) - t
            assert (d < 0 if side < 0 else d > 0 if side > 0 else d >= 0) and abs(d) <= 2e-5 + 2e-7 * abs(t), (t, side, d)
    assert float(ex[3][1]) == 0.0 and float(ex[5][1]) == W - 1 and float(ey[5][1]) == H - 1
    cx, cy = [_reach(88.0, W, 0), _reach(13.5, W, 0)], [_reach(100.0, H, 0), _reach(57.25, H, 0)]
    pts = [(x, y) for x in ex for y in cy] + [(x, y) for x in cx for y in ey] + [(x, y) for x in ex for y in ey]
    px, py = np.array([p[0][0] for p in pts], F32), np.array([p[1][0] for p in pts], F32)
    n = len(pts)
    boxes = np.full((1, n + GUARD, 7), np.nan, F32)             # rows past d_k are NaN: never read
    boxes[0, :n] = np.stack([px, py, np.full(n, -1.0), np.zeros(n), np.zeros(n), np.full(n, 1.5), np.zeros(n)], 1)
    got = _pswarp_call(dev, feat, boxes, [n], 0.0, 0.0, 1.0)[0, :n].astype(np.float64)
    ix = np.repeat(np.array([p[0][1] for p in pts], F32)[None], 28, 0)
    iy = np.repeat(np.array([p[1][1] for p in pts], F32)[None], 28, 0)
    assert np.array_equal(ix, _kernel_pixel(boxes[0, :n, 0], W)[None].repeat(28, 0), equal_nan=True)
    exp, S, bad = _expected_scores(feat[0], ix, iy)
    assert np.array_equal(np.isnan(got), bad), "NaN exactly where a coordinate is non-finite: %s" % (
        [(float(ix[0, i]), float(iy[0, i])) for i in np.nonzero(np.isnan(got) != bad)[0][:8]])
    ok = ~bad
    off = ok & (S == 0)
    assert np.all(got[off] == 0.0), "off the map: exactly 0"
    assert off.sum() >= 100 and (ok & (S > 0)).sum() >= 30
    tol = C_PS * EPS32 * S
    err = np.abs(got - exp)
    i = int(np.nonzero(ok)[0][err[ok].argmax()])
    assert np.all(err[ok] <= tol[ok]), "worst %g at (%r, %r)" % (err[i], float(ix[0, i]), float(iy[0, i]))


def _far_boxes():
    """[N,7] metre boxes that reach the range edges the way a decoded box does: huge and infinite w / l, huge x / y,
    yaw 0, +-pi/2 and 1e6, beside ordinary boxes.  A part is either far off the map (a huge extent times its window
    coordinate, or a huge centre) or where the fp32 rotation is as accurate as for a moderate box (a long box's
    middle column, ordinary boxes), so the fp64 bound applies to every part on the map."""
    rows = []
    for r in (0.0, np.pi / 2, -np.pi / 2, 1e6):
        for w, l in ((1e5, 2.0), (2.0, 1e5), (1e30, 2.0), (2.0, 1e30), (FMAX, 2.0), (INF, 2.0), (2.0, INF),
                     (INF, INF), (3e38, 3e38)):
            rows.append([30.0, 0.0, -1.0, w, l, 1.5, r])
        for x, y in ((8.6e8, 0.0), (30.0, 8.6e8), (-8.6e8, 0.0), (1e30, 1e30), (FMAX, 0.0), (INF, 0.0), (0.0, -INF),
                     (NAN, 0.0), (20.0, NAN)):
            rows.append([x, y, -1.0, 1.6, 3.9, 1.5, r])
        rows.append([35.0, 2.0, -1.0, 1.6, 3.9, 1.5, r])                 # ordinary
        rows.append([69.0, 39.0, -1.0, 4.0, 9.0, 1.5, r])                # over the far corner
    rows.append([30.0, 0.0, -1.0, 1.6, 3.9, 1.5, NAN])
    rows.append([30.0, 0.0, -1.0, 1.6, 3.9, 1.5, INF])
    return np.asarray(rows, F32)


@pytest.mark.gpu
def test_pswarp_boxes_far_off_and_non_finite(dev):
    """Decoded-box-shaped inputs at the KITTI grid offsets and scale, two frames (the second holding the first's
    boxes reversed) over one grid-stride pass: the score is NaN iff some part has a non-finite position, exactly 0
    when every part is off the map, and within the fp64 bound otherwise."""
    rs = np.random.RandomState(12)
    feat = rs.normal(0, 1, (2, H, W, 28)).astype(F32)
    b7 = _far_boxes()
    n = len(b7)
    boxes = np.full((2, n + GUARD, 7), np.inf, F32)
    boxes[0, :n], boxes[1, :n] = b7, b7[::-1]
    got = _pswarp_call(dev, feat, boxes, [n, n], OFF_X, OFF_Y, SSCALE)
    for b in range(2):
        bx = boxes[b, :n]
        with np.errstate(over="ignore", invalid="ignore"):
            xs, ys = O.gen_sample_grid(torch.from_numpy(bx[:, [0, 1, 3, 4, 6]]), grid_offsets=(OFF_X, OFF_Y),
                                       spatial_scale=SSCALE)
        ix, iy = _kernel_pixel(xs.numpy(), W), _kernel_pixel(ys.numpy(), H)
        exp, S, bad = _expected_scores(feat[b], ix, iy)
        g = got[b, :n].astype(np.float64)
        assert np.array_equal(np.isnan(g), bad), "frame %d: NaN rows %s, expected %s" % (
            b, np.nonzero(np.isnan(g))[0], np.nonzero(bad)[0])
        ok = ~bad
        with np.errstate(invalid="ignore"):
            far = ok & np.all((ix < -2) | (ix > W + 1) | (iy < -2) | (iy > H + 1), 0)
        assert np.all(g[far] == 0.0) and far.sum() >= 25 and bad.sum() >= 40 and (ok & (S > 0)).sum() >= 12
        # the rest, wholly or partly on the map: parts off it add exactly 0, the others are held to the bound
        assert np.all(np.abs(g[ok] - exp[ok]) <= C_PS * EPS32 * S[ok]), "frame %d: boxes on the map" % b


# ====================================================================== 3. guided anchors (sassd_decode_select)
@functools.lru_cache(maxsize=None)
def _exp_edge(a):
    """(largest fp32 e with torch's exp(e) * a finite, the next fp32 above it) for anchor size a: the product's
    overflow for a > 1, exp's own for a < 1"""
    a = torch.tensor(a, dtype=torch.float32)
    e = torch.tensor(float(np.log(FMAX / max(float(a), 1.0))), dtype=torch.float32)
    while torch.isinf(torch.exp(e) * a):
        e = torch.nextafter(e, torch.tensor(-INF))
    while torch.isfinite(torch.exp(torch.nextafter(e, torch.tensor(INF))) * a):
        e = torch.nextafter(e, torch.tensor(INF))
    return float(e), float(torch.nextafter(e, torch.tensor(INF)))


def _nonfinite_decode_case(seed):
    """B = 2, 3 classes on the real 200x176 grid: per frame 600 anchors given class logits NaN / +-inf / +-1e4 /
    ties at sigmoid 1 (one class NaN beside a passing class, the case the reference drops), regressions at the expf
    overflow edge and NaN, NaN direction logits; every other anchor stays below the threshold."""
    rs = np.random.RandomState(seed)
    B, ncls = 2, 3
    Na = ncls * H * W * 2
    codes = rs.normal(0, 0.5, (B, Na, 7)).astype(F32)
    cls = rs.uniform(-9, -2.5, (B, Na, ncls)).astype(F32)
    dirl = rs.normal(0, 1, (B, Na, 2)).astype(F32)
    mask = (rs.uniform(size=(B, Na)) > 0.1).astype(np.uint8)
    anchors = np.stack([rs.uniform(0, 70, Na), rs.uniform(-40, 40, Na), rs.uniform(-2, -1, Na),
                        rs.choice([0.6, 1.6, 1.76], Na), rs.choice([0.8, 3.9, 0.6], Na), rs.uniform(1.4, 1.8, Na),
                        rs.choice([0.0, 1.57], Na)], -1).astype(F32)
    logit_pool = np.array([NAN, INF, -INF, 1e4, -1e4, 20.0, 30.0, 2.0, -1.0], F32)
    for b in range(B):
        sel = np.sort(rs.choice(Na, 600, replace=False))
        mask[b, sel] = 1
        cls[b, sel] = rs.choice(logit_pool, (600, ncls))
        cls[b, sel[:60], 0] = 3.0                                        # a passing class beside a NaN one
        cls[b, sel[:60], 1] = NAN
        cls[b, sel[60:90]] = [30.0, 20.0, INF]                           # tied at sigmoid 1: class 0
        for j, a in enumerate(sel[90:330]):                              # w / l / h at the overflow edge
            c = 3 + j % 3
            lo, hi = _exp_edge(float(anchors[a, c]))
            codes[b, a, c] = (lo, hi, np.nextafter(F32(lo), F32(-INF)), 1e4, -1e4, INF)[(j // 3) % 6]
            cls[b, a] = [2.0, -1.0, -1.0]
        nanreg = sel[330:400]
        codes[b, nanreg, rs.randint(0, 7, nanreg.size)] = NAN            # NaN regression, finite passing logits
        cls[b, nanreg] = [-1.0, 2.0, -1.0]
        nd = sel[400:480]
        dirl[b, nd] = np.array([[NAN, 1.0], [1.0, NAN], [NAN, NAN], [-INF, INF]], F32)[np.arange(nd.size) % 4]
        cls[b, nd] = [2.0, 2.0, -1.0]
    head = np.concatenate([
        codes.reshape(B, ncls, H, W, 14).transpose(0, 2, 3, 1, 4).reshape(B, H, W, ncls * 14),
        cls.reshape(B, ncls, H, W, 2 * ncls).transpose(0, 2, 3, 1, 4).reshape(B, H, W, 2 * ncls * ncls),
        dirl.reshape(B, ncls, H, W, 4).transpose(0, 2, 3, 1, 4).reshape(B, H, W, ncls * 4)], -1)
    return dict(head=np.ascontiguousarray(head), codes=codes, cls=cls, dirl=dirl, mask=mask, anchors=anchors, ncls=ncls)


@pytest.mark.gpu
def test_decode_select_on_non_finite_head_outputs(dev):
    """sassd_decode_select vs get_guided_anchors (torch CPU fp32): selection (a NaN class score wins the max and is
    never selected), labels, anchor order and d_k exactly; NaN regressions give a NaN component under the anchor's
    label; NaN direction logits pick the reference's direction; w / l / h within 4 ulp with inf one ulp past FLT_MAX;
    z within the bound of test_detection_tail or equal where h is not finite."""
    from sassd_b200 import ops
    case = _nonfinite_decode_case(21)
    B, ncls = 2, case["ncls"]
    Na = ncls * H * W * 2
    with np.errstate(invalid="ignore"):
        s64 = _sig64(case["cls"])
    fin = np.isfinite(s64)
    assert np.all(np.abs(s64[fin] - GUIDED_THR) >= 1e-6)
    g, lab, idx, _ = O.get_guided_anchors(torch.from_numpy(case["codes"]), torch.from_numpy(case["cls"]),
                                          torch.from_numpy(case["dirl"]), torch.from_numpy(case["anchors"]),
                                          torch.from_numpy(case["mask"]).bool(), ncls, GUIDED_THR, return_index=True)
    counts = [len(i) for i in idx]
    k_cap = max(counts) + GUARD
    head = torch.from_numpy(case["head"]).to(dev)
    an, mk = torch.from_numpy(case["anchors"]).to(dev), torch.from_numpy(case["mask"]).to(dev)
    ws = torch.empty((ops._L().sassd_decode_select_workspace_bytes(B, Na),), dtype=torch.uint8, device=dev)
    runs = []
    for _ in range(2):
        boxes, labels = _filled((B, k_cap, 7), torch.float32, dev), _filled((B, k_cap), torch.int32, dev)
        index, d_k = _filled((B, k_cap), torch.int32, dev), _filled((B,), torch.int32, dev)
        status = torch.zeros((1,), dtype=torch.int32, device=dev)
        ops._call("sassd_decode_select", None, ops._ptr(head), head.shape[-1], B, H, W, ncls, ops._ptr(an), 0,
                  ops._ptr(mk), Na, ctypes.c_float(GUIDED_THR), ops._ptr(boxes), ops._ptr(labels), ops._ptr(index),
                  ops._ptr(d_k), k_cap, ops._ptr(status), ops._ptr(ws), ws.numel(), ops._stream())
        torch.cuda.synchronize()
        assert int(status.item()) == 0
        runs.append((boxes, labels, index, d_k))
    assert all(_bits(x) == _bits(y) for x, y in zip(*runs)), "second call differs"
    boxes, labels, index, d_k = runs[0]
    for b in range(B):
        k = counts[b]
        assert int(d_k[b]) == k
        for t in (boxes, labels, index):
            assert _untouched(t[b, k:]), "frame %d: rows past d_k written" % b
    boxes, labels, index = boxes.cpu().numpy(), labels.cpu().numpy(), index.cpu().numpy()
    nan_cls, edge, nanreg, nandir = 0, 0, 0, 0
    for b in range(B):
        k, ei = counts[b], idx[b].numpy()
        sel = np.nonzero(case["mask"][b])[0]
        nan_cls += int(np.isnan(case["cls"][b, sel]).any(-1).sum())
        assert np.array_equal(index[b, :k], ei), "frame %d: anchor index list" % b
        assert np.array_equal(labels[b, :k], lab[b].numpy()), "frame %d: labels" % b
        got, exp = boxes[b, :k], g[b].numpy()
        a_sel, c_sel = case["anchors"][ei], case["codes"][b, ei]
        with np.errstate(over="ignore", invalid="ignore"):
            diag = np.sqrt(a_sel[:, 4] * a_sel[:, 4] + a_sel[:, 3] * a_sel[:, 3])
            for j in (0, 1):                                       # x, y: correctly rounded fp32, exact
                assert _nan_equal_ordered(got[:, j], c_sel[:, j] * diag + a_sel[:, j]), "frame %d: x, y" % b
        assert _nan_equal_ordered(got[:, 6], exp[:, 6]), "frame %d: yaw" % b
        assert np.array_equal(np.isnan(got[:, 2:6]), np.isnan(exp[:, 2:6])), "frame %d: NaN components" % b
        whl = ~np.isnan(exp[:, 3:6])
        assert _ulps(np.where(whl, got[:, 3:6], 0), np.where(whl, exp[:, 3:6], 0)).max(initial=0) <= 4, \
            "frame %d: w / l / h" % b
        hz = np.isfinite(exp[:, 5]) & np.isfinite(got[:, 5]) & np.isfinite(exp[:, 2])
        dz = np.abs(got[hz, 2].astype(np.float64) - exp[hz, 2])
        assert np.all(dz <= 4 * _ulp(exp[hz, 5] / 2) + _ulp(exp[hz, 2])), "frame %d: z" % b
        same_h = ~hz & (np.isinf(exp[:, 5]) == np.isinf(got[:, 5]))
        assert _nan_equal_ordered(got[same_h, 2], exp[same_h, 2]), "frame %d: z with an infinite h" % b
        edge += int(np.isinf(exp[:, 3:6]).sum())
        nanreg += int(np.isnan(got[:, :6]).any(1).sum())
        dl = case["dirl"][b, ei]
        nandir += int(np.isnan(dl).any(1).sum())
    assert nan_cls >= 200 and edge >= 100 and nanreg >= 100 and nandir >= 100, (nan_cls, edge, nanreg, nandir)


# ====================================================================== 4. rescoring + NMS (sassd_rescore_nms)
def _nonfinite_frame(seed, odd_boxes):
    """Candidates: ordinary car boxes in 9 m cells (some overlapping pairs), with ``odd_boxes`` also boxes with NaN /
    inf / zero / 1e30 extents and NaN / inf centres (each twice); scores NaN / +-inf / +-1e4 / finite, many +inf and
    1e4 logits tied at 1.0."""
    rs = np.random.RandomState(seed)
    rows = []
    for i in range(120):
        cx, cy = 4.5 + 9.0 * (i % 12), -50.0 + 9.0 * (i // 12)
        b = [cx, cy, -1.6, 1.6 + rs.normal(0, 0.05), 3.9 + rs.normal(0, 0.1), 1.56, rs.uniform(-np.pi, np.pi)]
        rows.append(b)
        if i % 3 == 0:                                                    # an overlapping neighbour
            rows.append([cx + rs.uniform(-0.3, 0.3), cy + rs.uniform(-0.3, 0.3)] + b[2:6] + [b[6] + rs.uniform(-.2, .2)])
    odd = []
    for w, l in ((NAN, 3.9), (1.6, NAN), (INF, 3.9), (1.6, INF), (0.0, 3.9), (0.0, 0.0), (1e30, 3.9), (1e30, 1e30),
                 (FMAX, FMAX)):
        for r in (0.0, np.pi / 2, 1e6):
            odd.append([20.0 + rs.uniform(-1, 1), rs.uniform(-5, 5), -1.6, w, l, 1.56, r])
    for x, y in ((NAN, 0.0), (INF, 0.0), (0.0, -INF), (1e30, 0.0)):
        odd.append([x, y, -1.6, 1.6, 3.9, 1.56, 0.3])
    odd.append([20.0, 0.0, -1.6, 1.6, 3.9, 1.56, NAN])
    if odd_boxes:
        rows += odd + odd                                               # duplicates of every odd box
    bx = np.asarray(rows, F32)
    n = len(bx)
    lg = rs.choice(np.array([NAN, INF, -INF, 1e4, -1e4], F32), n)
    fin = rs.uniform(size=n) < 0.5
    lg[fin] = (-0.8 + 1e-3 * rs.permutation(4000)[:fin.sum()]).astype(F32)   # distinct finite logits
    lb = rs.randint(0, 3, n).astype(np.int32)
    perm = rs.permutation(n)
    return bx[perm], lg[perm], lb[perm]


def _rescore_call(dev, frames, det_cap):
    from sassd_b200 import ops
    B = len(frames)
    k_cap = max(len(f[0]) for f in frames) + GUARD
    boxes = np.full((B, k_cap, 7), np.nan, F32)
    scores = np.full((B, k_cap), np.inf, F32)                            # past d_k: would pass if read
    labels = np.zeros((B, k_cap), np.int32)
    for b, (bx, lg, lb) in enumerate(frames):
        boxes[b, :len(bx)], scores[b, :len(bx)], labels[b, :len(bx)] = bx, lg, lb
    d_k = torch.tensor([len(f[0]) for f in frames], dtype=torch.int32, device=dev)
    bx_d, sc_d, lb_d = (torch.from_numpy(x).to(dev) for x in (boxes, scores, labels))
    ws = torch.empty((ops._L().sassd_rescore_nms_workspace_bytes(B, k_cap, NMS_CAP),), dtype=torch.uint8, device=dev)
    runs = []
    for _ in range(2):
        det, nd = _filled((B, det_cap, 9), torch.float32, dev), _filled((B,), torch.int32, dev)
        status = torch.zeros((1,), dtype=torch.int32, device=dev)
        ops._call("sassd_rescore_nms", None, ops._ptr(bx_d), ops._ptr(sc_d), ops._ptr(lb_d), ops._ptr(d_k), B, k_cap,
                  ctypes.c_float(SCORE_THR), ctypes.c_float(IOU_THR), NMS_CAP, ops._ptr(det), ops._ptr(nd), det_cap,
                  ops._ptr(status), ops._ptr(ws), ws.numel(), ops._stream())
        torch.cuda.synchronize()
        assert int(status.item()) == 0
        for b in range(B):
            assert _untouched(det[b, int(nd[b]):]), "frame %d: rows past ndet written" % b
        runs.append((det, nd))
    assert _bits(runs[0][0]) == _bits(runs[1][0]) and _bits(runs[0][1]) == _bits(runs[1][1])
    return runs[0][0].cpu().numpy(), runs[0][1].cpu().numpy()


def _pairs_within_polygon_bound(bev):
    n = len(bev)
    i, j = np.triu_indices(n, 1)
    cnt = O.overlap_points(bev[i], bev[j])
    assert cnt.max(initial=0) <= 16, "a pair needs %d polygon points" % cnt.max()
    return i, j


def _plain(bev):
    """BEV boxes whose corners are finite and moderate: on pairs of these the fp32 IoU has no overflow, so the CPU
    restatement (no FMA contraction) decides the threshold as the CUDA kernels do"""
    return np.all(np.isfinite(bev) & (np.abs(bev) < 1e6), 1)


def _mask_bits(mask, n):
    return np.unpackbits(np.ascontiguousarray(mask).view(np.uint8), axis=1, bitorder="little")[:, :n].astype(bool)


def _sweep(mask, n):
    """the reference's greedy sweep over a bitmask: kept indices into the sorted list"""
    remv = np.zeros(mask.shape[1], np.uint64)
    keep = []
    for i in range(n):
        if not (int(remv[i // 64]) >> (i % 64)) & 1:
            keep.append(i)
            remv[i // 64:] |= mask[i, i // 64:]
    return np.asarray(keep, np.int64)


@pytest.mark.gpu
def test_rescore_nms_on_non_finite_scores_and_boxes(dev):
    """sassd_rescore_nms at B = 2: NaN scores never pass, +inf and 1e4 logits tie at 1.0 and keep candidate order.
    Frame 1 (ordinary boxes) equals get_rescore_bboxes bit for bit.  Frame 0 adds boxes with NaN / inf / zero / 1e30
    extents and non-finite centres: its NMS bitmask equals the reference nmsLauncher's bit for bit (when oracle/_ref/
    has it, with a warning when it has not) and oracle/nms.c's on every pair of plain boxes, and the fused path
    keeps what the reference sweep over that bitmask keeps, in order, bit for bit.  Every pair fed to the kernels stays within 16 polygon points."""
    import os
    from sassd_b200 import ops
    frames = [_nonfinite_frame(31, True), _nonfinite_frame(32, False)]
    det, nd = _rescore_call(dev, frames, 1024)
    tied = 0
    for b, (bx, lg, lb) in enumerate(frames):
        s = torch.sigmoid(torch.from_numpy(lg))
        p = torch.nonzero(s > SCORE_THR).view(-1)
        order = torch.sort(s[p], descending=True, stable=True)[1]
        src = p[order].numpy()                                           # candidate of each sorted passer
        bev = O.boxes3d_to_bev(torch.from_numpy(bx[src])).numpy()
        _pairs_within_polygon_bound(bev)
        n = len(bev)
        tied += int((s[p] == 1.0).sum())
        with np.errstate(invalid="ignore"):
            iou = O.iou_matrix(bev)
        pl = _plain(bev)
        pp = pl[:, None] & pl[None, :] & ~np.eye(n, dtype=bool)
        assert np.abs(iou[pp] - IOU_THR).min() > 1e-5, "frame %d is not decisive" % b
        got = ops.nms_mask(torch.from_numpy(np.ascontiguousarray(bev)).to(dev), IOU_THR).cpu().numpy().view(np.uint64)
        upper = np.triu(np.ones((n, n), bool), 1)
        gb, wb = _mask_bits(got, n), _mask_bits(O.nms_mask(bev, IOU_THR), n)
        diff = np.nonzero(upper & pp & (gb != wb))
        assert diff[0].size == 0, "frame %d: %d plain pairs differ from nms.c, first %s %s" % (
            b, diff[0].size, bev[diff[0][0]], bev[diff[1][0]])
        odd = upper & ~pp & (gb != wb)
        print("frame %d: %d passers (%d not plain), %d tied at 1.0; %d pairs with a non-plain box decided otherwise "
              "by nms.c (no FMA contraction)" % (b, n, int((~pl).sum()), int((s[p] == 1.0).sum()), int(odd.sum())))
        if os.path.isfile(REF_LIB):
            fn = getattr(ctypes.CDLL(REF_LIB), "_Z11nmsLauncherPKfPyif")
            fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_float]
            fn.restype = None
            d_bev = torch.from_numpy(np.ascontiguousarray(bev)).to(dev)
            rmask = torch.zeros((n, (n + 63) // 64), dtype=torch.int64, device=dev)
            torch.cuda.synchronize()
            fn(ctypes.c_void_p(d_bev.data_ptr()), ctypes.c_void_p(rmask.data_ptr()), n, ctypes.c_float(IOU_THR))
            torch.cuda.synchronize()
            rb = _mask_bits(rmask.cpu().numpy().view(np.uint64), n)
            diff = np.nonzero(upper & (gb != rb))
            assert diff[0].size == 0, "frame %d: %d pairs differ from nmsLauncher, first %s %s" % (
                b, diff[0].size, bev[diff[0][0]], bev[diff[1][0]])
        elif not pl.all():
            warnings.warn("oracle/_ref/libiou3d_ref.so is absent: frame %d's %d pairs with a non-plain box are held "
                          "only to the kernel's own bitmask" % (b, int((upper & ~pp).sum())))
        keep = _sweep(got, n)
        assert nd[b] == len(keep), (b, nd[b], len(keep))
        assert _nan_equal_ordered(det[b, :nd[b], :7], bx[src[keep]]), "frame %d: kept boxes / order" % b
        assert np.array_equal(det[b, :nd[b], 8], lb[src[keep]].astype(F32))
        assert np.abs(det[b, :nd[b], 7] - s[p][order][keep].numpy()).max() <= 1e-6      # CUDA expf vs torch
        if b == 0:
            assert np.isnan(det[b, :nd[b], :7]).any() and np.isinf(det[b, :nd[b], :7]).any()   # odd boxes are kept
        else:
            eb, es, el = (x[0] for x in O.get_rescore_bboxes([torch.from_numpy(bx)], [torch.from_numpy(lg)],
                                                              [torch.from_numpy(lb).long()], SCORE_THR, IOU_THR))
            assert nd[b] == len(eb) and np.array_equal(det[b, :nd[b], :7], eb), "frame %d vs get_rescore_bboxes" % b
            assert np.array_equal(det[b, :nd[b], 8].astype(np.int64), el)
    assert tied >= 40


# ====================================================================== 5. PSWarp targets (sassd_assign_pswarp)
def _assign_case():
    """B = 2 frames of axis-aligned GT cars.  Guided boxes near every GT (IoU from ~0.3 to 1), and boxes that a
    weight-derived decode gives: NaN in each of x, y, z, w, l, h, yaw, infinite w / l / h (expf overflow), zero w,
    x at 4.2e9 m.  Frame 0 holds NaN boxes: a NaN in z, w, l or h makes the box's IoU row NaN (a NaN centre or yaw
    only empties the BEV polygon: IoU 0), so every GT's maximum is NaN and no GT forces a box (GT 4's best box, at IoU
    ~0.68, stays 0); frame 1 has no NaN box and GT 4 forces its best box."""
    rs = np.random.RandomState(41)
    gts, boxes = [], []
    for b in range(2):
        g = np.array([[10.0 + 9 * j, -6.0 + 4 * j, -1.7, 1.6, 3.9, 1.56, 0.0] for j in range(5)], F32)
        rows = []
        for j, gj in enumerate(g):
            # IoU ~1 .. ~0.3; GT 4's best box is at ~0.68, below the 0.7 threshold, so only forcing makes it positive
            for sh in ((0.0, 0.05, 0.3, 0.8, 1.6) if j < 4 else (0.3, 0.8)):
                rows.append(gj + np.array([sh, rs.uniform(-0.02, 0.02), 0, 0, 0, 0, 0], F32))
        base = g[1] + np.array([0.1, 0, 0, 0, 0, 0, 0], F32)
        odd = []
        for c, v in ((3, INF), (4, INF), (5, INF), (3, 0.0), (0, 4.2e9)) + (
                ((0, NAN), (1, NAN), (2, NAN), (3, NAN), (4, NAN), (5, NAN), (6, NAN)) if b == 0 else ()):
            r = base.copy()
            r[c] = v
            odd.append(r)
        bx = np.concatenate([np.asarray(rows, F32), np.asarray(odd, F32)])
        gts.append(g)
        boxes.append(bx[rs.permutation(len(bx))])
    return gts, boxes


@pytest.mark.gpu
def test_assign_pswarp_on_non_finite_guided_boxes(dev):
    """sassd_assign_pswarp vs create_target with RotateIou3dSimilarity (oracle/targets.py, numpy fp32, where
    minimum / maximum / argmax let a NaN through as the reference's torch calls do): labels exactly, NaN IoUs where
    the oracle's are NaN and the others within 1e-5, npos; slots past d_k -1 with IoU 0 over pre-filled outputs; a
    second call bit-identical."""
    from oracle import targets as OT
    from sassd_b200 import ops
    gts, boxes = _assign_case()
    B, gt_cap = 2, 5 + 2
    ks = np.array([len(x) for x in boxes], np.int32)
    n = int(ks.max()) + GUARD
    bx = np.full((B, n, 7), np.nan, F32)
    gt = np.full((B, gt_cap, 7), np.nan, F32)
    for b in range(B):
        bx[b, :ks[b]] = boxes[b]
        gt[b, :len(gts[b])] = gts[b]
    d_gt, d_bx = torch.from_numpy(gt).to(dev), torch.from_numpy(bx).to(dev)
    dn = torch.tensor([len(g) for g in gts], dtype=torch.int32, device=dev)
    dk = torch.from_numpy(ks).to(dev)
    ws = torch.empty((ops._L().sassd_loss_workspace_bytes(B, gt_cap),), dtype=torch.uint8, device=dev)
    runs = []
    for _ in range(2):
        labels, ious, npos = _filled((B, n), torch.int32, dev), _filled((B, n), torch.float32, dev), \
            _filled((B,), torch.int32, dev)
        status = torch.zeros((1,), dtype=torch.int32, device=dev)
        ops._call("sassd_assign_pswarp", None, ops._ptr(d_gt), ops._ptr(dn), B, gt_cap, ops._ptr(d_bx), n,
                  ops._ptr(None), 0, ops._ptr(dk), ctypes.c_float(0.7), ctypes.c_float(0.7), ops._ptr(labels),
                  ops._ptr(ious), ops._ptr(npos), ops._ptr(status), ops._ptr(ws), ws.numel(), ops._stream())
        torch.cuda.synchronize()
        assert int(status.item()) == 0
        runs.append((labels, ious, npos))
    assert all(_bits(x) == _bits(y) for x, y in zip(*runs)), "second call differs"
    lab, iou, npos = (t.cpu().numpy() for t in runs[0])
    ignored = 0
    for b in range(B):
        k = ks[b]
        assert np.all(lab[b, k:] == -1) and np.all(iou[b, k:].view(np.int32) == 0), "frame %d: slots past d_k" % b
        with np.errstate(invalid="ignore", over="ignore"):
            lb, _, mb = OT.create_target(boxes[b], None, gts[b], None, OT.iou3d, 0.7, 0.7, encode=False)
        assert np.array_equal(lab[b, :k], lb), "frame %d: labels %s vs %s" % (b, lab[b, :k], lb)
        nan = np.isnan(mb)
        assert np.array_equal(np.isnan(iou[b, :k]), nan), "frame %d: NaN IoUs" % b
        # finite IoUs within 1e-5: box_overlap's corners are contracted on the GPU and rounded op by op in the
        # oracle's C, which moves a corner by up to ~2 ulp of its coordinate (ulp(46 m) = 3.8e-6 m) and the IoU of a
        # 1.6 m x 3.9 m box by up to ~2 * 3.8e-6 / 1.6 = 5e-6 (measured on an H100: 2.2e-6); every label is decided at
        # least 1e-3 from the 0.7 threshold
        assert np.abs(mb[~nan] - 0.7).min() > 1e-3
        assert np.abs(iou[b, :k][~nan] - mb[~nan]).max() <= 1e-5, "frame %d: IoUs" % b
        assert npos[b] == (lb > 0).sum()
        ignored += int((lb[nan] == -1).sum())
        below = (mb > 0.6) & (mb < 0.7)
        if b == 0:
            assert nan.sum() == 4 and not np.any(lb[~nan] == -1)          # NaN boxes ignored
            assert np.all(lb[below] == 0)                                   # and no GT forces
        else:
            assert not nan.any() and np.any(lb[below] == 1)                 # GT 4 forces its best box
    assert ignored == 4


# ====================================================================== 6. KITTI formatting (sassd_kitti_format)
def _same_rows(dev_a, host_a, what):
    """the fields of one frame's annotations, kept identically: NaN and inf where the host has them, finite values
    within tests/test_kitti_format.py's bounds"""
    from tests.test_kitti_format import ALPHA_TOL, BBOX_TOL
    assert len(dev_a["name"]) == len(host_a["name"]) and set(dev_a) == set(host_a), what
    for k in ("name", "truncated", "occluded", "image_idx", "score", "dimensions"):
        assert np.array_equal(dev_a[k], host_a[k], equal_nan=k in ("score", "dimensions")), (what, k)
    for k, tol in (("location", None), ("rotation_y", None), ("alpha", ALPHA_TOL), ("bbox", BBOX_TOL)):
        d, h = np.asarray(dev_a[k], np.float64), np.asarray(host_a[k], np.float64)
        assert dev_a[k].dtype == host_a[k].dtype, (what, k)
        fin = np.isfinite(h)
        assert np.array_equal(np.isnan(d), np.isnan(h)) and np.array_equal(d[np.isinf(h)], h[np.isinf(h)]), (what, k)
        assert np.all(np.isfinite(d[fin])), (what, k)
        bound = np.spacing(np.abs(h[fin]).astype(np.float32)) if tol is None else tol
        assert np.all(np.abs(d[fin] - h[fin]) <= bound), (what, k)


@pytest.mark.gpu
def test_kitti_format_on_non_finite_rows(dev, golden_dir):
    """sassd_kitti_format vs kitti_bbox2results on detections with NaN / +-inf / 0 / 1e30 fields and centres at 4e9 m
    (rows the tail keeps: NaN and inf boxes survive the NMS, far boxes keep score 0.5): the same rows are kept, in
    order, with NaN where the host's numpy gives NaN (np.minimum / np.maximum and the keep test let it through) and
    the same clipping; rows past n_out untouched over a pre-filled buffer; a second call bit-identical."""
    from sassd_b200 import ops
    from sassd_b200.results import annos_from_rows, meta_block
    from tests.test_kitti_format import NAMES, SHAPES, _calibs, _host, _random_dets
    rng = np.random.default_rng(51)
    calibs = _calibs(golden_dir)
    dets, metas = [], []
    for b in range(3):
        d = _random_dets(rng, 60, b)
        cases = [(0, NAN), (1, NAN), (2, NAN), (3, NAN), (4, NAN), (5, NAN), (6, NAN), (0, INF), (0, -INF), (1, INF),
                 (2, -INF), (3, INF), (4, INF), (5, INF), (6, INF), (3, 0.0), (5, 0.0), (0, 4.2e9), (1, 1e30),
                 (6, 1e6)]
        for i, (c, v) in enumerate(cases):
            d[2 * i, c] = v                                              # every other row of the first 40
        d[45, [0, 1]] = [4.2e9, -16.0]
        dets.append(d)
        metas.append(dict(calib=calibs[b % 2], img_shape=SHAPES[b], sample_idx=b))
    B, cap = len(dets), 64 + GUARD
    det = np.zeros((B, cap, 9), F32)
    for b, d in enumerate(dets):
        det[b, :len(d)] = d
    d_det = torch.from_numpy(det).to(dev)
    nd = torch.tensor([len(d) for d in dets], dtype=torch.int32, device=dev)
    meta = torch.from_numpy(np.stack([meta_block(m["calib"], m["img_shape"]) for m in metas])).to(dev)
    runs = []
    for _ in range(2):
        rows = _filled((B, cap, ops._lib.KITTI_ROW), torch.float64, dev)
        n_out = _filled((B,), torch.int32, dev)
        ops._call("sassd_kitti_format", None, ops._ptr(d_det), ops._ptr(nd), B, cap, ops._ptr(meta), ops._ptr(rows),
                  ops._ptr(n_out), ops._stream())
        torch.cuda.synchronize()
        for b in range(B):
            assert _untouched(rows[b, int(n_out[b]):]), "frame %d: rows past n_out written" % b
        runs.append((rows, n_out))
    assert _bits(runs[0][0]) == _bits(runs[1][0]) and _bits(runs[0][1]) == _bits(runs[1][1])
    got = annos_from_rows(runs[0][0].cpu().numpy(), runs[0][1].cpu().numpy(), NAMES, [m["sample_idx"] for m in metas])
    n_nan = 0
    for b, (d, m) in enumerate(zip(dets, metas)):
        with np.errstate(invalid="ignore", over="ignore"):
            host = _host(d, m)
        _same_rows(got[b], host, "frame %d" % b)
        n_nan += int(np.isnan(host["bbox"]).any(1).sum())
    assert n_nan >= 10                                                  # NaN rows are kept, as on the host


# ====================================================================== 7. the whole step on constructed checkpoints
# conv_box's channels per anchor: x y z w l h r; the x bias puts every guided box near 4e9 m (1e10 pixels), the w
# bias makes expf overflow, the class bias selects a few thousand anchors
VARIANTS = {"x_far": (0, 1e9), "x_inf": (0, 3e38), "w_inf": (3, 100.0)}


def _bad_state_dict(variant):
    from sassd_b200 import checkpoint
    sd = dict(checkpoint.make_synthetic_state_dict(0, 1))
    ch, val = VARIANTS[variant]
    b = sd["rpn_head.conv_box.bias"].clone()
    b[ch::7] = val
    sd["rpn_head.conv_box.bias"] = b
    sd["rpn_head.conv_cls.bias"] = sd["rpn_head.conv_cls.bias"] + 0.5
    return sd


def _car_model(sd, prec):
    import sassd_b200 as S
    from sassd_b200 import checkpoint
    from tests.checkpoint_weights import CAR_CFG
    model, _, _ = S.build_from_config(S.Config.fromfile(CAR_CFG), device="cuda:0")
    checkpoint.load_state_dict_into(model, sd)
    if prec != "f16x3":
        from sassd_b200 import ops
        model.set_precision(ops.PREC_FP32)
    return model


def _same_dets(a, b, what):
    assert len(a) == len(b), what
    for x, y in zip(a, b):
        assert (x["boxes_lidar"] is None) == (y["boxes_lidar"] is None), what
        if y["boxes_lidar"] is not None:
            for k in ("boxes_lidar", "scores", "label_preds"):
                assert np.array_equal(x[k], y[k]), "%s: %s" % (what, k)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["f16x3", "fp32"])
@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_step_on_boxes_far_off_the_map(dev, variant, prec):
    """forward_points eager and captured and detect_stream complete on every guided box lying past 2^31 pixels
    (x_far: PSWarp samples nothing, every score is exactly 0, so the boxes keep sigmoid(0) = 0.5 as under the
    reference's zero padding) or at an infinite position or size (x_inf, w_inf: every PSWarp score is NaN and every
    box is dropped)."""
    from sassd_b200.synth import synth_cloud
    model = _car_model(_bad_state_dict(variant), prec)
    model.extra_head.det_cap = NMS_CAP          # x_far keeps every guided box: its BEV boxes are degenerate at 4e9 m
    clouds = [synth_cloud(3), synth_cloud(9)]
    out, aux = model.forward_points(clouds, return_aux=True)
    ks = aux["d_k"].cpu().numpy()
    ps = aux["ps_scores"].cpu().numpy()
    assert np.all(ks > 50), ks
    gb = aux["guided"].cpu().numpy()
    for b, k in enumerate(ks):
        if variant == "x_far":
            assert np.all(ps[b, :k] == 0.0), "frame %d: PSWarp scores" % b
            d = out[b]
            assert d["boxes_lidar"] is not None and np.all(d["scores"] == 0.5)
            assert np.all(d["boxes_lidar"][:, 0] > 8.6e8)             # (x + 0) * 2.5 >= 2^31 pixels
        else:
            assert np.all(np.isnan(ps[b, :k])), "frame %d: PSWarp scores" % b
            assert out[b]["boxes_lidar"] is None, "frame %d: a box with a NaN score was kept" % b
        col = gb[b, :k, 3 if variant == "w_inf" else 0]
        assert np.all(col > 8.6e8) and (variant == "x_far") == bool(np.isfinite(col).all()), "frame %d" % b
    model.enable_cuda_graph(2, 32768)
    try:
        _same_dets(model.forward_points(clouds), out, "captured %s %s" % (variant, prec))
        got = list(model.detect_stream([clouds, clouds], 2, 32768, depth=2))
        _same_dets(got[0], out, "detect_stream %s %s" % (variant, prec))
        _same_dets(got[1], out, "detect_stream %s %s, second slot" % (variant, prec))
    finally:
        model.disable_cuda_graph()


@pytest.mark.gpu
def test_checkpoint_sweep_with_a_bad_checkpoint_beside_seed_0(dev):
    """A sweep of [w_inf checkpoint, seed 0] completes, eager and captured, and its seed-0 member's detections and
    losses equal a sweep of seed 0 alone, bit for bit."""
    from sassd_b200 import checkpoint
    from sassd_b200.detectors import CheckpointSweep
    from sassd_b200.synth import synth_cloud
    good = _car_model(checkpoint.make_synthetic_state_dict(0, 1), "f16x3")
    bad = _car_model(_bad_state_dict("w_inf"), "f16x3")
    clouds = [synth_cloud(3), synth_cloud(9)]
    gts = [np.array([[20.0, 0.0, -1.7, 1.6, 3.9, 1.56, 0.3], [35.0, 8.0, -1.6, 1.7, 4.1, 1.5, -1.2]], F32),
           np.array([[12.0, -5.0, -1.7, 1.6, 3.9, 1.56, 1.5]], F32)]
    labels = [np.array([1, 1]), np.array([1])]
    both, alone = CheckpointSweep([bad, good]), CheckpointSweep([good])
    try:
        for captured in (False, True):
            if captured:
                both.enable_cuda_graph(2, 32768)
                alone.enable_cuda_graph(2, 32768)
            (rb, lb), (rg, lg) = both.forward_points(clouds, gt_bboxes=gts, gt_labels=labels)
            (ra, la), = alone.forward_points(clouds, gt_bboxes=gts, gt_labels=labels)
            _same_dets(rg, ra, "seed-0 member, captured=%s" % captured)
            assert lg == la, "seed-0 member's losses, captured=%s" % captured
            assert all(d["boxes_lidar"] is None for d in rb)
    finally:
        both.disable_cuda_graph()
        alone.disable_cuda_graph()


@pytest.mark.gpu
def test_uncalibrated_seed_1_weights_on_20k_point_frames(dev):
    """Seed 1's synthetic weights (BatchNorm statistics not calibrated) on car_cfg's 20 k-point synthetic frames,
    eager and captured, once: the step completes (a capacity flag is a result, not a fault)."""
    from sassd_b200 import checkpoint
    from sassd_b200.lib import SassdError
    from sassd_b200.synth import synth_cloud
    model = _car_model(checkpoint.make_synthetic_state_dict(1, 1), "f16x3")
    clouds = [synth_cloud(s) for s in range(4)]
    try:
        for captured in (False, True):
            if captured:
                model.enable_cuda_graph(4, 32768)
            try:
                out = model.forward_points(clouds)
                assert len(out) == 4
            except SassdError as e:
                assert "CAP" in str(e), str(e)
    finally:
        model.disable_cuda_graph()
    torch.cuda.synchronize()
