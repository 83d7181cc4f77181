"""SA-SSD's training targets and losses (csrc/targets.cu) at their thresholds, ties, capacities and extremes.

Inputs are built by hand and go through the C ABI (``ops``); every output is compared with the numpy oracle
(oracle/targets.py) and the loss values also with a plain fp64 restatement written here.

CPU: the constructions land on the intended fp32 IoUs (exactly f32(thr) and one ulp either side, for NearestIou and
RotateIou3d); the oracle reproduces tests/golden/loss_edges.npz (the reference's own create_target_torch,
SSDRotateHead.loss and PSWarpHead.loss on these constructions, made by make_golden_loss_edges.py) - labels and IoU bits
exactly.
GPU: labels, IoU bits and positive counts equal the oracle; box targets within 2 ulp; empty and masked slots are written
(-1 / 0) over NaN-filled outputs, rows past d_rows stay untouched and a second call gives the same bits; GT capacities
1, 255 and 256 with 0, 1, cap and cap + 1 boxes; the PSWarp slot layout at its edges; B = 1, 2, 16 on the real
200 x 176 grid; loss elements at extreme logits, the smooth-L1 knee, large yaws and signed-zero direction targets.
"""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import targets as OT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32
EPS32 = float(np.finfo(np.float32).eps)          # 2^-23
S = f32(2.0 ** -20)                              # length unit of the constructions: every coordinate is dyadic
PI2 = f32(np.pi / 2)
CLASSES = ["Car", "Pedestrian", "Cyclist"]
THR = {"Car": (0.6, 0.45), "Pedestrian": (0.5, 0.35), "Cyclist": (0.5, 0.35)}
H, W = 4, 8                                      # head grid of the constructed RPN case: 64 anchors per class
P = H * W * 2
BETA = f32(1.0 / 9.0)
LOGITS = f32([0.0, 1e-8, -1e-8, 15.0, -15.0, 88.0, -88.0, 89.0, -89.0, 1e4, -1e4])


def ulps(t):
    """f32(t) one ulp below, at and above."""
    t = f32(t)
    return [np.nextafter(t, f32(-1)), t, np.nextafter(t, f32(2))]


def ratio(t):
    """The first integers (p, q), 2^23 <= q < 2^24 and p + q even, whose fp32 quotient f32(p) / f32(q) is t: the
    quotient rounds (__fdiv_rn and numpy divide alike), everything before it is exact.  IoUs one ulp from a simple
    fraction like 3/5 need denominators this large: |p/q - 3/5| >= 1/(5q)."""
    for lo in range(2 ** 23, 2 ** 24, 2 ** 18):
        q = np.arange(lo, lo + 2 ** 18, dtype=np.int64)
        p = np.rint(q * float(t)).astype(np.int64)
        ok = np.nonzero((p.astype(f32) / q.astype(f32) == f32(t)) & ((p + q) % 2 == 0))[0]
        if len(ok):
            return int(p[ok[0]]), int(q[ok[0]])
    raise ValueError(t)


def _box(x, y, z, w, l, h, ry=0.0):
    return [f32(x), f32(y), f32(z), f32(w), f32(l), f32(h), f32(ry)]


def _swapped(b):
    """The same near box given with w / l exchanged and ry = pi/2."""
    return [b[0], b[1], b[2], b[4], b[3], b[5], PI2]


# ------------------------------------------------------------------------------------------------ constructions
def threshold_cells(cls, y0):
    """For each of pos and neg of ``cls``, one ulp below, at and above: an anchor (wa*S x 1) and a GT (wg*S x 1) that
    overlap by o*S in x, with o / (wa + wg - o) = p / q from ratio(t), so the near IoU lands on t (wa, wg even, every
    coordinate an integer multiple of S below 2^24, wa + wg even below 2^25: each fp32 step is exact but the last
    division); plus an anchor equal to the
    GT so that the GT's maximum (1) lies elsewhere and the threshold anchor is labelled by the thresholds alone.  Odd
    cells give the GT swapped (ry = pi/2), even cells the anchor.  Returns (gts, anchors, [(anchor, gt, target)])."""
    gts, anchors, checks = [], [], []
    k = 0
    for thr in THR[cls]:
        for t in ulps(thr):
            o, u = ratio(t)
            wa = 2 * ((u + o + 3) // 4)
            wg = u + o - wa
            y = y0 + 8 * k
            a = _box(wa * S / 2, y, -1.0, wa * S, 1, 1.5)
            g = _box((wa - o) * S + wg * S / 2, y, -1.0, wg * S, 1, 1.5)
            twin = list(g)
            if k % 2:
                g = _swapped(g)
            else:
                a = _swapped(a)
            checks.append((len(anchors), len(gts), t))
            gts.append(g)
            anchors += [a, twin]
            k += 1
    return gts, anchors, checks


def tie_cells(y0):
    """Car ties and forcing: (gts, gt_labels, gt_types extra rows, anchors)."""
    gts, labels, anchors = [], [], []
    # duplicate GT with different labels: the anchor equal to both takes the first one's label (3)
    d = _box(0, y0, -1.0, 4, 2, 1.5)
    gts += [d, d]; labels += [3, 1]
    anchors += [d]
    # a GT 4 x 2 whose maximum 0.6 is shared by the anchors shifted by -1 and +1 (all forced), and one whose maximum
    # 2/14 < neg is shared by anchors shifted by -3 and +3 (forced although below the negative threshold)
    for k, sh in enumerate((1, 3)):
        y = y0 + 8 * (k + 1)
        gts.append(_box(0, y, -1.0, 4, 2, 1.5)); labels.append(1)
        anchors += [_box(-sh, y, -1.0, 4, 2, 1.5), _box(sh, y, -1.0, 4, 2, 1.5)]
    # one anchor tied across two GT: the first listed (label 2) wins the argmax
    y = y0 + 24
    gts += [_box(-1, y, -1.0, 4, 2, 1.5), _box(1, y, -1.0, 4, 2, 1.5)]; labels += [2, 1]
    anchors += [_box(0, y, -1.0, 4, 2, 1.5)]
    # a GT far from every anchor: its maximum is 0, it forces nothing
    gts.append(_box(0, -900, -1.0, 4, 2, 1.5)); labels.append(1)
    return gts, labels, anchors


def _pad(anchors, cls_index):
    """Pad a class block to P anchors with boxes far from everything."""
    out = [list(a) for a in anchors]
    while len(out) < P:
        i = len(out)
        out.append(_box(2000 + 10 * i + 1000 * cls_index, 500, -1.0, 1.6, 3.9, 1.56, (i % 2) * PI2))
    return out


def rpn_case():
    """Two frames, three classes on one shared anchor set [3P, 7].  Frame 0: the Car threshold and tie cells, the
    Pedestrian threshold cells, a GT of a type that is no anchor class (gt_class -1) lying on an anchor, no Cyclist.
    Frame 1: no Car, the Pedestrian GT again but every Pedestrian anchor masked, the Cyclist threshold cells."""
    blocks, checks, cells = [], {}, {}
    for ci, cls in enumerate(CLASSES):
        g, a, ch = threshold_cells(cls, 100 * ci)
        if cls == "Car":
            tg, tl, ta = tie_cells(60)
            cells[cls] = (g + tg, [1] * len(g) + tl)
            a = a + ta
            a.append(_box(0, -300, -1.0, 1.6, 3.9, 1.56))       # the anchor under the "Van"
        else:
            cells[cls] = (g, [ci + 1] * len(g))
        checks[cls] = ch
        blocks.append(_pad(a, ci))
    anchors = np.asarray(sum(blocks, []), f32)
    van = _box(0, -300, -1.0, 1.6, 3.9, 1.56)
    frames = []
    for b in range(2):
        rows, types_, labels = [], [], []
        present = ("Car", "Pedestrian") if b == 0 else ("Pedestrian", "Cyclist")
        for cls in present:
            g, l = cells[cls]
            rows += g; labels += l; types_ += [cls] * len(g)
        if b == 0:
            rows.append(van); labels.append(1); types_.append("Van")
        frames.append((np.asarray(rows, f32), np.asarray(labels, np.int64), np.array(types_)))
    mask = np.ones((2, 3 * P), bool)
    mask[0, [40, P + 50]] = False                 # two masked padding anchors
    mask[1, P:2 * P] = False                      # frame 1: every Pedestrian anchor masked
    return dict(anchors=np.broadcast_to(anchors, (2,) + anchors.shape).copy(), mask=mask,
                gts=[f[0] for f in frames], gt_labels=[f[1] for f in frames], gt_types=[f[2] for f in frames],
                checks=checks, cells=cells)


def pswarp_case():
    """Two frames of (GT, guided boxes).  A box (p*S, 1, 1) centred in a GT (q*S, 1, 1) has 3D IoU p / q (a nested
    rectangle: the BEV overlap is the box's own area, exactly): cells at 0.7 one ulp below, at and above, each
    GT also matched exactly by a box (IoU 1); duplicate GT; two boxes tied for a GT's maximum; a GT that overlaps no
    box (frame 1, which has no GT rows in front)."""
    gts, boxes, checks = [], [], []
    for k, t in enumerate(ulps(0.7)):
        p, q = ratio(t)
        y = 8 * k
        g = _box(0, y, -1.0, q * S, 1, 1)
        checks.append((len(boxes) + 1, len(gts), t))
        gts.append(g)
        boxes += [g, _box(0, y, -1.0, p * S, 1, 1)]
    d = _box(0, 40, -1.0, 4, 2, 1.5)
    gts += [d, d]
    boxes += [_box(0.5, 40, -1.0, 4, 2, 1.5)]
    gts.append(_box(0, 48, -1.0, 4, 2, 1.5))
    boxes += [_box(-1, 48, -1.0, 4, 2, 1.5), _box(1, 48, -1.0, 4, 2, 1.5), _box(30, 30, -1.0, 2, 4, 1.5, 1.0)]
    g0 = np.asarray(gts, f32)
    b0 = np.concatenate([g0, np.asarray(boxes, f32)])      # GT rows first, as get_guided_anchors prepends them
    g1 = np.asarray([_box(0, 8, -1.0, 4, 2, 1.5), _box(0, -700, -1.0, 4, 2, 1.5)], f32)
    b1 = np.asarray([_box(0.25, 8, -1.0, 4, 2, 1.5), _box(0, 8.5, -0.9, 4, 2, 1.5), _box(9, 9, -1.0, 1, 1, 1)], f32)
    return dict(gts=[g0, g1], guided=[b0, b1], checks=checks, n_gt_rows=[len(g0), 0])


def head_case(seed=0):
    """Head outputs for the RPN case ([2, 3, H, W, 14 / 6 / 4], the reference's layout) and PSWarp scores: every class
    logit from LOGITS, direction logits 100 apart, box codes at |p - t| = 1/9 and one ulp either side on the anchors
    whose target is 0 (those equal to their GT), yaw predictions up to +-100 rad."""
    rng = np.random.default_rng(seed)
    B, nc = 2, 3
    box = (rng.normal(0, 0.3, (B, nc, H, W, 14))).astype(f32)
    box[..., 6] = rng.uniform(-100, 100, box[..., 6].shape)
    box[..., 13] = rng.uniform(-100, 100, box[..., 13].shape)
    cls = LOGITS[rng.integers(0, len(LOGITS), (B, nc, H, W, 2 * nc))]
    dirp = rng.normal(0, 2, (B, nc, H, W, 4)).astype(f32)
    dirp[..., 1] = dirp[..., 0] + f32(100) * rng.choice(f32([-1, 1]), dirp[..., 0].shape)
    dirp[..., 3] = dirp[..., 2] - f32(100)
    knee = np.array([-BETA, BETA] + [s * np.nextafter(BETA, f32(v)) for s in (1, -1) for v in (0, 1)], f32)
    flat = box.reshape(B, -1, 7)                     # anchor order of the concatenated class blocks
    case = rpn_case()
    for b in range(B):
        eq = np.nonzero((case["anchors"][b][:, None, :] == case["gts"][b][None, :, :]).all(-1).any(1))[0]
        for j, i in enumerate(eq):
            flat[b, i, :6] = knee[(np.arange(6) + j) % len(knee)]
    scores = LOGITS[rng.integers(0, len(LOGITS), sum(len(g) for g in pswarp_case()["guided"]))]
    return dict(box_preds=flat.reshape(box.shape), cls_preds=cls.astype(f32), dir_preds=dirp, ps_scores=scores)


def inputs_digest(arrays):
    """sha256 over the named input arrays' bytes, in name order: the fixture records it beside its outputs."""
    h = hashlib.sha256()
    for k in sorted(arrays):
        a = np.ascontiguousarray(arrays[k])
        h.update(k.encode()); h.update(str(a.dtype).encode()); h.update(str(a.shape).encode()); h.update(a.tobytes())
    return h.hexdigest()


def fixture_inputs():
    rc, pc, hc = rpn_case(), pswarp_case(), head_case()
    out = dict(anchors=rc["anchors"], mask=rc["mask"], ps_counts=np.array([len(x) for x in pc["guided"]], np.int32),
               guided=np.concatenate(pc["guided"]), **hc)
    for b in range(2):
        out["gt%d" % b] = rc["gts"][b]
        out["gt_labels%d" % b] = rc["gt_labels"][b]
        out["gt_types%d" % b] = rc["gt_types"][b].astype("U16")
        out["ps_gt%d" % b] = pc["gts"][b]
    return out


def _gcls(types_):
    return np.array([CLASSES.index(t) if t in CLASSES else -1 for t in types_], np.int64)


def oracle_rpn(anchors, mask, gts, gt_types, gt_labels, num_class=3):
    pos = [THR[c][0] for c in CLASSES[:num_class]]
    neg = [THR[c][1] for c in CLASSES[:num_class]]
    return OT.rpn_targets(anchors, mask, gts, [_gcls(t) for t in gt_types], gt_labels, pos, neg, num_class)


# ------------------------------------------------------------------------------------------------------------ CPU
def test_constructions_land_on_the_intended_fp32_ious():
    rc = rpn_case()
    for ci, cls in enumerate(CLASSES):
        g, _ = rc["cells"][cls]
        blk = rc["anchors"][0, ci * P:(ci + 1) * P]
        for ai, gi, t in rc["checks"][cls]:
            v = OT.near_iou(blk[ai:ai + 1], np.asarray(g[gi:gi + 1], f32))[0, 0]
            assert v.view(np.int32) == f32(t).view(np.int32), (cls, ai, v, t)
        assert len(rc["checks"][cls]) == 6
    # the pos threshold exactly, and pos +- 1 ulp, are three distinct values
    assert len({float(t) for _, _, t in rc["checks"]["Car"]}) == 6
    pc = pswarp_case()
    for ai, gi, t in pc["checks"]:
        i = pc["n_gt_rows"][0] + ai
        v = OT.iou3d(pc["guided"][0][i:i + 1], pc["gts"][0][gi])
        assert v[0, 0].view(np.int32) == f32(t).view(np.int32), (ai, v, t)
    # ties are exact ties
    iou = OT.near_iou(np.asarray(rc["anchors"][0][:P]), rc["cells"]["Car"][0])
    assert (iou == iou.max(0, keepdims=True)).sum(0).max() >= 2


def test_oracle_reproduces_the_reference_edge_fixture(golden_dir):
    z = np.load(os.path.join(golden_dir, "loss_edges.npz"))
    inp = fixture_inputs()
    assert inputs_digest(inp) == str(z["inputs_sha256"]), "the constructions differ from the fixture's inputs"
    for k, v in inp.items():
        assert np.array_equal(z[k], v), k
    rc = rpn_case()
    L, T, M = oracle_rpn(rc["anchors"], rc["mask"], rc["gts"], rc["gt_types"], rc["gt_labels"])
    assert np.array_equal(L, z["rpn_labels"])
    assert np.array_equal(M.view(np.int32), z["rpn_ious"].view(np.int32))
    assert np.abs(T - z["rpn_targets"]).max() <= 1e-6
    # the thresholds decide: at pos and above positive, one ulp below pos ignored, neg ignored, one below neg negative
    for ci, cls in enumerate(CLASSES):
        b = 1 if cls == "Cyclist" else 0
        got = [int(L[b, ci * P + ai]) for ai, _, _ in rc["checks"][cls]]
        assert got == [-1, ci + 1, ci + 1, 0, -1, -1], (cls, got)
    # forcing, ties and the first maximum (Car block of frame 0, tie anchors after the 12 threshold anchors)
    assert L[0, 12:19].tolist() == [3, 1, 1, 1, 1, 2, 0]
    assert (L[1, :P] == 0).all() and (L[1, P:2 * P] == -1).all()
    pc = pswarp_case()
    c = np.r_[0, np.cumsum(z["ps_counts"])]
    for b in range(2):
        lb, _, mb = OT.create_target(pc["guided"][b], None, pc["gts"][b], None, OT.iou3d, 0.7, 0.7, encode=False)
        assert np.array_equal(lb, z["ps_labels"][c[b]:c[b + 1]])
        assert np.array_equal(mb.view(np.int32), z["ps_ious"][c[b]:c[b + 1]].view(np.int32))
    n0 = pc["n_gt_rows"][0]
    assert [int(z["ps_labels"][n0 + ai]) for ai, _, _ in pc["checks"]] == [0, 1, 1]
    # losses: the reference sums fp32 elements in fp32 (torch), the oracle in fp64
    exp = oracle_losses(inp)
    for k, v in exp.items():
        ref = float(z["loss_" + k][0])
        assert abs(v - ref) <= 2e-6 * abs(ref), (k, v, ref)


def oracle_losses(inp):
    B, nc = 2, 3
    rc = rpn_case()
    L, T, _ = oracle_rpn(rc["anchors"], rc["mask"], rc["gts"], rc["gt_types"], rc["gt_labels"])
    out = OT.rpn_losses(inp["box_preds"].reshape(B, -1, 7), inp["cls_preds"].reshape(B, -1, nc),
                        inp["dir_preds"].reshape(B, -1, 2), L, T, rc["anchors"])
    pc = pswarp_case()
    labs = [OT.create_target(pc["guided"][b], None, pc["gts"][b], None, OT.iou3d, 0.7, 0.7, encode=False)[0]
            for b in range(B)]
    out.update(OT.pswarp_loss(inp["ps_scores"], np.concatenate(labs), B))
    return out


# ------------------------------------------------------------------------------------------------------------ GPU
def _host(t):
    return t.detach().cpu().numpy()


def _ulp_diff(a, b):
    a, b = np.asarray(a, f32).view(np.int32).astype(np.int64), np.asarray(b, f32).view(np.int32).astype(np.int64)
    return np.abs(a - b)


def _dev(a, dtype=None):
    t = torch.from_numpy(np.ascontiguousarray(a))
    return (t if dtype is None else t.to(dtype)).cuda()


def _nan(shape, dtype=torch.float32):
    """An output buffer full of garbage: NaN for floats, 0xFF bytes for integers."""
    t = torch.empty(shape, dtype=dtype, device="cuda")
    t.view(torch.uint8).fill_(0xFF)
    return t


def _filled_ws(batch, gt_cap):
    from sassd_b200 import ops
    ws = ops.Workspace()
    ops._loss_ws(batch, gt_cap, torch.device("cuda"), ws).fill_(0xFF)
    return ws


def _assign_rpn(anchors, mask, num_class, gt, gcls, glab, d_ngt, pos, neg, status, ws):
    """sassd_assign_rpn through ops._call on outputs pre-filled with NaN / 0xFF."""
    import ctypes
    from sassd_b200 import ops
    B, gt_cap = gt.shape[0], gt.shape[1]
    na = anchors.shape[-2]
    labels, targets, ious, npos = _nan((B, na), torch.int32), _nan((B, na, 7)), _nan((B, na)), _nan((B,), torch.int32)
    w = ops._loss_ws(B, gt_cap, gt.device, ws)
    ops._call("sassd_assign_rpn", None, ops._ptr(anchors), 1 if anchors.dim() == 3 else 0, ops._ptr(mask), na,
              num_class, ops._ptr(gt), ops._ptr(gcls), ops._ptr(glab), ops._ptr(d_ngt), B, gt_cap,
              (ctypes.c_float * num_class)(*pos), (ctypes.c_float * num_class)(*neg), ops._ptr(labels),
              ops._ptr(targets), ops._ptr(ious), ops._ptr(npos), ops._ptr(status), ops._ptr(w), w.numel(),
              ops._stream())
    return labels, targets, ious, npos


def _stage(gts, gcls, glab, gt_cap):
    from sassd_b200.single_stage_heads import gt_arrays
    return tuple(_dev(a) for a in gt_arrays(gts, gcls, glab, gt_cap=gt_cap))


def _check_rpn(anchors_dev, mask, gts, gt_types, gt_labels, num_class, gt_cap, ws, A=None):
    """Run the kernel twice and compare with the oracle; returns the oracle's (L, T, M)."""
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    B = len(gts)
    gt, gc, gl, d_ngt = _stage(gts, [_gcls(t) for t in gt_types], gt_labels, gt_cap)
    pos = [THR[c][0] for c in CLASSES[:num_class]]
    neg = [THR[c][1] for c in CLASSES[:num_class]]
    m = _dev(mask.astype(np.uint8))
    r1 = _assign_rpn(anchors_dev, m, num_class, gt, gc, gl, d_ngt, pos, neg, status, ws)
    r2 = _assign_rpn(anchors_dev, m, num_class, gt, gc, gl, d_ngt, pos, neg, status, ws)
    for x, y in zip(r1, r2):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), "a second call gives other bits"
    A = _host(anchors_dev) if A is None else A
    A = np.broadcast_to(A, (B,) + A.shape[-2:])
    k = [min(len(g), gt_cap) for g in gts]
    L, T, M = oracle_rpn(A, mask, [g[:n] for g, n in zip(gts, k)], [t[:n] for t, n in zip(gt_types, k)],
                         [l[:n] for l, n in zip(gt_labels, k)], num_class)
    lab, tgt, iou, npos = (_host(x) for x in r1)
    assert np.array_equal(lab, L)
    assert np.array_equal(iou.view(np.int32), M.view(np.int32))
    assert _ulp_diff(tgt, T).max() <= 2
    assert (tgt[L <= 0] == 0).all() and not np.isnan(tgt).any()
    assert np.array_equal(npos, (L > 0).sum(1))
    over = any(len(g) > gt_cap for g in gts)
    assert int(status.item()) == (64 if over else 0)
    return L, T, M


@pytest.mark.gpu
@pytest.mark.parametrize("gt_cap", [None, 256])
@pytest.mark.parametrize("per_frame", [False, True])
def test_rpn_thresholds_ties_and_forcing_match_the_oracle_and_the_fixture(golden_dir, gt_cap, per_frame):
    z = np.load(os.path.join(golden_dir, "loss_edges.npz"))
    rc = rpn_case()
    anchors = _dev(rc["anchors"] if per_frame else rc["anchors"][0])
    cap = gt_cap or max(len(g) for g in rc["gts"])
    L, _, M = _check_rpn(anchors, rc["mask"], rc["gts"], rc["gt_types"], rc["gt_labels"], 3, cap, _filled_ws(2, cap))
    assert np.array_equal(L, z["rpn_labels"]) and np.array_equal(M.view(np.int32), z["rpn_ious"].view(np.int32))


def _grid_anchors():
    from sassd_b200.anchors import AnchorGeneratorStride
    return np.ascontiguousarray(AnchorGeneratorStride()([1, 200, 176]).reshape(-1, 7), f32)


def _grid_gts(rng, n, lo=(2.0, -38.0), hi=(68.0, 38.0)):
    g = np.c_[rng.uniform(lo[0], hi[0], n), rng.uniform(lo[1], hi[1], n), np.full(n, -1.78),
              rng.uniform(1.4, 1.8, n), rng.uniform(3.4, 4.4, n), rng.uniform(1.4, 1.7, n),
              rng.choice([0.0, np.pi / 2, 0.3, -1.2], n)]
    # on-grid copies: exact anchor boxes make ties and IoU 1
    return g.astype(f32)


@pytest.mark.gpu
@pytest.mark.parametrize("gt_cap", [1, 255, 256])
def test_gt_capacity_and_counts_on_the_real_grid(gt_cap):
    """d_ngt = 0, 1, gt_cap and gt_cap + 1 in one batch: the last sets SASSD_FLAG_GT_CAP and uses exactly the first
    gt_cap boxes; the GT table of assign_kernel is full at 256."""
    A = _grid_anchors()
    rng = np.random.default_rng(gt_cap)
    counts = [0, 1, gt_cap, gt_cap + 1]
    gts = [_grid_gts(rng, n) for n in counts]
    k = min(gt_cap, 4)
    gts[2][:k] = A[[1000, 1001, 20001, 20001]][:k]              # exact anchors, one duplicated
    types_ = [np.array(["Car"] * len(g)) for g in gts]
    labels = [np.ones(len(g), np.int64) for g in gts]
    mask = rng.random((4, len(A))) < 0.9
    L, _, _ = _check_rpn(_dev(A), mask, gts, types_, labels, 1, gt_cap, _filled_ws(4, gt_cap))
    assert (L[0][mask[0]] == 0).all() and (L[0][~mask[0]] == -1).all()
    assert (L[2] > 0).sum() >= min(gt_cap, 4)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 2, 16])
@pytest.mark.parametrize("per_frame", [False, True])
def test_batches_on_the_real_grid_and_per_frame_normalisation(B, per_frame):
    """Frames with GT, without GT, with every anchor masked, with only far GT (zero positives) and with GT of a class
    absent from the frame: labels / IoUs / npos exact, and the RPN losses of a random head within the derived bound
    of the oracle and of fp64."""
    from sassd_b200 import ops
    from sassd_b200.anchors import AnchorGeneratorStride
    rng = np.random.default_rng(100 + B)
    nc = 3
    gens = [AnchorGeneratorStride(sizes=s) for s in ([1.6, 3.9, 1.56], [0.6, 0.8, 1.73], [0.6, 1.76, 1.73])]
    A = np.concatenate([g([1, 200, 176]).reshape(-1, 7) for g in gens]).astype(f32)
    if per_frame:
        A = np.broadcast_to(A, (B,) + A.shape).copy()
        A[:, :, :2] += rng.uniform(-0.1, 0.1, (B, 1, 2)).astype(f32)
    gts, types_, labels = [], [], []
    for b in range(B):
        kind = b % 5
        n = [6, 0, 6, 3, 5][kind]
        g = _grid_gts(rng, n) if kind != 3 else _grid_gts(rng, n, (200.0, 200.0), (300.0, 300.0))
        t = np.array(["Car", "Pedestrian", "Van", "Car", "Pedestrian", "Car"][:n])
        if kind == 4:
            t = np.array(["Car"] * n)                        # no Pedestrian or Cyclist in this frame
        gts.append(g); types_.append(t); labels.append(np.array([CLASSES.index(x) + 1 if x in CLASSES else 1
                                                                  for x in t], np.int64))
    mask = rng.random((B, A.shape[-2])) < 0.85
    if B > 2:
        mask[2] = False                                         # frame 2: every anchor masked
    ws = _filled_ws(B, 8)
    L, T, _ = _check_rpn(_dev(A), mask, gts, types_, labels, nc, 8, ws)
    if B > 3:
        assert (L[2] == -1).all() and (L[3] > 0).sum() == 0 and (L[1] > 0).sum() == 0
    # the losses on a random head, normalised per frame by each frame's own positives
    AA = np.broadcast_to(A, (B,) + A.shape[-2:])
    head, box, cls, dirp = _random_head(rng, B, 200, 176, nc)
    out = _nan((3,))
    ops.rpn_loss(_dev(head), nc, _dev(A), _dev(L.astype(np.int32)), _dev(T), _dev((L > 0).sum(1).astype(np.int32)),
                 out, ws=ws)
    got = _host(out)
    _assert_rpn_losses(got, box, cls, dirp, L, T, AA)


# ---------------------------------------------------------------------------------------------- PSWarp slot layout
@pytest.mark.gpu
@pytest.mark.parametrize("head_cap_kind", ["zero", "one", "gt_cap"])
@pytest.mark.parametrize("head_full", [False, True])
@pytest.mark.parametrize("k_kind", ["zero", "fill", "over"])
def test_pswarp_slot_layout_at_its_edges(head_cap_kind, head_full, k_kind):
    """Slots [0, head_cap) hold d_head[b] boxes, [head_cap, n) hold min(d_k[b], n - head_cap); every other slot is -1
    with IoU 0 even over NaN-filled outputs; labels and IoU bits equal the oracle on the selected boxes."""
    from sassd_b200 import ops
    pc = pswarp_case()
    gts = pc["gts"]
    gt_cap = max(len(g) for g in gts)
    head_cap = {"zero": 0, "one": 1, "gt_cap": gt_cap}[head_cap_kind]
    n = head_cap + 12
    B = 3
    gts = gts + [gts[0][:3]]
    boxes = np.full((B, n, 7), np.nan, f32)                    # slots past the counts hold garbage
    d_head = np.array([head_cap if head_full else 0] * B, np.int32)
    d_k = np.array([{"zero": 0, "fill": n - head_cap, "over": n - head_cap + 5}[k_kind]] * B, np.int32)
    d_k[2] = min(d_k[2], 3)
    for b in range(B):
        g = gts[b]
        boxes[b, :min(d_head[b], len(g))] = g[:d_head[b]]
        if d_head[b] > len(g):
            boxes[b, len(g):d_head[b]] = g[0]
        guided = pc["guided"][b % 2][pc["n_gt_rows"][b % 2]:]
        k = min(d_k[b], n - head_cap)
        src = np.concatenate([guided] * (k // max(len(guided), 1) + 1))[:k]
        boxes[b, head_cap:head_cap + k] = src
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    gt, _, _, dn = _stage(gts, None, None, gt_cap)
    ws = _filled_ws(B, gt_cap)
    import ctypes
    labels, ious, npos = _nan((B, n), torch.int32), _nan((B, n)), _nan((B,), torch.int32)
    w = ops._loss_ws(B, gt_cap, gt.device, ws)
    bd, dh, dk = _dev(boxes), _dev(d_head), _dev(d_k)
    ops._call("sassd_assign_pswarp", None, ops._ptr(gt), ops._ptr(dn), B, gt_cap, ops._ptr(bd), n,
              ops._ptr(dh if head_cap else None), head_cap, ops._ptr(dk), ctypes.c_float(0.7), ctypes.c_float(0.7),
              ops._ptr(labels), ops._ptr(ious), ops._ptr(npos), ops._ptr(status), ops._ptr(w), w.numel(),
              ops._stream())
    lab, iou, npos = _host(labels), _host(ious), _host(npos)
    l2, i2, _ = ops.assign_pswarp(gt, dn, bd, dk, 0.7, 0.7, status, d_head=dh if head_cap else None,
                                  head_cap=head_cap, ws=ws)
    assert np.array_equal(_host(l2), lab) and np.array_equal(_host(i2).view(np.int32), iou.view(np.int32))
    for b in range(B):
        sel = np.r_[np.arange(min(d_head[b], head_cap)), head_cap + np.arange(min(d_k[b], n - head_cap))]
        rest = np.setdiff1d(np.arange(n), sel)
        assert (lab[b, rest] == -1).all() and (iou[b, rest].view(np.int32) == 0).all()
        if len(sel) == 0:
            assert npos[b] == 0
            continue
        lb, _, mb = OT.create_target(boxes[b, sel], None, gts[b], None, OT.iou3d, 0.7, 0.7, encode=False)
        assert np.array_equal(lab[b, sel], lb), b
        # axis-aligned boxes bit for bit; rotated ones within 1e-6 (box_overlap's rotated corners, as in
        # test_losses.py: the kernel may contract products the oracle's C rounds one by one)
        straight = boxes[b, sel, 6] == 0
        assert np.array_equal(iou[b, sel][straight].view(np.int32), mb[straight].view(np.int32)), b
        assert np.abs(iou[b, sel] - mb).max() <= 1e-6, b
        assert npos[b] == (lb > 0).sum()
    assert int(status.item()) == 0


@pytest.mark.gpu
def test_pswarp_fixture_labels_and_ious(golden_dir):
    from sassd_b200 import ops
    z = np.load(os.path.join(golden_dir, "loss_edges.npz"))
    pc = pswarp_case()
    ks = z["ps_counts"]
    boxes = np.zeros((2, int(ks.max()), 7), f32)
    c = np.r_[0, np.cumsum(ks)]
    for b in range(2):
        boxes[b, :ks[b]] = z["guided"][c[b]:c[b + 1]]
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    gt, _, _, dn = _stage(pc["gts"], None, None, 256)
    lab, iou, npos = ops.assign_pswarp(gt, dn, _dev(boxes), _dev(ks.astype(np.int32)), 0.7, 0.7, status,
                                       ws=_filled_ws(2, 256))
    lab, iou = _host(lab), _host(iou)
    assert np.array_equal(np.concatenate([lab[b, :ks[b]] for b in range(2)]), z["ps_labels"])
    assert np.array_equal(np.concatenate([iou[b, :ks[b]] for b in range(2)]).view(np.int32),
                          z["ps_ious"].view(np.int32))


# ---------------------------------------------------------------------------------------------- points in boxes
@pytest.mark.gpu
def test_points_in_boxes_at_256_boxes_foreign_frames_and_rows_past_d_rows():
    from sassd_b200 import ops
    rng = np.random.default_rng(7)
    B, cap = 2, 256
    gx, gy = np.meshgrid(np.arange(16) * 4.0 + 2.0, np.arange(16) * 4.0 - 30.0)
    g0 = np.c_[gx.ravel(), gy.ravel(), np.full(256, -1.7), np.full(256, 1.6), np.full(256, 3.9), np.full(256, 1.5),
               rng.uniform(-3, 3, 256)].astype(f32)
    g1 = g0[:3].copy()
    pts = [np.c_[np.zeros(4000), rng.uniform(0, 66, 4000), rng.uniform(-32, 34, 4000), rng.uniform(-2, 0, 4000)],
           np.c_[np.ones(800), rng.uniform(0, 14, 800), rng.uniform(-32, -22, 800), rng.uniform(-2, 0, 800)]]
    # rows of frames outside [0, batch): never labelled, offsets 0
    pts.append(np.c_[rng.choice([-1.0, 2.0, 5.0], 300), rng.uniform(0, 66, 300), rng.uniform(-32, 34, 300),
                     rng.uniform(-2, 0, 300)])
    pm = np.concatenate(pts).astype(f32)
    n = len(pm)
    rows_cap = 4 * n
    pm_dev = torch.zeros((rows_cap, 4), dtype=torch.float32, device="cuda")
    pm_dev[:n] = _dev(pm)
    pm_dev[n:, 1:] = _dev(np.tile(g0[:1, :3], (rows_cap - n, 1)))  # past d_rows: points inside box 0 of frame 0
    gt, _, _, dn = _stage([g0, g1], None, None, cap)
    d_rows = torch.tensor([n], dtype=torch.int32, device="cuda")
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    for _ in range(2):
        labels, offsets, npos = _nan((rows_cap,), torch.int32), _nan((rows_cap, 3)), _nan((1,), torch.int32)
        ops._call("sassd_points_in_boxes", None, ops._ptr(pm_dev), ops._ptr(d_rows), rows_cap, ops._ptr(gt),
                  ops._ptr(dn), B, cap, ops._ptr(labels), ops._ptr(offsets), ops._ptr(npos), ops._ptr(status),
                  ops._stream())
        lab, off = _host(labels), _host(offsets)
        assert (lab[n:] == -1).all() and (off[n:].view(np.int32) == -1).all(), "rows past d_rows were written"
        ol = np.zeros(n, np.int32)
        oo = np.zeros((n, 3), f32)
        for b, g in enumerate([g0, g1]):
            sel = pm[:, 0] == b
            fl, rg = OT.pts_in_boxes3d(pm[sel, 1:], g)
            ol[sel] = fl.max(0)
            oo[sel] = rg
        assert np.array_equal(lab[:n], ol) and np.array_equal(off[:n].view(np.int32), oo.view(np.int32))
        assert int(npos.item()) == int(ol.sum()) and ol[:4000].sum() > 100 and not lab[4800:n].any()
    assert int(status.item()) == 0


# ---------------------------------------------------------------------------------------------- loss elements
def _focal64(x, t, w):
    x, t, w = (np.asarray(v, np.float64) for v in (x, t, w))
    with np.errstate(over="ignore"):
        p = 1.0 / (1.0 + np.exp(-x))
    pt = (1 - p) * t + p * (1 - t)
    bce = np.maximum(x, 0) - x * t + np.log1p(np.exp(-np.abs(x)))
    return bce * (0.25 * t + 0.75 * (1 - t)) * w * pt * pt, bce * (0.25 * t + 0.75 * (1 - t)) * w, pt


def _sl1_64(d):
    d = np.abs(np.asarray(d, np.float64))
    beta = float(BETA)
    return np.where(d < beta, 0.5 * d * d / beta, d - float(f32(0.5 / 9.0)))


def _ce64(l0, l1, label):
    l0, l1 = np.asarray(l0, np.float64), np.asarray(l1, np.float64)
    m = np.maximum(l0, l1)
    return m + np.log(np.exp(l0 - m) + np.exp(l1 - m)) - np.where(label > 0, l1, l0)


# Bounds.  Every element is non-negative and the kernel sums elements in fp64, so a loss can only be off by what each
# fp32 element is off, summed, plus the two fp32 roundings of the result ((float)sum, then / B * scale: 3 roundings).
# (a) kernel vs oracle: both evaluate the same fp32 expression; they differ only where a transcendental does.  The
#     focal element bce * wt * pt^2 uses expf twice and log1pf once: CUDA's expf / log1pf are within 2 / 1 ulp, numpy's
#     float32 exp / log1p within 1 ulp each, so p = 1/(1+e) is off by at most 3 + 2 = 5 half-ulps ... bounded by 4 ulp
#     relative, pt^2 by 8, bce by 5: 13 ulp per side, 26 in all; the sin-difference element uses sinf / cosf (2 ulp in
#     CUDA, 1 in numpy) twice per product: 6 ulp per side; the direction term expf / logf: 7 per side.  k = 32 covers
#     every case with margin below an order of magnitude: k * eps32 = 3.8e-6 relative at most, and far less in sum.
# (b) kernel vs exact fp64: the same 13 + 3 roundings of the fp32 arithmetic itself, k = 32 again, plus the
#     cancellation in 1 - p when p is near 1 (t = 1, x >> 0): p carries an absolute error up to DELTA = 4 eps32, which
#     1 - p keeps as an absolute error, so the element is off by up to bce * alpha * w * (2 pt DELTA + DELTA^2); and in
#     the sin-difference |pe - te| when pe ~ te: absolute error 3 eps32 (|pe| + |te|), which the smooth-L1 passes on
#     at most 1:1 (its slope is min(d / beta, 1)).  Between the kernel and the oracle that absolute error is at most
#     (2 + 2 + 0.5) + (1 + 1 + 0.5) = 7 ulp of the larger product: 8 eps32 (|pe| + |te|) is used for (a) and (b).
K = 32
DELTA = 4 * EPS32


def _focal_bound(x, t, w):
    e, awb, pt = _focal64(x, t, w)
    cancel = np.where(np.asarray(t) > 0, awb * (2 * pt * DELTA + DELTA * DELTA), 0.0)
    return e, K * EPS32 * np.abs(e), cancel


def _assert_close(got, exp, rel_sum, abs_sum, what):
    """|got - exp| <= K eps32 * sum|elements| + absolute cancellation + 3 roundings of the result."""
    bound = rel_sum + abs_sum + 3 * EPS32 * abs(exp)
    assert abs(got - exp) <= bound, (what, got, exp, bound)


def _random_head(rng, B, Hh, Ww, nc):
    na = 2 * nc
    N = nc * Hh * Ww * 2
    box = rng.normal(0, 0.3, (B, N, 7)).astype(f32)
    box[..., 6] = rng.uniform(-100, 100, (B, N))
    cls = np.where(rng.random((B, N, nc)) < 0.2, LOGITS[rng.integers(0, len(LOGITS), (B, N, nc))],
                   rng.normal(-2, 2, (B, N, nc))).astype(f32)
    dirp = rng.normal(0, 2, (B, N, 2)).astype(f32)
    dirp[:, ::7, 1] = dirp[:, ::7, 0] + f32(100)
    dirp[:, 3::7, 1] = dirp[:, 3::7, 0] - f32(100)
    # anchor i = ((c * hw + pix) * 2 + rot) -> head[b, pix, c * 14 + rot * 7 + e], the layout rpn_loss_kernel reads
    hw = Hh * Ww
    def lay(a, width):
        return a.reshape(B, nc, hw, 2, width).transpose(0, 2, 1, 3, 4).reshape(B, hw, nc * 2 * width)
    head = np.concatenate([lay(box, 7), lay(cls, nc), lay(dirp, 2)], -1).reshape(B, Hh, Ww, -1)
    assert head.shape[-1] == na * 7 + na * nc + na * 2
    return np.ascontiguousarray(head, f32), box, cls, dirp


def _assert_rpn_losses(got, box, cls, dirp, L, T, A):
    B, N, nc = cls.shape
    exp_o = OT.rpn_losses(box, cls, dirp, L, T, A)
    npos = np.maximum((L > 0).sum(1, keepdims=True), 1).astype(np.float64)
    pos, cared = (L > 0), (L >= 0)
    onehot = (L[..., None] == np.arange(1, nc + 1)).astype(np.float64)
    e, rel, cancel = _focal_bound(cls, onehot, (cared / npos)[..., None])
    cls_sum, cls_rel, cls_abs = e.sum() / B, rel.sum() / B, cancel.sum() / B
    p6, t6 = box[..., 6].astype(np.float64), T[..., 6].astype(np.float64)
    pe, te = np.sin(p6) * np.cos(t6), np.cos(p6) * np.sin(t6)
    d = np.concatenate([(box[..., :6].astype(np.float64) - T[..., :6]), (pe - te)[..., None]], -1)
    loc_e = _sl1_64(d) * (pos / npos)[..., None]
    loc_sum = 2 * loc_e.sum() / B
    loc_rel = 2 * K * EPS32 * loc_e.sum() / B
    loc_abs = 2 * (8 * EPS32 * (np.abs(pe) + np.abs(te)) * pos / npos).sum() / B
    dl = ((T[..., 6] + A[..., 6]) > 0).astype(np.int64)
    dir_e = _ce64(dirp[..., 0], dirp[..., 1], dl) * pos / npos
    dir_sum = 0.2 * dir_e.sum() / B
    for k, (g, ex, r, a) in {"rpn_loc_loss": (got[0], loc_sum, loc_rel, loc_abs),
                             "rpn_cls_loss": (got[1], cls_sum, cls_rel, cls_abs),
                             "rpn_dir_loss": (got[2], dir_sum, K * EPS32 * dir_sum, 0.0)}.items():
        _assert_close(float(g), exp_o[k], r, a, k + " vs oracle")       # (a)
        _assert_close(float(g), ex, r, a, k + " vs fp64")                # (b)
        _assert_close(exp_o[k], ex, r, a, k + " oracle vs fp64")


@pytest.mark.gpu
def test_loss_elements_at_extremes_b16():
    """rpn_loss, pswarp_loss and aux_loss at B = 16 on constructed labels / targets: logits 0, +-1e-8, +-15, +-88,
    +-89, +-1e4; |p - t| at 1/9 and one ulp either side; yaws up to +-100 rad; tg[6] + a[6] at +0 and -0; direction
    logits 100 apart; frames with zero positives and wholly masked frames."""
    from sassd_b200 import ops
    rng = np.random.default_rng(3)
    B, nc, Hh, Ww = 16, 3, 4, 8
    N = nc * Hh * Ww * 2
    head, box, cls, dirp = _random_head(rng, B, Hh, Ww, nc)
    L = rng.integers(-1, nc + 1, (B, N)).astype(np.int64)
    L[3] = -1                                                   # wholly masked
    L[4] = np.minimum(L[4], 0)                                  # no positives
    T = rng.normal(0, 0.5, (B, N, 7)).astype(f32)
    T[..., 6] = rng.uniform(-3, 3, (B, N))
    A = np.broadcast_to(np.zeros((N, 7), f32), (B, N, 7)).copy()
    A[..., 6] = rng.choice(f32([0.0, PI2, -PI2]), (B, N))
    # the smooth-L1 knee: targets 0, predictions +-1/9 and one ulp either side
    knee = np.array([BETA, -BETA, np.nextafter(BETA, f32(0)), np.nextafter(BETA, f32(1)),
                     -np.nextafter(BETA, f32(0)), -np.nextafter(BETA, f32(1))], f32)
    T[:, :64, :6] = 0
    box[:, :64, :6] = knee[np.arange(64 * 6).reshape(64, 6) % 6]
    # signed-zero direction targets: tg[6] + a[6] = +0 and -0 (both "not > 0")
    T[:, 64:72, 6] = f32(0.0); A[:, 64:72, 6] = f32(0.0)
    T[:, 72:80, 6] = f32(-0.0); A[:, 72:80, 6] = f32(-0.0)
    assert (np.signbit(T[:, 72:80, 6] + A[:, 72:80, 6])).all() and not np.signbit(T[:, 64:72, 6] + A[:, 64:72, 6]).any()
    L[:, :80] = np.maximum(L[:, :80], 1)
    L[3] = -1; L[4] = np.minimum(L[4], 0)
    # rebuild the head from the edited box codes
    hw = Hh * Ww
    lay = lambda a, w: a.reshape(B, nc, hw, 2, w).transpose(0, 2, 1, 3, 4).reshape(B, hw, nc * 2 * w)  # noqa: E731
    head = np.ascontiguousarray(np.concatenate([lay(box, 7), lay(cls, nc), lay(dirp, 2)], -1).reshape(B, Hh, Ww, -1))
    ws = _filled_ws(B, 1)
    out = _nan((3,))
    args = (_dev(head), nc, _dev(A), _dev(L.astype(np.int32)), _dev(T), _dev((L > 0).sum(1).astype(np.int32)), out)
    ops.rpn_loss(*args, ws=ws)
    first = _host(out).copy()
    _assert_rpn_losses(first, box, cls, dirp, L, T, A)
    ops.rpn_loss(*args, ws=ws)
    assert np.array_equal(_host(out).view(np.int32), first.view(np.int32))
    # Isolated elements, where one transcendental decides the sum.  Yaws near k*pi against a target yaw 0: the
    # sin-difference element is sin(p)^2 / (2 beta) with |sin p| ~ 1e-3, so a sine with an absolute (not relative)
    # error of ~2^-21 after a cheap argument reduction is off by ~1e-3 relative, far past K eps32.
    n1 = 1 * 1 * Hh * Ww * 2
    k = np.arange(n1) % 31 + 1
    dlt = f32(1e-3) * (1 + np.arange(n1) % 7) * np.where(np.arange(n1) % 2, f32(-1), f32(1))
    b1 = np.zeros((1, n1, 7), f32)
    b1[0, :, 6] = (k * np.float64(np.pi) + dlt).astype(f32)
    c1 = np.full((1, n1, 1), f32(-12))
    d1 = rng.normal(0, 2, (1, n1, 2)).astype(f32)
    L1 = np.ones((1, n1), np.int64)
    T1 = np.zeros((1, n1, 7), f32)
    A1 = np.zeros((1, n1, 7), f32)
    lay1 = lambda a, w: a.reshape(1, 1, hw, 2, w).transpose(0, 2, 1, 3, 4).reshape(1, hw, 2 * w)  # noqa: E731
    h1 = np.ascontiguousarray(np.concatenate([lay1(b1, 7), lay1(c1, 1), lay1(d1, 2)], -1).reshape(1, Hh, Ww, -1))
    o1 = _nan((3,))
    ops.rpn_loss(_dev(h1), 1, _dev(A1), _dev(L1.astype(np.int32)), _dev(T1), _dev(np.array([n1], np.int32)), o1, ws=ws)
    _assert_rpn_losses(_host(o1), b1, c1, d1, L1, T1, A1)
    # Background scores near -27 alone (the element ~e^(3x) stays a normal fp32): p = 1 / (1 + e^|x|) and
    # log1p(e^-|x|) are the whole element, and its three exps err in the same direction, so an exp computed as exp2
    # of a rounded x * log2(e) puts ~40 ulp on every element at these x (where that product rounds by almost half an
    # ulp), past K + 3 = 35; CUDA's expf (2 ulp) stays near 10.
    s1 = np.where(np.arange(64) % 2, f32(-27.65625), f32(-26.703125)).reshape(1, 64).astype(f32)
    l1 = np.zeros((1, 64), np.int32)
    o2 = _nan((1,))
    ops.pswarp_loss(_dev(s1), _dev(l1), _dev(np.zeros(1, np.int32)), o2, ws=ws)
    e, rel, cancel = _focal_bound(s1, np.zeros_like(s1), np.ones_like(s1))
    for ex in (OT.pswarp_loss(s1, l1, 1)["loss_cls"], e.sum()):
        _assert_close(float(_host(o2)[0]), ex, rel.sum(), cancel.sum(), "isolated loss_cls")
    # PSWarp: scores over every logit, labels -1 / 0 / 1, one normaliser for the batch
    n = 40
    sc = LOGITS[rng.integers(0, len(LOGITS), (B, n))]
    pl = rng.integers(-1, 2, (B, n)).astype(np.int32)
    pl[5] = -1
    out1 = _nan((1,))
    ops.pswarp_loss(_dev(sc), _dev(pl), _dev((pl > 0).sum(1).astype(np.int32)), out1, ws=ws)
    exp_o = OT.pswarp_loss(sc, pl, B)["loss_cls"]
    tot = max(int((pl > 0).sum()), 1)
    e, rel, cancel = _focal_bound(sc, (pl > 0).astype(np.float64), (pl >= 0) / tot)
    for ex in (exp_o, e.sum() / B):
        _assert_close(float(_host(out1)[0]), ex, rel.sum() / B, cancel.sum() / B, "loss_cls")
    # aux: every point, logits at the extremes, offsets at the knee
    rows_cap, rows = 4096, 3000
    pc_ = np.zeros(rows_cap, f32); pc_[:rows] = LOGITS[rng.integers(0, len(LOGITS), rows)]
    pc_[rows:] = np.nan                                         # past d_rows: never read
    preg = rng.normal(0, 0.3, (rows_cap, 3)).astype(f32)
    preg[:600] = knee[np.arange(1800).reshape(600, 3) % 6]
    plab = (rng.random(rows_cap) < 0.3).astype(np.int32)
    poff = np.zeros((rows_cap, 3), f32); poff[600:] = rng.normal(0, 0.3, (rows_cap - 600, 3))
    out2 = _nan((2,))
    d_rows = torch.tensor([rows], dtype=torch.int32, device="cuda")
    npos = int(plab[:rows].sum())
    ops.aux_loss(_dev(pc_), _dev(preg), _dev(plab), _dev(poff), d_rows, B, torch.tensor([npos], dtype=torch.int32,
                 device="cuda"), out2, ws=ws)
    got = _host(out2)
    exp_o = OT.aux_losses(pc_[:rows], preg[:rows], plab[:rows], poff[:rows], B)
    e, rel, cancel = _focal_bound(pc_[:rows], plab[:rows] > 0, np.full(rows, 1.0 / max(npos, 1)))
    r = _sl1_64(preg[:rows].astype(np.float64) - poff[:rows]) * (plab[:rows] > 0)[:, None] / max(npos, 1)
    for ex, key, rs, ab, g in ((e.sum() / B, "aux_loss_cls", rel.sum() / B, cancel.sum() / B, got[0]),
                               (r.sum() / B, "aux_loss_reg", K * EPS32 * r.sum() / B, 0.0, got[1])):
        _assert_close(float(g), exp_o[key], rs, ab, key + " vs oracle")
        _assert_close(float(g), ex, rs, ab, key + " vs fp64")


@pytest.mark.gpu
def test_kernels_reproduce_the_edge_fixture_losses(golden_dir):
    """The reference's SSDRotateHead.loss / PSWarpHead.loss values of the fixture, from the kernels' own targets."""
    from sassd_b200 import ops
    z = np.load(os.path.join(golden_dir, "loss_edges.npz"))
    rc = rpn_case()
    B, nc = 2, 3
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    gt, gc, gl, dn = _stage(rc["gts"], [_gcls(t) for t in rc["gt_types"]], rc["gt_labels"], 256)
    ws = _filled_ws(B, 256)
    lab, tgt, _, npos = ops.assign_rpn(_dev(rc["anchors"]), _dev(rc["mask"].astype(np.uint8)), nc, gt, gc, gl, dn,
                                       [THR[c][0] for c in CLASSES], [THR[c][1] for c in CLASSES], status, ws=ws)
    box = z["box_preds"].reshape(B, -1, 7)
    hw = H * W
    lay = lambda a, w: a.reshape(B, nc, hw, 2, w).transpose(0, 2, 1, 3, 4).reshape(B, hw, nc * 2 * w)  # noqa: E731
    head = np.concatenate([lay(box, 7), lay(z["cls_preds"].reshape(B, -1, nc), nc),
                           lay(z["dir_preds"].reshape(B, -1, 2), 2)], -1).reshape(B, H, W, -1)
    out = _nan((4,))
    ops.rpn_loss(_dev(head), nc, _dev(rc["anchors"]), lab, tgt, npos, out[:3], ws=ws)
    pc = pswarp_case()
    ks = z["ps_counts"]
    boxes = np.zeros((B, int(ks.max()), 7), f32)
    scores = np.zeros((B, int(ks.max())), f32)
    c = np.r_[0, np.cumsum(ks)]
    for b in range(B):
        boxes[b, :ks[b]] = pc["guided"][b]
        scores[b, :ks[b]] = z["ps_scores"][c[b]:c[b + 1]]
    pgt, _, _, pdn = _stage(pc["gts"], None, None, 256)
    pl, _, pn = ops.assign_pswarp(pgt, pdn, _dev(boxes), _dev(ks.astype(np.int32)), 0.7, 0.7, status, ws=ws)
    ops.pswarp_loss(_dev(scores), pl, pn, out[3:4], ws=ws)
    got = dict(zip(("rpn_loc_loss", "rpn_cls_loss", "rpn_dir_loss", "loss_cls"), _host(out).tolist()))
    exp = oracle_losses({k: z[k] for k in ("box_preds", "cls_preds", "dir_preds", "ps_scores")})
    assert int(status.item()) == 0
    for k, v in got.items():
        ref = float(z["loss_" + k][0])
        # the kernel against the oracle at the (a) bound's size, and the reference (fp32 torch sums) at 2e-6
        assert abs(v - exp[k]) <= 4e-6 * abs(exp[k]), (k, v, exp[k])
        assert abs(v - ref) <= 4e-6 * abs(ref), (k, v, ref)


@pytest.mark.gpu
def test_loss_points_b16_with_empty_frames_matches_the_oracle():
    """loss_points at B = 16 on synthetic clouds, frames 1, 6 and 11 without GT, against the oracle at 2e-6."""
    from tests.test_losses import _frames, _model
    model = _model()
    B = 16
    pts, gts, labels = _frames(B, 1, empty=(1, 6, 11))
    res, aux = model.loss_points(pts, gts, labels, return_aux=True)
    fr = _host(aux["frame_rows"])
    n0 = int(fr[-1])
    pm = _host(aux["points_mean"])[:n0]
    ol, oo = OT.aux_targets(pm, gts)
    assert np.array_equal(_host(aux["point_labels"])[:n0], ol)
    exp = OT.aux_losses(_host(aux["point_cls"])[:n0], _host(aux["point_reg"])[:n0], ol, oo, B)
    anchors = model.anchor_set.anchors
    A = np.broadcast_to(anchors, (B,) + anchors.shape)
    mask = _host(aux["mask"]).astype(bool)
    pos, neg = model.rpn_head.thresholds(model.train_cfg.rpn, model.class_names)
    L, T, M = OT.rpn_targets(A, mask, gts, [l - 1 for l in labels], labels, pos, neg, 1)
    assert np.array_equal(_host(aux["rpn_labels"]), L)
    assert np.array_equal(_host(aux["rpn_ious"]).view(np.int32), M.view(np.int32))
    assert _ulp_diff(_host(aux["rpn_targets"]), T).max() <= 2
    box, cls, dirp = [t.reshape(B, -1, w) for t, w in zip(model.rpn_head._split(aux["head"]), (7, 1, 2))]
    exp.update(OT.rpn_losses(_host(box), _host(cls), _host(dirp), L, T, A))
    gt_cap = aux["ps_boxes"].shape[1] - aux["guided"].shape[1]
    boxes, scores, d_k = _host(aux["ps_boxes"]), _host(aux["ps_scores"]), _host(aux["d_k"])
    olab, osc = [], []
    for b in range(B):
        sel = np.r_[np.arange(len(gts[b])), gt_cap + np.arange(d_k[b])]
        lb, _, _ = OT.create_target(boxes[b, sel], None, gts[b], None, OT.iou3d, 0.7, 0.7, encode=False)
        assert np.array_equal(_host(aux["ps_labels"])[b, sel], lb)
        olab.append(lb); osc.append(scores[b, sel])
    exp.update(OT.pswarp_loss(np.concatenate(osc), np.concatenate(olab), B))
    for k, v in exp.items():
        # the (a) bound: K eps32 per non-negative element plus three roundings of the result, 2e-6 relative at most
        # for these well-conditioned logits (|x| < 8: no cancellation)
        assert abs(res[k] - v) <= 2e-6 * max(abs(v), 1e-30), (k, res[k], v)
