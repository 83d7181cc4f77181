"""The detection tail at its capacities: guided-anchor selection and decode (sassd_decode_select), PSWarp sampling
(sassd_pswarp), rescoring + stable sort + rotated NMS (sassd_rescore_nms) and the NMS bitmask (sassd_nms_mask).

Every size in this part of the step comes from the data, so the inputs here are constructed to reach the edges: the
real 200x176 head grid, chunk and grid-pass boundaries, every capacity (k_cap, NMS_CAP = 4096, det_cap) at cap-1, cap
and cap+1, tied scores, touching and degenerate boxes.  Each stage is compared with the plain reference of the same
operation (oracle/ref_pipeline.py) and the NMS bitmask with the unmodified reference CUDA kernel, bit for bit.
Tolerances are written next to their assertions.
"""
import ctypes
import hashlib
import lzma
import os

import numpy as np
import pytest
import torch

from oracle import ref_pipeline as O
from sassd_b200.synth import synth_cloud

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
H, W = 200, 176                 # the head / PSWarp grid of the KITTI configs
DS_CHUNK = 1024                 # anchors per CTA of the selection kernels (csrc/head.cu)
GUIDED_THR, SCORE_THR, IOU_THR = 0.1, 0.3, 0.1
NMS_CAP, K_CAP = 4096, 8192     # ops.NMS_CAP, SSDRotateHead.k_cap
FLAG_GUIDED_CAP, FLAG_NMS_CAP, FLAG_DET_CAP = 4, 8, 32
EPS32 = float(np.finfo(np.float32).eps)
MARGIN = 1e-6                   # every constructed score keeps this distance from its threshold (sigmoid scale)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _sig64(x):
    return 1.0 / (1.0 + np.exp(-np.asarray(x, np.float64)))


def _ordered(a):
    i = np.ascontiguousarray(a, np.float32).view(np.int32).astype(np.int64)
    return np.where(i < 0, -(i & 0x7fffffff), i)


def _ulps(a, b):
    """distance in fp32 units in the last place (+0 and -0 are 0 apart)"""
    return np.abs(_ordered(a) - _ordered(b))


def _ulp(x):
    return np.spacing(np.abs(np.asarray(x, np.float32))).astype(np.float64)


# ====================================================================== 1. guided anchors (sassd_decode_select)
def _selection(kind, n_anchors, k_cap, rs):
    """anchor indices (ascending) that a frame of the given kind selects"""
    nch = -(-n_anchors // DS_CHUNK)
    if kind == "chunk":             # exactly one full chunk: the count ends on a chunk boundary
        return np.arange(2 * DS_CHUNK, 3 * DS_CHUNK)
    if kind == "last":              # everything in the last (partial) chunk
        lo = (nch - 1) * DS_CHUNK
        return np.sort(rs.choice(np.arange(lo, n_anchors), min(200, n_anchors - lo), replace=False))
    n = {"cap-1": k_cap - 1, "cap": k_cap, "cap+1": k_cap + 1}.get(kind, kind)
    return np.sort(rs.choice(n_anchors, int(n), replace=False))


def _decode_case(ncls, per_frame, kinds, k_cap, seed):
    """Head map [B,H,W,stride] in the product's channel layout (conv_box | conv_cls | conv_dir_cls, anchor
    a = ((cls_a*H + y)*W + x)*2 + rot), anchors [B or 1,Na,7], mask [B,Na], and the per-anchor arrays the oracle reads.
    Frame b selects exactly the anchors of _selection(kinds[b]); 64 masked-out anchors per frame carry the highest
    score; yaw +0 / -0 / tiny negative is crossed with both direction labels; equal direction logits and (multi-class)
    equal top class logits occur."""
    rs = np.random.RandomState(seed)
    B, na = len(kinds), 2 * ncls
    Na = ncls * H * W * 2
    codes = rs.normal(0, 0.5, (B, Na, 7)).astype(np.float32)
    codes[..., 3:6] = rs.normal(0, 0.3, (B, Na, 3))
    codes[..., 6] = rs.uniform(-1, 1, (B, Na))
    cls = rs.uniform(-9, -2.5, (B, Na, ncls)).astype(np.float32)          # sigmoid <= 0.076: below 0.1
    dirl = rs.normal(0, 1, (B, Na, 2)).astype(np.float32)
    mask = (rs.uniform(size=(B, Na)) > 0.15).astype(np.uint8)
    nt = B if per_frame else 1
    anchors = np.stack([rs.uniform(0, 70, (nt, Na)), rs.uniform(-40, 40, (nt, Na)), rs.uniform(-2, -1, (nt, Na)),
                        rs.uniform(0.5, 2, (nt, Na)), rs.uniform(0.7, 4.5, (nt, Na)), rs.uniform(1.4, 1.8, (nt, Na)),
                        rs.choice([0.0, 1.57], (nt, Na))], -1).astype(np.float32)
    sels, edges = [], []
    for b, kind in enumerate(kinds):
        sel = _selection(kind, Na, k_cap, rs)
        sels.append(sel)
        mask[b, sel] = 1
        edges.append(sel[:0])
        if sel.size:
            cls[b, sel, :] = rs.uniform(-9, 6, (sel.size, ncls))
            top = rs.randint(ncls, size=sel.size)
            cls[b, sel, top] = rs.uniform(-1.5, 6, sel.size)                  # sigmoid >= 0.18: selected
            if ncls > 1:                                                        # tied top classes: first class wins
                t = np.arange(0, sel.size, 7)
                other = (top[t] + 1 + rs.randint(ncls - 1, size=t.size)) % ncls
                best = cls[b, sel[t], top[t]]
                cls[b, sel[t], :] = np.minimum(cls[b, sel[t], :], best[:, None])
                cls[b, sel[t], other] = best
            d = sel[3::10]
            dirl[b, d, 1] = dirl[b, d, 0]                                       # tied direction logits: label 0
            # decoded yaw rt + ra exactly +0, -0 and -1e-30, each with both direction labels
            e = sel[np.linspace(0, sel.size - 1, min(sel.size, 24)).astype(int)]
            for j, a in enumerate(e):
                anchors[b if per_frame else 0, a, 6] = -0.0
                codes[b, a, 6] = (0.0, -0.0, -1e-30)[j % 3]
                dirl[b, a] = (1.0, 0.0) if (j // 3) % 2 == 0 else (0.0, 1.0)
            edges[b] = e
        rest = np.setdiff1d(np.arange(Na), sel)
        hidden = rs.choice(rest, 64, replace=False)
        mask[b, hidden] = 0
        cls[b, hidden, :] = 9.0                                                 # the best scores, never selectable
    head = np.concatenate([
        codes.reshape(B, ncls, H, W, 14).transpose(0, 2, 3, 1, 4).reshape(B, H, W, ncls * 14),
        cls.reshape(B, ncls, H, W, 2 * ncls).transpose(0, 2, 3, 1, 4).reshape(B, H, W, 2 * ncls * ncls),
        dirl.reshape(B, ncls, H, W, 4).transpose(0, 2, 3, 1, 4).reshape(B, H, W, ncls * 4)], -1)
    assert head.shape[-1] == na * 7 + na * ncls + na * 2
    return dict(head=np.ascontiguousarray(head), codes=codes, cls=cls, dirl=dirl, mask=mask,
                anchors=anchors if per_frame else anchors[0], sels=sels, edges=edges)


# (num_class, per-frame anchor tables, k_cap, selected count / kind per frame)
_MIXED = ["zero", "one", "chunk", 2048, "last", "cap-1", "cap", 1, 1023, 1025, 4095, 4096, 4097, 777, "last", 3000]
DECODE_CASES = [
    (1, False, K_CAP, ["cap"]),
    (3, False, K_CAP, ["cap+1"]),
    (1, True, 300, ["zero", "one", "cap-1"]),
    (3, False, 300, ["cap", "last", "one"]),
    (1, False, 300, ["cap+1", "cap", "zero"]),
    (3, True, 300, ["one", "cap+1", "cap-1"]),
    (1, False, K_CAP, _MIXED),
    (3, True, K_CAP, _MIXED),
    (1, True, K_CAP, _MIXED[:15] + ["cap+1"]),
]


@pytest.mark.parametrize("ncls,per_frame,k_cap,kinds", DECODE_CASES,
                         ids=["c%d-%s-B%d-cap%d-%d" % (c, "frame" if p else "shared", len(k), kc, i)
                              for i, (c, p, kc, k) in enumerate(DECODE_CASES)])
def test_decode_select_matches_oracle(dev, ncls, per_frame, k_cap, kinds):
    """sassd_decode_select vs get_guided_anchors / second_box_decode (torch fp32): selection, labels and anchor order
    exactly; overflow keeps the first k_cap selected anchors in anchor order and raises GUIDED_CAP; boxes per
    component within the ulp bounds stated below."""
    from sassd_b200 import ops
    kinds = [0 if k == "zero" else 1 if k == "one" else k for k in kinds]
    case = _decode_case(ncls, per_frame, kinds, k_cap, seed=len(kinds) * 100 + ncls * 10 + k_cap % 7)
    B, Na = len(kinds), ncls * H * W * 2
    # threshold margin: no score may be decided by libm (max over classes of the fp64 sigmoid of the fp32 logits)
    score64 = _sig64(case["cls"]).max(-1)
    assert np.abs(score64 - GUIDED_THR).min() >= MARGIN
    counts = [len(s) for s in case["sels"]]
    want_flag = any(c > k_cap for c in counts)
    status = torch.zeros((1,), dtype=torch.int32, device=dev)
    boxes, labels, index, d_k = ops.decode_select(torch.from_numpy(case["head"]).to(dev), ncls,
                                                  torch.from_numpy(case["anchors"]).to(dev),
                                                  torch.from_numpy(case["mask"]).to(dev), GUIDED_THR, k_cap, status)
    g, lab, idx, _ = O.get_guided_anchors(torch.from_numpy(case["codes"]), torch.from_numpy(case["cls"]),
                                          torch.from_numpy(case["dirl"]), torch.from_numpy(case["anchors"]),
                                          torch.from_numpy(case["mask"]).bool(), ncls, GUIDED_THR, return_index=True)
    boxes, labels, index, d_k = boxes.cpu().numpy(), labels.cpu().numpy(), index.cpu().numpy(), d_k.cpu().numpy()
    assert int(status.item()) == (FLAG_GUIDED_CAP if want_flag else 0), (int(status.item()), counts, k_cap)
    worst = np.zeros(2)
    for b in range(B):
        exp_idx = idx[b].numpy()
        assert np.array_equal(exp_idx, case["sels"][b]), "frame %d: construction" % b    # masked anchors never selected
        k = min(counts[b], k_cap)
        assert d_k[b] == k, (b, d_k[b], counts[b], k_cap)
        # overflow: the kept prefix is the first k_cap selected anchors in anchor order
        assert np.array_equal(index[b, :k], exp_idx[:k]), "frame %d: anchor index list" % b
        assert np.array_equal(labels[b, :k], lab[b].numpy()[:k]), "frame %d: labels" % b
        got, exp = boxes[b, :k], g[b].numpy()[:k]
        # x, y = code * sqrt(l^2 + w^2) + anchor: correctly rounded fp32 operations, so exact against the same
        # operations in numpy.  torch's vectorised CPU sqrt is not correctly rounded (1 ulp off on ~0.7 % of inputs),
        # so against torch: |code| * ulp(diag) + one rounding of the product and one of the sum.
        an = case["anchors"][b] if per_frame else case["anchors"]
        a_sel, c_sel = an[exp_idx[:k]], case["codes"][b, exp_idx[:k]]
        diag = np.sqrt(a_sel[:, 4] * a_sel[:, 4] + a_sel[:, 3] * a_sel[:, 3])
        for j in (0, 1):
            prod = c_sel[:, j] * diag
            assert np.array_equal(got[:, j], prod + a_sel[:, j]), "frame %d: x, y" % b
            assert np.all(np.abs(got[:, j].astype(np.float64) - exp[:, j]) <=
                          np.abs(c_sel[:, j]) * _ulp(diag) + _ulp(prod) + _ulp(exp[:, j])), "frame %d: x, y vs torch" % b
        # r = code + anchor (+ pi flip): exact, sign of zero included
        assert np.array_equal(_ordered(got[:, 6]), _ordered(exp[:, 6])), "frame %d: yaw" % b
        # w, l, h = exp(code) * anchor: CUDA's expf is within 2 ulp (CUDA math API), torch's CPU exp within 1 ulp,
        # plus the product's rounding on each side: <= 4 ulp.  Measured on an H100: max 2 ulp.
        u = _ulps(got[:, 3:6], exp[:, 3:6])
        assert u.max(initial=0) <= 4, "frame %d: w/l/h differ by %d ulp" % (b, u.max())
        # z = (code * h_a + z_a + h_a/2) - h_g/2: the exact part is shared, h_g/2 carries the exp bound above, then one
        # rounding of z itself (measured on an H100: at most 0.67 of this bound)
        dz = np.abs(got[:, 2].astype(np.float64) - exp[:, 2])
        bound = 4 * _ulp(exp[:, 5] / 2) + _ulp(exp[:, 2])
        assert np.all(dz <= bound), "frame %d: z" % b
        if k:
            worst = np.maximum(worst, [u.max(), (dz / bound).max()])
        # yaw edges: flip iff (r > 0) != dir_label, with r = +0, -0, -1e-30 never > 0
        e = case["edges"][b]
        if e.size:
            pos = np.searchsorted(case["sels"][b], e)
            keep = pos < k
            dl = case["dirl"][b, e[keep]]
            flipped = dl[:, 1] > dl[:, 0]
            r = boxes[b, pos[keep], 6]
            assert np.all(r[flipped] == np.float32(np.pi)) and np.all(np.abs(r[~flipped]) <= 1e-30)
    print("decode: max w/l/h %d ulp, max |dz| / bound %.2f" % (worst[0], worst[1]))


# ====================================================================== 2. PSWarp (sassd_pswarp)
OFF_X, OFF_Y, SSCALE = 0.0, 40.0, 2.5            # grid_offsets, 1 / featmap_stride of the KITTI configs


def _pswarp_edge_boxes():
    """[N,7] boxes whose 28 sample points land on the map's edges (pixel = (metres + offset) * 2.5)."""
    f32 = np.float32
    rows = []

    def box(px, py, w, l, r):
        rows.append([px / SSCALE - OFF_X, py / SSCALE - OFF_Y, -1.0, w, l, 1.5, r])

    # every sample point on one pixel centre (zero-size boxes): corners, last column / row, interior
    for px, py in ((0, 0), (W - 1, H - 1), (W - 1, 50), (30, H - 1), (87, 100), (0, H - 1), (W - 1, 0)):
        for r in (0.0, np.pi, -np.pi / 2):
            box(px, py, 0.0, 0.0, r)
    # points in (W-2, W-1) / (H-2, H-1): the east / south neighbour is the last column / row
    for py in (20.3, 120.7, H - 1.5):
        box(W - 1.5, py, 0.2, 0.3, 0.0)
    for px in (10.2, 100.6, W - 1.5):
        box(px, H - 1.5, 0.3, 0.2, 0.0)
    # points in (-1, 0) and (W-1, W), (H-1, H): one neighbour off the map
    for px, py in ((-0.5, 60.4), (W - 0.5, 60.4), (80.3, -0.5), (80.3, H - 0.5), (-0.5, -0.5), (W - 0.5, H - 0.5)):
        box(px, py, 0.2, 0.2, 0.0)
    # wholly off the map
    for px, py in ((-5.0, 50.0), (W + 4.0, 50.0), (50.0, -6.0), (50.0, H + 5.0), (-40.0, -40.0), (500.0, 80.0)):
        box(px, py, 0.4, 0.6, 0.3)
    # yaw +-pi, +-pi/2 with very long and very wide boxes
    for r in (np.pi, -np.pi, np.pi / 2, -np.pi / 2):
        box(88.0, 100.0, 0.3, 60.0, r)
        box(88.0, 100.0, 30.0, 0.5, r)
        box(170.0, 190.0, 2.0, 40.0, r)
    return np.asarray(rows, f32)


def _pswarp_ref64(feat_hwc, x32, y32):
    """fp64 bilinear sampling (zero padding, align_corners) of part p's channel p at the fp32 sample positions of the
    reference's gen_sample_grid.  Normalising then un-normalising is the identity in exact arithmetic, so the pixel
    position is x32 itself.  Returns (score [N], S [N]) with S = (1/28) sum over parts of the |features| of the valid
    bilinear neighbours ("the sampled features")."""
    P, N = x32.shape
    ix, iy = x32.astype(np.float64), y32.astype(np.float64)
    x0, y0 = np.floor(ix), np.floor(iy)
    we, ws = ix - x0, iy - y0
    part = np.arange(P)[:, None].repeat(N, 1)
    acc = np.zeros((P, N))
    mag = np.zeros((P, N))
    for dx, dy, wt in ((0, 0, (1 - we) * (1 - ws)), (1, 0, we * (1 - ws)), (0, 1, (1 - we) * ws), (1, 1, we * ws)):
        xx, yy = x0 + dx, y0 + dy
        ok = (xx >= 0) & (xx < W) & (yy >= 0) & (yy < H)
        f = np.where(ok, feat_hwc[np.clip(yy, 0, H - 1).astype(int), np.clip(xx, 0, W - 1).astype(int), part], 0.0)
        acc += wt * f
        mag += np.abs(f)
    return acc.mean(0), mag.sum(0) / P


# |error| <= C_PS * eps32 * S (S: _pswarp_ref64), derived for the kernel and for the reference's own fp32 path:
#  * arithmetic: per part 3 roundings in each of the 4 weight * feature terms (1 - w, w_a * w_b, * f) and 3 in their
#    sum, then 5 in the 28-lane tree and 1 in the / 28: 12 u = 6 eps relative to sum |w f| <= sum |f|;
#  * position: the pixel coordinate goes through / (W-1), * 2 - 1, + 1, / 2, * (W-1) (<= 4 u (W-1) pixels) and the fp32
#    sin / cos / rotation of gen_sample_grid (<= 4 u (W-1) for boxes below ~70 m): 8 u (W-1) = 4 eps (W-1) pixels per
#    axis; bilinear interpolation moves by at most that times the sum of |f| of the neighbours.
C_PS = 6 + 4 * (W - 1) + 4 * (H - 1)


def test_pswarp_edges_and_grid_passes(dev):
    """sassd_pswarp vs gen_sample_grid + bilinear_gridsample: points on the last row / column, just inside and
    outside the map, wholly off it (exactly 0), yaw +-pi and +-pi/2, very long / wide boxes; 6000 boxes in one frame
    (more than one pass of the grid-stride loop: 4 CTAs x 8 warps per SM), an empty frame beside it."""
    from sassd_b200 import ops
    rs = np.random.RandomState(7)
    B, C, n, k_cap = 2, 28, 6000, 6016
    feat = rs.normal(0, 1, (B, H, W, C)).astype(np.float32)
    edge = _pswarp_edge_boxes()
    ne = len(edge)
    b7 = np.stack([rs.uniform(-5, 75, n), rs.uniform(-45, 45, n), np.full(n, -1.0), rs.uniform(0.5, 3, n),
                   rs.uniform(0.5, 6, n), np.full(n, 1.5), rs.uniform(-np.pi, np.pi, n)], 1).astype(np.float32)
    late = 4224 + 500                   # beyond one pass on 132 SMs: edges in both passes
    b7[:ne] = edge
    b7[late:late + ne] = edge
    boxes = rs.normal(0, 50, (B, k_cap, 7)).astype(np.float32)     # rows past d_k are garbage, never read
    boxes[0, :n] = b7
    d_k = torch.tensor([n, 0], dtype=torch.int32, device=dev)
    got = ops.pswarp(torch.from_numpy(feat).to(dev), torch.from_numpy(boxes).to(dev), d_k, OFF_X, OFF_Y, SSCALE)
    got = got.cpu().numpy()[0, :n].astype(np.float64)

    xs, ys = O.gen_sample_grid(torch.from_numpy(b7[:, [0, 1, 3, 4, 6]]), grid_offsets=(OFF_X, OFF_Y),
                               spatial_scale=SSCALE)
    ref32 = O.bilinear_gridsample(torch.from_numpy(feat[0]).permute(2, 0, 1).contiguous(), xs, ys)
    ref32 = ref32.mean(0).view(-1).numpy().astype(np.float64)
    x32, y32 = xs.numpy(), ys.numpy()
    ref64, S = _pswarp_ref64(feat[0].astype(np.float64), x32, y32)
    # the construction reaches what it claims to
    e = np.r_[0:ne, late:late + ne]
    ex, ey = x32[:, e], y32[:, e]
    assert np.any((ex == W - 1) & (ey == H - 1)) and np.sum(ex == np.floor(ex)) >= 28 * 20, "pixel centres"
    assert np.any((ex > W - 2) & (ex < W - 1)) and np.any((ey > H - 2) & (ey < H - 1)), "last-column / row strips"
    assert np.any((ex > -1) & (ex < 0)) and np.any((ex > W - 1) & (ex < W)) and np.any((ey > H - 1) & (ey < H))
    off = np.all((x32 <= -1) | (x32 >= W) | (y32 <= -1) | (y32 >= H), 0)
    assert off[e].sum() >= 2 * 6 and np.all(S[off] == 0)
    tol = C_PS * EPS32 * S
    assert np.all(np.abs(ref32 - ref64) <= tol), "the bound does not hold for the reference's own fp32 path"
    err = np.abs(got - ref64)
    assert np.all(err <= tol), "PSWarp: worst error %g at box %d (tol %g)" % (err.max(), err.argmax(), tol[err.argmax()])
    assert np.all(got[off] == 0.0)                  # wholly off the map: exactly 0
    print("pswarp: max |err| / (eps S) = %.1f (bound %d); fp32 reference %.1f" %
          ((err / (EPS32 * np.maximum(S, 1e-30))).max(), C_PS, (np.abs(ref32 - ref64) / (EPS32 * np.maximum(S, 1e-30))).max()))


# ====================================================================== 3. rescoring + sort + NMS (sassd_rescore_nms)
CELL = 9.0                                       # scene cells [m]: nothing reaches into a neighbouring cell


def _wrap(r):
    return (r + np.pi) % (2 * np.pi) - np.pi


def _bev(b7):
    return O.boxes3d_to_bev(torch.from_numpy(np.ascontiguousarray(b7, np.float32))).numpy()


def _car(rs, m):
    return 1.6 + rs.normal(0, 0.05, m), 3.9 + rs.normal(0, 0.1, m)


def _cluster(rs, cx, cy, tight, yaw_pi2):
    """An object's overlapping anchors: 20-80 boxes within +-0.3 m / +-0.2 rad of a car box (tight), or 20-40 within
    +-1.5 m / +-0.6 rad; a few exact duplicates; optionally yaw near +-pi/2, where w and l swap in BEV.  Redrawn until
    every pair's oracle IoU is more than 1e-4 from the 0.1 threshold."""
    m = rs.randint(20, 81) if tight else rs.randint(20, 41)
    dxy, dr = (0.3, 0.2) if tight else (1.5, 0.6)
    for _ in range(200):
        yaw0 = (rs.choice([np.pi / 2, -np.pi / 2]) + rs.uniform(-1e-3, 1e-3)) if yaw_pi2 else rs.uniform(-np.pi, np.pi)
        w, l = _car(rs, m)
        b = np.stack([cx + rs.uniform(-dxy, dxy, m), cy + rs.uniform(-dxy, dxy, m), rs.uniform(-1.8, -1.5, m), w, l,
                      np.full(m, 1.56), _wrap(yaw0 + rs.uniform(-dr, dr, m))], 1).astype(np.float32)
        dup = rs.choice(m, 4, replace=False)
        b[dup[1]] = b[dup[0]]
        b[dup[3]] = b[dup[2]]
        iou = O.iou_matrix(_bev(b))
        if np.abs(iou[~np.eye(m, dtype=bool)] - IOU_THR).min() > 1e-4:
            return b
    raise AssertionError("could not draw a decisive cluster")


def _touching_pair(rs, cx, cy, k):
    """Two car boxes edge to edge (gap 0, a few 1e-5 m either way), side by side or end to end, axis-aligned or
    rotated."""
    w, l = _car(rs, 1)
    w, l = float(w[0]), float(l[0])
    gap = (0.0, 1e-5, 3e-5, -1e-5, 5e-5)[k % 5]
    a = 0.0 if k % 2 == 0 else rs.uniform(-np.pi, np.pi)
    # BEV x extent is column 3, y extent column 4; spin() maps the box's x axis to (cos a, -sin a)
    if (k // 2) % 2 == 0:
        d, u = w + gap, np.array([np.cos(a), -np.sin(a)])
    else:
        d, u = l + gap, np.array([np.sin(a), np.cos(a)])
    c0 = np.array([cx, cy]) - u * d / 2
    c1 = c0 + u * d
    return np.array([[c0[0], c0[1], -1.6, w, l, 1.56, a], [c1[0], c1[1], -1.6, w, l, 1.56, a]], np.float32)


def _tip_pair(rs, cx, cy, k):
    """Two rotated boxes whose corners point at each other along the line between their centres, overlapping by eps
    (or apart): the centre distance is within eps of the sum of the circumscribed radii, the edge of the NMS's
    circumscribed-circle shortcut."""
    eps = (-1e-3, 1e-4, 1e-3, 1e-2, 5e-2)[k % 5]
    (wa, wb), (la, lb) = _car(rs, 2)
    phi = rs.uniform(-np.pi, np.pi)
    ra, rb = np.hypot(wa / 2, la / 2), np.hypot(wb / 2, lb / 2)
    aa = _wrap(np.arctan2(la / 2, wa / 2) - phi)       # corner (+w/2, +l/2) of A along +phi
    ab = _wrap(np.arctan2(lb / 2, wb / 2) - phi)       # corner (-w/2, -l/2) of B along -phi
    d = ra + rb - eps
    u = np.array([np.cos(phi), np.sin(phi)])
    c0 = np.array([cx, cy]) - u * d / 2
    c1 = c0 + u * d
    return np.array([[c0[0], c0[1], -1.6, wa, la, 1.56, aa], [c1[0], c1[1], -1.6, wb, lb, 1.56, ab]], np.float32)


def _scene(n, seed):
    """n BEV-disjoint groups: clusters (tight, loose, yaw near +-pi/2), touching pairs and corner-to-corner pairs, one
    group per 9 m cell, shuffled into candidate order."""
    rs = np.random.RandomState(seed)
    g = np.arange(14) * CELL
    cells = [(x, y) for x in g + 4.5 for y in g - 63.0]
    rs.shuffle(cells)
    parts, have = [], 0
    for i, (cx, cy) in enumerate(cells):
        if have >= n:
            break
        kind = i % 6
        if kind == 0:
            p = _touching_pair(rs, cx, cy, i // 6)
        elif kind == 1:
            p = _tip_pair(rs, cx, cy, i // 6)
        else:
            p = _cluster(rs, cx, cy, tight=kind < 4, yaw_pi2=kind == 5)
        parts.append(p)
        have += len(p)
    assert have >= n, "scene grid too small"
    b7 = np.concatenate(parts)[:n]
    return b7[rs.permutation(n)]


_GRID = (-0.8 + 1e-3 * np.arange(5000)).astype(np.float32)    # distinct logits: sigmoid gaps >= 1.4e-5 >> fp32 ulp


def _pass_logits(n, mode, rs):
    if mode == "all0":
        return np.zeros(n, np.float32)
    if mode == "blocks":                         # runs of equal logits
        return rs.choice(_GRID[rs.permutation(len(_GRID))[:max(1, n // 8)]], n)
    return _GRID[rs.permutation(len(_GRID))[:n]]


def _frame(n_pass, n_below, mode, seed):
    """candidates (boxes [K,7], logits [K], labels [K]) with n_pass above the 0.3 score threshold and n_below below it,
    interleaved in candidate order"""
    rs = np.random.RandomState(seed)
    b = _scene(n_pass, seed) if n_pass else np.zeros((0, 7), np.float32)
    lp = _pass_logits(n_pass, mode, rs)
    below = np.stack([rs.uniform(0, 120, n_below), rs.uniform(-60, 60, n_below), np.full(n_below, -1.6),
                      rs.uniform(1, 2, n_below), rs.uniform(3, 4, n_below), np.full(n_below, 1.5),
                      rs.uniform(-3, 3, n_below)], 1).astype(np.float32)
    lb = rs.uniform(-6, -0.9, n_below).astype(np.float32)
    order = rs.permutation(n_pass + n_below)
    boxes = np.concatenate([b, below])[order]
    logits = np.concatenate([lp, lb])[order]
    labels = rs.randint(0, 3, n_pass + n_below).astype(np.int32)
    return boxes, logits, labels


def _run_rescore(dev, frames, k_cap, det_cap, iou_thr=IOU_THR):
    from sassd_b200 import ops
    B = len(frames)
    boxes = np.zeros((B, k_cap, 7), np.float32)
    scores = np.zeros((B, k_cap), np.float32)
    labels = np.zeros((B, k_cap), np.int32)
    for b, (bx, lg, lb) in enumerate(frames):
        boxes[b, :len(bx)], scores[b, :len(bx)], labels[b, :len(bx)] = bx, lg, lb
        # the score threshold is never decided within libm's error
        assert len(lg) == 0 or np.abs(_sig64(lg) - SCORE_THR).min() >= MARGIN
    d_k = torch.tensor([len(f[0]) for f in frames], dtype=torch.int32, device=dev)
    status = torch.zeros((1,), dtype=torch.int32, device=dev)
    det, nd = ops.rescore_nms(torch.from_numpy(boxes).to(dev), torch.from_numpy(scores).to(dev),
                              torch.from_numpy(labels).to(dev), d_k, SCORE_THR, iou_thr, det_cap, status)
    return det.cpu().numpy(), nd.cpu().numpy(), int(status.item())


def _oracle(bx, lg, lb):
    e = O.get_rescore_bboxes([torch.from_numpy(bx)], [torch.from_numpy(lg)], [torch.from_numpy(lb).long()],
                             SCORE_THR, IOU_THR)
    return e[0][0], e[1][0], e[2][0]


def _decisive(bx, lg):
    """min |IoU - thr| over every pair of score-passing candidates (oracle IoU, host libm, no FMA): the kept set is
    only decided identically by the oracle when this exceeds 1e-5 (the rule of test_nms_mask_and_keep)"""
    p = _sig64(lg) > SCORE_THR
    if p.sum() < 2:
        return 1.0
    iou = O.iou_matrix(_bev(bx[p]))
    return float(np.abs(iou[~np.eye(int(p.sum()), dtype=bool)] - IOU_THR).min())


def _check_frame(det, nd, exp, tag, rows=None):
    eb, es, el = exp
    if eb is None:
        assert nd == 0, tag
        return
    rows = len(eb) if rows is None else rows
    assert nd == rows, "%s: %d detections, oracle %d" % (tag, nd, rows)
    # kept set and order, boxes and labels bit for bit; scores: CUDA expf vs torch's sigmoid, 1e-6
    assert np.array_equal(det[:nd, :7], eb[:rows]), "%s: kept boxes / order differ" % tag
    assert np.array_equal(det[:nd, 8].astype(np.int64), el[:rows]), "%s: labels" % tag
    assert np.abs(det[:nd, 7] - es[:rows]).max() <= 1e-6, "%s: scores" % tag


# (candidates above 0.3, candidates below it, logit mode)
RESCORE_FRAMES = [(0, 0, "distinct"), (0, 40, "distinct"), (1, 3, "distinct"), (63, 5, "distinct"), (64, 0, "all0"),
                  (65, 7, "blocks"), (1023, 200, "distinct"), (1024, 0, "blocks"), (1025, 300, "all0"),
                  (2048, 500, "blocks"), (4095, 700, "distinct"), (4096, 800, "blocks"), (300, 30, "all0"),
                  (500, 50, "blocks"), (129, 10, "distinct"), (2, 2, "all0")]


def test_rescore_nms_batch16_at_the_capacities(dev):
    """B = 16 in one launch, candidate counts 0 .. 4096 (the compaction's second 1024-wide pass, the bitonic sort past
    1024 keys, up to all 64 column blocks of the [4096][64] mask), clustered / touching / degenerate scenes, tied
    scores: detections equal get_rescore_bboxes' in kept set, order, boxes and labels, bit for bit."""
    frames = [_frame(p, q, m, 1000 + i) for i, (p, q, m) in enumerate(RESCORE_FRAMES)]
    det, nd, status = _run_rescore(dev, frames, K_CAP, NMS_CAP)
    assert status == 0                          # 4096 passers is exactly the cap; det_cap 4096 cannot overflow
    decisive = 0
    for b, (bx, lg, lb) in enumerate(frames):
        tag = "frame %d (%d candidates, %s)" % (b, RESCORE_FRAMES[b][0], RESCORE_FRAMES[b][2])
        margin = _decisive(bx, lg)
        assert margin > 1e-5, "%s: min |IoU - thr| = %g" % (tag, margin)
        decisive += 1
        _check_frame(det[b], nd[b], _oracle(bx, lg, lb), tag)
    assert decisive == len(frames)              # the scenes are built so that every frame is decisive


def test_rescore_nms_cap_keeps_the_first_4096_passers(dev):
    """More than 4096 candidates pass: NMS_CAP is raised and the NMS runs on the first 4096 passers in candidate
    order, exactly; the other frame of the launch is unaffected."""
    big, small = _frame(5000, 500, "blocks", 2001), _frame(100, 10, "distinct", 2002)
    det, nd, status = _run_rescore(dev, [big, small], K_CAP, NMS_CAP)
    assert status == FLAG_NMS_CAP
    bx, lg, lb = big
    passers = np.nonzero(_sig64(lg) > SCORE_THR)[0]
    cut = passers[NMS_CAP - 1] + 1              # candidates up to and including the 4096th passer
    pre = (bx[:cut], lg[:cut], lb[:cut])
    assert _decisive(*pre[:2]) > 1e-5
    _check_frame(det[0], nd[0], _oracle(*pre), "NMS_CAP frame")
    _check_frame(det[1], nd[1], _oracle(*small), "frame beside it")


def _disjoint_frame(n, seed):
    """n mutually disjoint car boxes (6 m grid), distinct scores: every one is kept"""
    rs = np.random.RandomState(seed)
    side = int(np.ceil(np.sqrt(n)))
    gx, gy = np.meshgrid(np.arange(side) * 6.0, np.arange(side) * 6.0 - 60.0)
    w, l = _car(rs, n)
    bx = np.stack([gx.ravel()[:n], gy.ravel()[:n], np.full(n, -1.6), w, l, np.full(n, 1.56),
                   rs.uniform(-np.pi, np.pi, n)], 1).astype(np.float32)
    return bx, _pass_logits(n, "distinct", rs), rs.randint(0, 3, n).astype(np.int32)


def test_rescore_nms_det_cap(dev):
    """512 kept with det_cap 512: no flag; 600 kept: DET_CAP, ndet == det_cap and the rows are the oracle's first 512
    in score order."""
    f512, f600 = _disjoint_frame(512, 3001), _disjoint_frame(600, 3002)
    det, nd, status = _run_rescore(dev, [f512], 1024, 512)
    assert status == 0 and nd[0] == 512
    _check_frame(det[0], nd[0], _oracle(*f512), "512 kept")
    det, nd, status = _run_rescore(dev, [f600, f512], 1024, 512)
    assert status == FLAG_DET_CAP
    exp = _oracle(*f600)
    assert len(exp[0]) == 600
    _check_frame(det[0], nd[0], exp, "600 kept", rows=512)
    _check_frame(det[1], nd[1], _oracle(*f512), "512 kept beside it")


# ====================================================================== 4. NMS bitmask vs the reference kernel
TAIL_NMS_CASES = [2048, 4095, 4096]
TAIL_NMS_THRS = [0.1, 0.0]
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libiou3d_ref.so")


def tail_nms_inputs(n):
    """(candidate boxes [n,7], logits [n], labels [n], score-sorted BEV boxes [n,5], sort order) of the clustered scene
    of n candidates, all above the score threshold, distinct scores (tests/golden/make_golden_nms.py stores the
    reference kernel's masks of these BEV boxes)"""
    bx, lg, lb = _frame(n, 0, "distinct", 4000 + n)
    order = torch.sort(torch.sigmoid(torch.from_numpy(lg)), descending=True, stable=True)[1].numpy()
    return bx, lg, lb, np.ascontiguousarray(_bev(bx[order])), order


def bev_digest(bev):
    """sha256 of the sorted BEV boxes' fp32 bytes: the committed masks name their inputs by it"""
    return hashlib.sha256(np.ascontiguousarray(bev, np.float32).tobytes()).hexdigest()


def pack_reference_mask(mask):
    """reference bitmask [n, colb] uint64 -> lzma-compressed bytes (uint8 array) of its upper triangle (column block >=
    row block, the only words the NMS reads; the reference kernel also fills the lower blocks)"""
    n, colb = mask.shape
    upper = np.arange(colb)[None, :] >= (np.arange(n) // 64)[:, None]
    words = np.where(upper, mask, np.uint64(0)).astype("<u8")
    return np.frombuffer(lzma.compress(words.tobytes(), preset=9 | lzma.PRESET_EXTREME), np.uint8)


def unpack_reference_mask(packed, n):
    return np.frombuffer(lzma.decompress(packed.tobytes()), "<u8").astype(np.uint64).reshape(n, (n + 63) // 64)


def _ref_sweep(mask, n):
    """the reference's host sweep over its bitmask (iou3d.cpp, nms_gpu): indices into the sorted list"""
    remv = np.zeros(mask.shape[1], np.uint64)
    keep = []
    for i in range(n):
        nb, ib = divmod(i, 64)
        if not (int(remv[nb]) >> ib) & 1:
            keep.append(i)
            remv[nb:] |= mask[i, nb:]
    return np.asarray(keep, np.int64)


def _check_mask_and_keep(dev, n, thr, rmask, inputs):
    from sassd_b200 import ops
    bx, lg, lb, bev, order = inputs
    colb = (n + 63) // 64
    upper = np.arange(colb)[None, :] >= (np.arange(n) // 64)[:, None]      # column block >= row block
    got = ops.nms_mask(torch.from_numpy(bev).to(dev), thr).cpu().numpy().view(np.uint64)
    bad = np.nonzero(upper & (got != rmask))
    assert bad[0].size == 0, "n=%d thr=%g: %d mask words differ from the reference kernel, first at row %d block %d" % (
        n, thr, bad[0].size, bad[0][0], bad[1][0])
    # the fused path (rescore + sort + [4096][64] mask + device sweep) keeps what the reference sweep keeps
    keep = _ref_sweep(rmask, n)
    det, nd, status = _run_rescore(dev, [(bx, lg, lb)], n, NMS_CAP, iou_thr=thr)
    assert status == 0 and nd[0] == len(keep), (status, nd[0], len(keep))
    assert np.array_equal(det[0, :nd[0], :7], bx[order[keep]])
    if thr == 0.0:
        # the scene reaches the circumscribed-circle shortcut's edge: overlapping pairs whose centre distance is
        # above 0.9 of the sum of the radii
        i, j = np.nonzero(np.unpackbits(rmask.view(np.uint8), axis=1, bitorder="little")[:, :n])
        i, j = i[j > i], j[j > i]
        c = 0.5 * (bev[:, :2] + bev[:, 2:4]).astype(np.float64)
        rad = 0.5 * np.hypot(bev[:, 2] - bev[:, 0], bev[:, 3] - bev[:, 1]).astype(np.float64)
        d2 = ((c[i] - c[j]) ** 2).sum(1)
        assert np.sum(d2 > 0.9 * (rad[i] + rad[j]) ** 2) >= 5


def _ref_launcher():
    if not os.path.isfile(REF_LIB):
        pytest.skip("oracle/_ref/libiou3d_ref.so absent: build() compiles the reference NMS kernel only when the "
                    "original project is checked out beside this one (the committed masks are checked regardless)")
    fn = getattr(ctypes.CDLL(REF_LIB), "_Z11nmsLauncherPKfPyif")
    fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_float]
    fn.restype = None
    return fn


@pytest.mark.parametrize("thr", TAIL_NMS_THRS)
@pytest.mark.parametrize("n", TAIL_NMS_CASES)
def test_nms_mask_matches_reference_kernel_live(dev, n, thr):
    """ops.nms_mask vs the unmodified reference nmsLauncher on clustered scenes at the cap, bit for bit (upper
    triangle), and the fused path's kept set vs the reference sweep over the reference mask."""
    fn = _ref_launcher()
    inputs = tail_nms_inputs(n)
    d_bev = torch.from_numpy(inputs[3]).to(dev)
    rmask = torch.zeros((n, (n + 63) // 64), dtype=torch.int64, device=dev)
    torch.cuda.synchronize()
    fn(ctypes.c_void_p(d_bev.data_ptr()), ctypes.c_void_p(rmask.data_ptr()), n, ctypes.c_float(thr))
    torch.cuda.synchronize()
    _check_mask_and_keep(dev, n, thr, rmask.cpu().numpy().view(np.uint64), inputs)


@pytest.mark.parametrize("thr", TAIL_NMS_THRS)
@pytest.mark.parametrize("n", TAIL_NMS_CASES)
def test_nms_mask_matches_committed_reference_masks(dev, golden_dir, n, thr):
    """The same check against the reference kernel's masks committed in tests/golden/nms_ref.npz."""
    ref = np.load(os.path.join(golden_dir, "nms_ref.npz"))
    inputs = tail_nms_inputs(n)
    assert bev_digest(inputs[3]) == str(ref["tail_bev_sha256_%d" % n]), "the scene differs from the masks' inputs"
    _check_mask_and_keep(dev, n, thr, unpack_reference_mask(ref["tail_mask_%d_%g" % (n, thr)], n), inputs)


# ====================================================================== 5. flags and status through the real step
def _model(dev, bias_shift=0.0, zero_pswarp=False):
    from sassd_b200 import checkpoint
    from tests.test_gpu_parity import _make_model
    model, sd = _make_model(dev)
    sd = dict(sd)
    if bias_shift:
        sd["rpn_head.conv_cls.bias"] = sd["rpn_head.conv_cls.bias"] + bias_shift
    if zero_pswarp:
        sd["extra_head.convs.3.weight"] = torch.zeros_like(sd["extra_head.convs.3.weight"])
    checkpoint.load_state_dict_into(model, sd)
    return model, sd


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert (x["boxes_lidar"] is None) == (y["boxes_lidar"] is None)
        if y["boxes_lidar"] is not None:
            for k in ("boxes_lidar", "scores", "label_preds"):
                np.testing.assert_array_equal(x[k], y[k])


def test_tied_pswarp_scores_through_the_step(dev):
    """A zero PSWarp 1x1 conv gives every guided anchor logit 0 (score 0.5, all tied) and a class bias +0.5 some 2000
    guided anchors: the kept order is candidate order, as in the oracle's stable sort."""
    from tests.test_gpu_parity import _check_against_oracle
    model, sd = _model(dev, bias_shift=0.5, zero_pswarp=True)
    clouds = [synth_cloud(9)]
    _, aux = model.forward_points(clouds, return_aux=True)
    k = int(aux["d_k"][0])
    assert 1025 <= k <= NMS_CAP, k
    assert np.all(aux["ps_scores"][0, :k].cpu().numpy() == 0.0)
    _check_against_oracle(model, sd, clouds, "tied scores", min_total=10)


def test_guided_cap_raises_and_status_resets(dev):
    """A frame with more guided anchors than k_cap raises SassdError(GUIDED_CAP) eagerly, from the captured step and
    from detect_stream; the next normal frame through the same graph / slot gives the eager detections."""
    from sassd_b200.lib import SassdError
    model, _ = _model(dev)
    small, big = [synth_cloud(9)], [synth_cloud(1)]
    maxpts = max(small[0].shape[0], big[0].shape[0])
    ks = int(model.forward_points(small, return_aux=True)[1]["d_k"][0])
    kb = int(model.forward_points(big, return_aux=True)[1]["d_k"][0])
    assert 0 < ks < kb, (ks, kb)
    model.rpn_head.k_cap = ks                    # the small frame sits exactly at the cap: no flag
    ref = model.forward_points(small)
    with pytest.raises(SassdError, match="GUIDED_CAP"):
        model.forward_points(big)
    _same(model.forward_points(small), ref)
    model.enable_cuda_graph(1, maxpts)
    try:
        _same(model.forward_points(small), ref)
        with pytest.raises(SassdError, match="GUIDED_CAP"):
            model.forward_points(big)
        _same(model.forward_points(small), ref)      # the replay resets the status word
        with pytest.raises(SassdError, match="GUIDED_CAP"):
            list(model.detect_stream([big, small], 1, maxpts, depth=1))
        _same(list(model.detect_stream([small], 1, maxpts, depth=1))[0], ref)   # same slot, next batch
    finally:
        model.disable_cuda_graph()


def test_nms_cap_raises_through_the_step(dev):
    """Class bias +0.72 gives ~6000 guided anchors (below k_cap 8192), all at score 0.5 with a zero PSWarp conv:
    NMS_CAP is raised eagerly, from the captured step and from detect_stream."""
    from sassd_b200.lib import SassdError
    model, _ = _model(dev, bias_shift=0.72, zero_pswarp=True)
    frame = [synth_cloud(9)]
    with pytest.raises(SassdError, match="NMS_CAP") as e:
        model.forward_points(frame)
    assert "GUIDED_CAP" not in str(e.value)
    model.enable_cuda_graph(1, 32768)
    try:
        with pytest.raises(SassdError, match="NMS_CAP"):
            model.forward_points(frame)
        with pytest.raises(SassdError, match="NMS_CAP"):
            list(model.detect_stream([frame], 1, 32768, depth=1))
    finally:
        model.disable_cuda_graph()
