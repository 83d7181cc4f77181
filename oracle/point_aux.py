"""ORACLE — test infrastructure only.

numpy / torch-CPU restatement of SA-SSD's auxiliary point-wise network in eval mode
(mmdet/models/necks/cmn.py:121-135, :175-189):

* ``tensor2points`` — mmdet/core/bbox/transforms.py:218-223 in fp32, each operation rounded;
* ``three_nn`` — pointnet2 three_nn (mmdet/ops/pointnet2/src/interpolate_gpu.cu:9-56): per unknown row the three
  smallest (d, known row) pairs in lexicographic order among the known rows of the same batch index, with
  d = fma(dz, dz, fma(dx, dx, dy * dy)) in fp32 (the SASS of that kernel for sm_90a); missing slots are idx 0,
  dist2 +inf (the reference's 1e40 as fp32);
* ``interpolate_weights`` / ``three_interpolate`` — pointnet2_utils.py:31, cmn.py:184-186, interpolate_gpu.cu:80-102;
* ``point_head`` — point_fc (no activation), point_cls, point_reg on cat([p0, p1, p2]);
* ``vxnet_middle`` — the ``middle`` list of VxNet.forward (cmn.py:214-231): conv1, conv2, conv3 outputs, from the
  building blocks of oracle/ref_pipeline.py.

The reference's loop is quadratic; ``three_nn`` gets its candidates from a k-d tree in fp64 and then decides among
every candidate that fp32 rounding could still place in the top three with the reference's own arithmetic.
"""
import numpy as np
import torch
from scipy.spatial import cKDTree

from . import ref_pipeline as _rp

OFFSET = (0.0, -40.0, -3.0)                                   # literals of cmn.py:122-129
LEVEL_VOXEL_SIZES = ((0.1, 0.1, 0.2), (0.2, 0.2, 0.4), (0.4, 0.4, 0.8))


def fma32(a, b, c):
    """fp32 fused multiply-add, correctly rounded: the fp64 product of two fp32 values is exact; the fp64 sum is
    rounded to odd (TwoSum error + parity fix) so that the final rounding to fp32 is not a double rounding."""
    p = np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32).astype(np.float64)
    cc = np.asarray(c, np.float32).astype(np.float64)
    p, cc = np.broadcast_arrays(p, cc)
    s = p + cc
    bb = s - p
    e = (p - (s - bb)) + (cc - bb)
    fix = (e != 0) & np.isfinite(s) & ((s.view(np.int64) & 1) == 0)
    if np.any(fix):
        s = s.copy()
        s[fix] = np.nextafter(s[fix], np.where(e[fix] > 0, np.inf, -np.inf))
    return s.astype(np.float32)


def sq_dist32(u, k):
    """u [..., 3], k [..., 3] fp32 -> fma(dz, dz, fma(dx, dx, dy * dy)) in fp32."""
    d = (np.asarray(u, np.float32) - np.asarray(k, np.float32)).astype(np.float32)
    return fma32(d[..., 2], d[..., 2], fma32(d[..., 0], d[..., 0], (d[..., 1] * d[..., 1]).astype(np.float32)))


def tensor2points(coords, voxel_size, offset=OFFSET):
    """coords [M,4] int (b,z,y,x) -> [M,4] fp32 (b, x, y, z) voxel centres: idx * vs + offset + 0.5 * vs."""
    c = np.asarray(coords)
    vs = np.asarray(voxel_size, np.float32)
    off = np.asarray(offset, np.float32)
    idx = c[:, [3, 2, 1]].astype(np.float32)
    out = np.empty((c.shape[0], 4), np.float32)
    out[:, 0] = c[:, 0].astype(np.float32)
    out[:, 1:] = ((idx * vs).astype(np.float32) + off).astype(np.float32) + (np.float32(0.5) * vs).astype(np.float32)
    return out


def _top3(u, kx, kidx, cand):
    """Lexicographic (d, row) top three of the unknown points u [n,3] among their candidate rows cand [n,c] (indices
    into kx, -1 = none): returns (idx [n,3], dist2 [n,3]) with the reference's sentinels."""
    n = u.shape[0]
    ok = cand >= 0
    c = np.where(ok, cand, 0)
    d = sq_dist32(u[:, None, :], kx[c])
    ok &= d < np.float32(np.inf)                         # the reference never inserts d = inf or NaN
    rows = np.where(ok, kidx[c], np.iinfo(np.int32).max)
    d = np.where(ok, d, np.float32(np.inf))
    o = np.argsort(rows, axis=1, kind="stable")
    rows, d, ok = (np.take_along_axis(a, o, 1) for a in (rows, d, ok))
    o = np.argsort(d, axis=1, kind="stable")[:, :3]
    rows, d, ok = (np.take_along_axis(a, o, 1) for a in (rows, d, ok))
    idx = np.zeros((n, 3), np.int32)
    dist2 = np.full((n, 3), np.inf, np.float32)
    k = min(3, o.shape[1])
    idx[:, :k] = np.where(ok, rows, 0)[:, :k]
    dist2[:, :k] = np.where(ok, d, np.float32(np.inf))[:, :k]
    return idx, dist2


def three_nn(unknown, known, k_query=8):
    """unknown [N,4], known [M,4] fp32 (b, x, y, z).  Returns (idx [N,3] int32 global known rows, dist2 [N,3] fp32)."""
    unknown = np.asarray(unknown, np.float32)
    known = np.asarray(known, np.float32)
    n = unknown.shape[0]
    idx = np.zeros((n, 3), np.int32)
    dist2 = np.full((n, 3), np.inf, np.float32)
    for b in np.unique(unknown[:, 0]):
        ui = np.nonzero(unknown[:, 0] == b)[0]
        ki = np.nonzero(known[:, 0] == b)[0].astype(np.int32)
        if ki.size == 0:
            continue
        kx = known[ki, 1:]
        ux = unknown[ui, 1:]
        tree = cKDTree(kx.astype(np.float64))
        kq = min(k_query, ki.size)
        r, cand = tree.query(ux.astype(np.float64), k=kq)
        r, cand = np.asarray(r).reshape(ui.size, kq), np.asarray(cand).reshape(ui.size, kq)
        # fp32 rounding moves a squared distance by a few ulp: every row within 1e-5 relative (plus an absolute margin
        # for tiny distances) of the third-nearest fp64 distance may still rank in the fp32 top three
        bound = r[:, min(2, kq - 1)] * (1.0 + 1e-5) + 1e-6
        cand = np.where(r <= bound[:, None], cand, -1)
        idx[ui], dist2[ui] = _top3(ux, kx, ki, cand)
        short = np.nonzero((kq < ki.size) & (r[:, -1] <= bound))[0]    # candidates beyond the k queried
        for j in short:
            ball = np.asarray(tree.query_ball_point(ux[j].astype(np.float64), bound[j]), np.int64)
            idx[ui[j]], dist2[ui[j]] = (a[0] for a in _top3(ux[j:j + 1], kx, ki, ball[None, :]))
    return idx, dist2


def interpolate_weights(dist2):
    """dist = sqrt(dist2); 1 / (dist + 1e-8) normalised by its sum over the three slots (fp32)."""
    dist = np.sqrt(np.asarray(dist2, np.float32)).astype(np.float32)
    with np.errstate(divide="ignore"):
        recip = (np.float32(1.0) / (dist + np.float32(1e-8)).astype(np.float32)).astype(np.float32)
    norm = ((recip[:, 0] + recip[:, 1]).astype(np.float32) + recip[:, 2]).astype(np.float32)
    return (recip / norm[:, None]).astype(np.float32)


def three_interpolate(feats, idx, weight):
    """feats [M,C], idx / weight [N,3] -> [N,C] = fma(w2, p2, fma(w1, p1, w0 * p0)) (interpolate_gpu.cu:80-102)."""
    f = np.asarray(feats, np.float32)
    w = np.asarray(weight, np.float32)
    if f.shape[0] == 0:
        return np.zeros((idx.shape[0], f.shape[1]), np.float32)
    p0, p1, p2 = f[idx[:, 0]], f[idx[:, 1]], f[idx[:, 2]]
    return fma32(w[:, 2:3], p2, fma32(w[:, 1:2], p1, (w[:, 0:1] * p0).astype(np.float32)))


def point_head(sd, points_mean, middle, prefix="neck."):
    """points_mean [N,4] (b, x, y, z); middle: three (features [M_l, C_l], coords [M_l,4]) of conv1, conv2, conv3.
    Returns dict(cls [N,1], reg [N,3], idx / dist2 [N,3,3] per level)."""
    ps, idxs, d2s = [], [], []
    for (feats, coords), vs in zip(middle, LEVEL_VOXEL_SIZES):
        known = tensor2points(coords, vs)
        idx, dist2 = three_nn(points_mean, known)
        w = interpolate_weights(dist2)
        ps.append(three_interpolate(np.asarray(feats, np.float32), idx, w))
        idxs.append(idx)
        d2s.append(dist2)
    x = torch.from_numpy(np.concatenate(ps, axis=1))
    pw = x @ sd[prefix + "point_fc.weight"].float().t()
    cls = pw @ sd[prefix + "point_cls.weight"].float().t()
    reg = pw @ sd[prefix + "point_reg.weight"].float().t()
    return dict(cls=cls.numpy(), reg=reg.numpy(), idx=np.stack(idxs, 1), dist2=np.stack(d2s, 1))


def vxnet_middle(sd, feats, coords, shape, prefix="neck.backbone."):
    """VxNet.forward up to conv3 (cmn.py:214-229), as ref_pipeline.vxnet_forward computes it: feats [N,4] f32, coords
    [N,4] (b,z,y,x).  Returns ``middle``: three (features, coords) after conv1, conv2 and conv3."""
    x = torch.as_tensor(feats, dtype=torch.float32)
    coords = np.asarray(coords, np.int32)
    shape = list(shape)
    middle = []
    nbr_subm = None
    for block, idxs, kind, key in _rp.VXNET_PLAN:
        if kind == "down":
            coords_out, nbr, shape_out = _rp.sparse_conv_rulebook(coords, shape)
            w = sd["%s%s.0.weight" % (prefix, block)]
            x = _rp.indice_conv(x, w.reshape(27, w.shape[3], w.shape[4]), nbr)
            x = torch.relu(_rp.bn_eval(x, sd, "%s%s.1" % (prefix, block)))
            coords, shape = coords_out, shape_out
            nbr_subm = None
        else:
            if nbr_subm is None:
                nbr_subm = _rp.subm_rulebook(coords, shape)
            for i in idxs:
                w = sd["%s%s.%d.weight" % (prefix, block, i)]
                x = _rp.indice_conv(x, w.reshape(27, w.shape[3], w.shape[4]), nbr_subm)
                x = torch.relu(_rp.bn_eval(x, sd, "%s%s.%d" % (prefix, block, i + 1)))
            if key > 0:
                middle.append((x, coords))
    return middle
