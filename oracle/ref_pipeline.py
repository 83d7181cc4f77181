"""ORACLE — test infrastructure only.

CPU restatement (numpy / torch-CPU fp32) of the SA-SSD inference hot path, one
function per reference function, each citing the reference file:line it
follows.  Nothing under ``sa-ssd_b200/`` imports this module; only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs do, and only as the checker / the timed CPU arm.

Pinning status (see DESIGN.md §Oracle):
  * voxelizer, SimpleVoxel, BEVNet, SSDRotateHead (+decode, guided anchors),
    PSWarpHead (+grid, sampling), anchors, anchors_mask: pinned against the
    reference's own Python executed in the build container
    (tests/golden/make_golden.py -> tests/golden/*.npz, tests/test_oracle_golden.py).
  * sparse backbone (spconv v1.0, traveller59/spconv tag v1.0, readme.md:58):
    third-party, NOT vendored under /root/reference, reference holds no tests
    for it  ->  "parity unpinned" by the reference; pinned here BY DEFINITION
    against torch.nn.functional.conv3d on the densified tensor
    (tests/test_oracle_spconv.py), following SURVEY.md §A.2.
  * rotated NMS: reference is CUDA-only; CPU restatement in oracle/nms.c, and on
    the GPU box the unmodified reference kernel built into oracle/_ref/.
"""
import ctypes
import os

import numpy as np
import torch
import torch.nn.functional as F

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def lib():
    """Load (building if needed) oracle/liboracle.so (voxelize.c + nms.c)."""
    global _LIB
    if _LIB is None:
        from . import build as _build
        path = _build.build_oracle()
        L = ctypes.CDLL(path)
        L.oracle_points_to_voxel.restype = ctypes.c_int
        L.oracle_nms_sorted.restype = ctypes.c_int
        L.oracle_nms_greedy.restype = ctypes.c_int
        L.oracle_iou_bev.restype = ctypes.c_float
        L.oracle_box_overlap.restype = ctypes.c_float
        _LIB = L
    return _LIB


def _p(a, t):
    return a.ctypes.data_as(ctypes.POINTER(t))


# --------------------------------------------------------------------------
# a1  voxelizer — points_ops.py:4-50,104-164 (via oracle/voxelize.c)
# --------------------------------------------------------------------------
def points_to_voxel(points, voxel_size, coors_range, max_points=5, max_voxels=20000):
    points = np.ascontiguousarray(points, dtype=np.float32)
    vs = np.ascontiguousarray(voxel_size, dtype=np.float32)
    rg = np.ascontiguousarray(coors_range, dtype=np.float32)
    n, ndim = points.shape
    voxels = np.zeros((max_voxels, max_points, ndim), np.float32)
    coors = np.zeros((max_voxels, 3), np.int32)
    num = np.zeros((max_voxels,), np.int32)
    m = lib().oracle_points_to_voxel(_p(points, ctypes.c_float), n, ndim, _p(vs, ctypes.c_float),
                                     _p(rg, ctypes.c_float), int(max_points), int(max_voxels),
                                     _p(voxels, ctypes.c_float), _p(coors, ctypes.c_int32),
                                     _p(num, ctypes.c_int32))
    if m < 0:
        raise MemoryError("oracle voxel table")
    return voxels[:m], coors[:m], num[:m]


# --------------------------------------------------------------------------
# a2  batch merge — single_stage.py:52-73
# --------------------------------------------------------------------------
def merge_batch(voxels_l, coors_l, num_l):
    voxels = np.concatenate(voxels_l, 0)
    num = np.concatenate(num_l, 0)
    coors = np.concatenate([np.pad(c, ((0, 0), (1, 0)), constant_values=i)
                            for i, c in enumerate(coors_l)], 0).astype(np.int32)
    return voxels, coors, num


# --------------------------------------------------------------------------
# a3  SimpleVoxel — vxnet.py:110-116
# --------------------------------------------------------------------------
def simple_voxel(voxels, num_points, num_input_features=4):
    v = torch.as_tensor(voxels)
    n = torch.as_tensor(num_points)
    return (v[:, :, :num_input_features].sum(dim=1) / n.type_as(v).view(-1, 1)).contiguous()


# --------------------------------------------------------------------------
# a5  rulebooks — spconv v1.0 get_indice_pairs semantics (SURVEY.md §A.2)
# canonical form: output rows sorted by flattened (b,z,y,x); per offset k the
# pair list is sorted by output row.
# --------------------------------------------------------------------------
def _flat(coords, shape):
    c = coords.astype(np.int64)
    return ((c[:, 0] * shape[0] + c[:, 1]) * shape[1] + c[:, 2]) * shape[2] + c[:, 3]


def subm_rulebook(coords, shape):
    """SubMConv3d(k=3): output sites == input sites (same order).  Pair (i, o, k)
    exists when site(o) + (kz-1, ky-1, kx-1) is an active input i.
    Returns nbr [N, 27] int32 (-1 = none)."""
    coords = np.asarray(coords, np.int32)
    n = coords.shape[0]
    nbr = np.full((n, 27), -1, np.int32)
    if n == 0:
        return nbr
    keys = _flat(coords, shape)
    order = np.argsort(keys, kind="stable")
    skeys = keys[order]
    k = 0
    for kz in range(3):
        for ky in range(3):
            for kx in range(3):
                q = coords.astype(np.int64).copy()
                q[:, 1] += kz - 1
                q[:, 2] += ky - 1
                q[:, 3] += kx - 1
                ok = ((q[:, 1] >= 0) & (q[:, 1] < shape[0]) & (q[:, 2] >= 0) & (q[:, 2] < shape[1]) &
                      (q[:, 3] >= 0) & (q[:, 3] < shape[2]))
                qk = _flat(q, shape)
                pos = np.searchsorted(skeys, qk)
                pos = np.clip(pos, 0, n - 1)
                hit = ok & (skeys[pos] == qk)
                nbr[hit, k] = order[pos[hit]]
                k += 1
    return nbr


def conv_out_shape(shape, ksize=3, stride=2, pad=1):
    return [int((s + 2 * pad - ksize) // stride + 1) for s in shape]


def sparse_conv_rulebook(coords, shape, ksize=3, stride=2, pad=1):
    """SparseConv3d(k=3, s=2, p=1): active outputs = every output cell whose
    3^3 window touches an active input (i = s*o - p + k).  Output rows sorted by
    flattened (b,z,y,x).  Returns (out_coords [Nout,4] i32, nbr [Nout,27] i32,
    out_shape)."""
    coords = np.asarray(coords, np.int32)
    out_shape = conv_out_shape(shape, ksize, stride, pad)
    n = coords.shape[0]
    if n == 0:
        return np.zeros((0, 4), np.int32), np.zeros((0, ksize ** 3), np.int32), out_shape
    cand = []
    c64 = coords.astype(np.int64)
    for kz in range(ksize):
        for ky in range(ksize):
            for kx in range(ksize):
                num = c64[:, 1:] + pad - np.array([kz, ky, kx])
                ok = np.all(num % stride == 0, axis=1)
                o = num // stride
                ok &= np.all((o >= 0) & (o < np.array(out_shape)), axis=1)
                cand.append(np.concatenate([c64[ok, :1], o[ok]], axis=1))
    cand = np.concatenate(cand, 0)
    okeys = np.unique(_flat(cand, out_shape))
    nout = okeys.shape[0]
    out = np.zeros((nout, 4), np.int64)
    r = okeys.copy()
    out[:, 3] = r % out_shape[2]; r //= out_shape[2]
    out[:, 2] = r % out_shape[1]; r //= out_shape[1]
    out[:, 1] = r % out_shape[0]; r //= out_shape[0]
    out[:, 0] = r
    ikeys = _flat(coords, shape)
    order = np.argsort(ikeys, kind="stable")
    skeys = ikeys[order]
    nbr = np.full((nout, ksize ** 3), -1, np.int32)
    k = 0
    for kz in range(ksize):
        for ky in range(ksize):
            for kx in range(ksize):
                q = out.copy()
                q[:, 1] = out[:, 1] * stride - pad + kz
                q[:, 2] = out[:, 2] * stride - pad + ky
                q[:, 3] = out[:, 3] * stride - pad + kx
                ok = ((q[:, 1] >= 0) & (q[:, 1] < shape[0]) & (q[:, 2] >= 0) & (q[:, 2] < shape[1]) &
                      (q[:, 3] >= 0) & (q[:, 3] < shape[2]))
                qk = _flat(q, shape)
                pos = np.clip(np.searchsorted(skeys, qk), 0, n - 1)
                hit = ok & (skeys[pos] == qk)
                nbr[hit, k] = order[pos[hit]]
                k += 1
    return out.astype(np.int32), nbr, out_shape


def nbr_to_indice_pairs(nbr, n_cap=None):
    """Neighbour table -> spconv-v1 style tables: indice_pairs [2, K, n_cap]
    (-1 padded; [0]=input row, [1]=output row; per offset sorted by output row)
    and indice_pair_num [K]."""
    n, K = nbr.shape
    n_cap = n if n_cap is None else n_cap
    pairs = np.full((2, K, n_cap), -1, np.int32)
    num = np.zeros((K,), np.int32)
    for k in range(K):
        o = np.nonzero(nbr[:, k] >= 0)[0]
        num[k] = o.shape[0]
        pairs[0, k, :o.shape[0]] = nbr[o, k]
        pairs[1, k, :o.shape[0]] = o
    return pairs, num


# --------------------------------------------------------------------------
# a6/a7  indice_conv + BN1d(eval) + ReLU — spconv v1.0 dataflow: per offset k
# ascending: gather -> mm -> scatter-add (SURVEY.md §A.2); cmn.py:138-173
# --------------------------------------------------------------------------
def indice_conv(feats, weight, nbr):
    """feats [Nin, Cin]; weight [K(=kz*9+ky*3+kx), Cin, Cout]; nbr [Nout, K]."""
    nout, K = nbr.shape
    out = torch.zeros((nout, weight.shape[2]), dtype=torch.float32)
    nbr_t = torch.as_tensor(nbr, dtype=torch.int64)
    for k in range(K):
        o = torch.nonzero(nbr_t[:, k] >= 0).view(-1)
        if o.numel() == 0:
            continue
        out.index_add_(0, o, feats.index_select(0, nbr_t[o, k]) @ weight[k])
    return out


def bn_eval(x, sd, prefix, eps=1e-3):
    w, b = sd[prefix + ".weight"], sd[prefix + ".bias"]
    m, v = sd[prefix + ".running_mean"], sd[prefix + ".running_var"]
    shape = [1, -1] + [1] * (x.dim() - 2)
    return (x - m.view(shape)) / torch.sqrt(v.view(shape) + eps) * w.view(shape) + b.view(shape)


VXNET_PLAN = [  # (block, [conv idx...], kind, rulebook key) — cmn.py:192-212
    ("conv0", (0, 3), "subm", 0), ("down0", (0,), "down", 0),
    ("conv1", (0, 3), "subm", 1), ("down1", (0,), "down", 1),
    ("conv2", (0, 3, 6), "subm", 2), ("down2", (0,), "down", 2),
    ("conv3", (0, 3, 6), "subm", 3),
]


def vxnet_forward(sd, feats, coords, shape, prefix="neck.backbone.", return_rulebooks=False):
    """VxNet.forward — cmn.py:214-231.  feats [N,4] f32, coords [N,4] (b,z,y,x).
    Returns (features [N3,64], coords [N3,4], shape) after extra_conv."""
    x = torch.as_tensor(feats, dtype=torch.float32)
    coords = np.asarray(coords, np.int32)
    shape = list(shape)
    books = {}
    nbr_subm = None
    for block, idxs, kind, key in VXNET_PLAN:
        if kind == "down":
            coords_out, nbr, shape_out = sparse_conv_rulebook(coords, shape)
            books["down%d" % key] = (nbr, coords_out, shape_out)
            w = sd["%s%s.0.weight" % (prefix, block)]
            x = indice_conv(x, w.reshape(27, w.shape[3], w.shape[4]), nbr)
            x = torch.relu(bn_eval(x, sd, "%s%s.1" % (prefix, block)))
            coords, shape = coords_out, shape_out
            nbr_subm = None
        else:
            if nbr_subm is None:
                nbr_subm = subm_rulebook(coords, shape)
                books["subm%d" % key] = (nbr_subm, coords, shape)
            for i in idxs:
                w = sd["%s%s.%d.weight" % (prefix, block, i)]
                x = indice_conv(x, w.reshape(27, w.shape[3], w.shape[4]), nbr_subm)
                x = torch.relu(bn_eval(x, sd, "%s%s.%d" % (prefix, block, i + 1)))
    # extra_conv: SparseConv3d(64,64,(1,1,1)) == features @ W[64,64]  (cmn.py:208-212)
    w = sd[prefix + "extra_conv.0.weight"]
    x = x @ w.reshape(w.shape[3], w.shape[4])
    x = torch.relu(bn_eval(x, sd, prefix + "extra_conv.1"))
    if return_rulebooks:
        return x, coords, shape, books
    return x, coords, shape


# --------------------------------------------------------------------------
# a8  dense() + view — spconv scatter_nd / cmn.py:112-114
# --------------------------------------------------------------------------
def dense_bev(feats, coords, shape, batch_size):
    C = feats.shape[1]
    D, H, W = shape
    out = torch.zeros((batch_size, D, H, W, C), dtype=torch.float32)
    c = torch.as_tensor(np.asarray(coords), dtype=torch.int64)
    out[c[:, 0], c[:, 1], c[:, 2], c[:, 3]] = feats
    out = out.permute(0, 4, 1, 2, 3).contiguous()          # [B, C, D, H, W]
    return out.view(batch_size, C * D, H, W)               # channel = c*D + d


# --------------------------------------------------------------------------
# a9  BEVNet — cmn.py:233-282
# --------------------------------------------------------------------------
def bevnet_forward(sd, x, prefix="neck.fcn."):
    for i in range(7):
        x = F.conv2d(x, sd["%sconv%d.weight" % (prefix, i)], None, padding=1)
        x = torch.relu(bn_eval(x, sd, "%sbn%d" % (prefix, i)))
    conv6 = x.clone()
    x = F.conv2d(x, sd[prefix + "conv7.weight"], None)
    x = torch.relu(bn_eval(x, sd, prefix + "bn7"))
    return x, conv6


# --------------------------------------------------------------------------
# a10  SSDRotateHead.forward — ssd_rotate_head.py:218-235
# --------------------------------------------------------------------------
def rpn_head_forward(sd, x, num_class, prefix="rpn_head."):
    N, _, H, W = x.shape
    box = F.conv2d(x, sd[prefix + "conv_box.weight"], sd[prefix + "conv_box.bias"])
    cls = F.conv2d(x, sd[prefix + "conv_cls.weight"], sd[prefix + "conv_cls.bias"])
    dirp = F.conv2d(x, sd[prefix + "conv_dir_cls.weight"], sd[prefix + "conv_dir_cls.bias"])
    box = box.view(N, num_class, -1, H, W).permute(0, 1, 3, 4, 2).contiguous()
    cls = cls.view(N, num_class, -1, H, W).permute(0, 1, 3, 4, 2).contiguous()
    dirp = dirp.view(N, num_class, -1, H, W).permute(0, 1, 3, 4, 2).contiguous()
    return box, cls, dirp


# --------------------------------------------------------------------------
# a11  second_box_decode — ssd_rotate_head.py:53-91 (no sin/cos vector, no smooth)
# --------------------------------------------------------------------------
def second_box_decode(enc, anchors):
    xa, ya, za, wa, la, ha, ra = torch.split(anchors, 1, dim=-1)
    xt, yt, zt, wt, lt, ht, rt = torch.split(enc, 1, dim=-1)
    za = za + ha / 2
    diagonal = torch.sqrt(la ** 2 + wa ** 2)
    xg = xt * diagonal + xa
    yg = yt * diagonal + ya
    zg = zt * ha + za
    lg = torch.exp(lt) * la
    wg = torch.exp(wt) * wa
    hg = torch.exp(ht) * ha
    rg = rt + ra
    zg = zg - hg / 2
    return torch.cat([xg, yg, zg, wg, lg, hg, rg], dim=-1)


# --------------------------------------------------------------------------
# a12  get_guided_anchors — ssd_rotate_head.py:307-372 (gt_* = None)
# --------------------------------------------------------------------------
def get_guided_anchors(box, cls, dirp, anchors, anchors_mask, num_class, thr=0.1, return_index=False):
    B = box.shape[0]
    bbox = second_box_decode(box.reshape(B, -1, 7), anchors)
    bcls = cls.reshape(B, -1, num_class)
    bdir = dirp.reshape(B, -1, 2)
    bmask = anchors_mask.reshape(B, -1)
    guided, labels, index, scores_out = [], [], [], []
    for b in range(B):
        sel0 = torch.nonzero(bmask[b]).view(-1)
        bp, cp, dp = bbox[b][sel0], bcls[b][sel0], bdir[b][sel0]
        dir_labels = torch.max(dp, dim=-1)[1]
        total = torch.sigmoid(cp)
        if num_class == 1:
            top_scores = total.squeeze(-1)
            top_labels = torch.zeros(total.shape[0], dtype=torch.int64)
        else:
            top_scores, top_labels = torch.max(total, dim=-1)
        sel = top_scores > thr
        bp = bp[sel].clone()
        top_labels = top_labels[sel]
        dir_labels = dir_labels[sel]
        opp = (bp[..., -1] > 0) ^ dir_labels.bool()
        bp[opp, -1] += np.pi
        guided.append(bp)
        labels.append(top_labels)
        index.append(sel0[sel])
        scores_out.append(top_scores[sel])
    if return_index:
        return guided, labels, index, scores_out
    return guided, labels


# --------------------------------------------------------------------------
# a13/a14  PSWarpHead — ssd_rotate_head.py:374-447
# --------------------------------------------------------------------------
def gen_sample_grid(box, window_size=(4, 7), grid_offsets=(0., 40.), spatial_scale=2.5):
    N = box.shape[0]
    win = window_size[0] * window_size[1]
    xg, yg, wg, lg, rg = torch.split(box, 1, dim=-1)
    xg = xg.unsqueeze(-1).expand(N, *window_size)
    yg = yg.unsqueeze(-1).expand(N, *window_size)
    rg = rg.unsqueeze(-1).expand(N, *window_size)
    cosT, sinT = torch.cos(rg), torch.sin(rg)
    xx = torch.linspace(-.5, .5, window_size[0]).type_as(box).view(1, -1) * wg
    yy = torch.linspace(-.5, .5, window_size[1]).type_as(box).view(1, -1) * lg
    xx = xx.unsqueeze(-1).expand(N, *window_size)
    yy = yy.unsqueeze(1).expand(N, *window_size)
    x = xx * cosT + yy * sinT + xg
    y = yy * cosT - xx * sinT + yg
    x = (x.permute(1, 2, 0).contiguous() + grid_offsets[0]) * spatial_scale
    y = (y.permute(1, 2, 0).contiguous() + grid_offsets[1]) * spatial_scale
    return x.view(win, -1), y.view(win, -1)


def bilinear_gridsample(image, sx, sy):
    C, H, W = image.shape
    image = image.unsqueeze(1)
    samples = torch.cat([sx.unsqueeze(2).unsqueeze(3), sy.unsqueeze(2).unsqueeze(3)], 3).clone()
    samples[:, :, :, 0] = samples[:, :, :, 0] / (W - 1)
    samples[:, :, :, 1] = samples[:, :, :, 1] / (H - 1)
    samples = samples * 2 - 1
    return F.grid_sample(image, samples, align_corners=True)


def pswarp_convs(sd, conv6, prefix="extra_head."):
    x = F.conv2d(conv6, sd[prefix + "convs.0.weight"], None, padding=1)
    x = torch.relu(bn_eval(x, sd, prefix + "convs.1"))
    return F.conv2d(x, sd[prefix + "convs.3.weight"], None)


def pswarp_forward(sd, conv6, guided, grid_offsets=(0., 40.), featmap_stride=.4, prefix="extra_head."):
    x = pswarp_convs(sd, conv6, prefix)
    scores = []
    for i, ga in enumerate(guided):
        if len(ga) == 0:
            scores.append(torch.empty(0))
            continue
        xs, ys = gen_sample_grid(ga[:, [0, 1, 3, 4, 6]], grid_offsets=grid_offsets,
                                 spatial_scale=1 / featmap_stride)
        out = bilinear_gridsample(x[i], xs, ys)
        scores.append(torch.mean(out, 0).view(-1))
    return scores


# --------------------------------------------------------------------------
# a16  boxes3d_to_bev_torch — iou3d_utils.py:47-60
# --------------------------------------------------------------------------
def boxes3d_to_bev(b):
    out = torch.empty((b.shape[0], 5), dtype=b.dtype)
    cu, cv = b[:, 0], b[:, 1]
    hl, hw = b[:, 3] / 2, b[:, 4] / 2
    out[:, 0], out[:, 1] = cu - hl, cv - hw
    out[:, 2], out[:, 3] = cu + hl, cv + hw
    out[:, 4] = b[:, 6]
    return out


# --------------------------------------------------------------------------
# a17  nms_gpu / rotate_nms_torch — iou3d_utils.py:114-128, bbox_nms.py:4-27,
# iou3d.cpp:73-120.  Sort ties: stable, index-ascending (the reference uses an
# unstable device sort; the canonical tie-break is ours, SURVEY.md §7.2).
# --------------------------------------------------------------------------
def nms_rotated(boxes_bev, scores, thr):
    n = boxes_bev.shape[0]
    if n == 0:
        return torch.empty((0,), dtype=torch.int64)
    order = torch.sort(scores, descending=True, stable=True)[1]
    b = np.ascontiguousarray(boxes_bev[order].numpy(), np.float32)
    keep = np.zeros((n,), np.int64)
    num = lib().oracle_nms_sorted(_p(b, ctypes.c_float), n, ctypes.c_float(thr), _p(keep, ctypes.c_int64))
    return order[torch.as_tensor(keep[:num])]


def nms_mask(boxes_sorted, thr):
    b = np.ascontiguousarray(boxes_sorted, np.float32)
    n = b.shape[0]
    cb = (n + 63) // 64
    mask = np.zeros((n, max(cb, 1)), np.uint64)
    if n:
        lib().oracle_nms_mask(_p(b, ctypes.c_float), n, ctypes.c_float(thr), _p(mask, ctypes.c_uint64))
    return mask[:, :cb]


def overlap_points(a, b):
    """polygon point count of box_overlap(a[i], b[i]) for BEV box pairs [n,5]: the reference keeps at most 16"""
    a = np.ascontiguousarray(a, np.float32)
    b = np.ascontiguousarray(b, np.float32)
    assert a.shape == b.shape and a.shape[-1] == 5
    out = np.zeros((a.shape[0],), np.int32)
    if len(out):
        lib().oracle_overlap_points(_p(a, ctypes.c_float), _p(b, ctypes.c_float), len(out), _p(out, ctypes.c_int32))
    return out


def iou_matrix(boxes):
    b = np.ascontiguousarray(boxes, np.float32)
    n = b.shape[0]
    out = np.zeros((n, n), np.float32)
    if n:
        lib().oracle_iou_matrix(_p(b, ctypes.c_float), n, _p(out, ctypes.c_float))
    return out


# --------------------------------------------------------------------------
# a15  get_rescore_bboxes — ssd_rotate_head.py:487-533
# --------------------------------------------------------------------------
def get_rescore_bboxes(guided, cls_scores, labels, score_thr=0.3, iou_thr=0.1):
    det_b, det_s, det_l = [], [], []
    for bp, sc, lb in zip(guided, cls_scores, labels):
        if sc.numel() == 0:
            det_b.append(None); det_s.append(None); det_l.append(None)
            continue
        bp = bp.view(-1, 7)
        s = torch.sigmoid(sc).view(-1)
        sel = s > score_thr
        bp, s, lb = bp[sel, :], s[sel], lb[sel]
        if s.numel() == 0:
            det_b.append(None); det_s.append(None); det_l.append(None)
            continue
        keep = nms_rotated(boxes3d_to_bev(bp), s, iou_thr)
        det_b.append(bp[keep, :].numpy()); det_s.append(s[keep].numpy()); det_l.append(lb[keep].numpy())
    return det_b, det_s, det_l


# --------------------------------------------------------------------------
# a18  anchors + anchors_mask — anchor3d_generator.py:3-41, kitti.py:80-88,333-343,
# geometry.py:404-426,675-709
# --------------------------------------------------------------------------
def create_anchors_3d_stride(feature_size, sizes, anchor_strides, anchor_offsets, rotations,
                             dtype=np.float32):
    x_stride, y_stride, z_stride = anchor_strides
    x_offset, y_offset, z_offset = anchor_offsets
    zc = np.arange(feature_size[0], dtype=dtype) * z_stride + z_offset
    yc = np.arange(feature_size[1], dtype=dtype) * y_stride + y_offset
    xc = np.arange(feature_size[2], dtype=dtype) * x_stride + x_offset
    sizes = np.reshape(np.array(sizes, dtype=dtype), [-1, 3])
    rotations = np.array(rotations, dtype=dtype)
    rets = list(np.meshgrid(xc, yc, zc, rotations, indexing="ij"))
    tile_shape = [1] * 5
    tile_shape[-2] = int(sizes.shape[0])
    for i in range(len(rets)):
        rets[i] = np.tile(rets[i][..., np.newaxis, :], tile_shape)
        rets[i] = rets[i][..., np.newaxis]
    sizes = np.reshape(sizes, [1, 1, 1, -1, 1, 3])
    tile_size_shape = list(rets[0].shape)
    tile_size_shape[3] = 1
    sizes = np.tile(sizes, tile_size_shape)
    rets.insert(3, sizes)
    ret = np.concatenate(rets, axis=-1)
    return np.transpose(ret, [2, 1, 0, 3, 4, 5])


def limit_period(val, offset=0.5, period=np.pi):
    return val - np.floor(val / period + offset) * period


def rbbox2d_to_near_bbox(rbboxes):
    rots = rbboxes[..., -1]
    r = np.abs(limit_period(rots, 0.5, np.pi))
    cond = (r > np.pi / 4)[..., np.newaxis]
    ctr = np.where(cond, rbboxes[:, [0, 1, 3, 2]], rbboxes[:, :4])
    return np.concatenate([ctr[:, :2] - ctr[:, 2:] / 2, ctr[:, :2] + ctr[:, 2:] / 2], axis=-1)


def make_anchors(anchor_cfgs, feature_map_size=(1, 200, 176)):
    """kitti.py:80-88 (test_mode): concat over classes of [H*W*2, 7]."""
    a = np.concatenate([create_anchors_3d_stride(list(feature_map_size), c["sizes"], c["anchor_strides"],
                                                 c["anchor_offsets"], c["rotations"]).reshape(-1, 7)
                        for c in anchor_cfgs], 0)
    return a, rbbox2d_to_near_bbox(a[..., [0, 1, 3, 4, 6]])


def anchors_mask(coors_zyx, anchors_bv, voxel_size, pc_range, grid_size, area_threshold=1):
    """kitti.py:333-343: occupancy count -> 2 cumsums -> per-anchor integral-image
    lookup (geometry.py:684-709) > threshold.  coors_zyx [M,3]; grid_size (x,y,z)."""
    H, W = int(grid_size[1]), int(grid_size[0])
    dense = np.zeros((H, W), np.float32)
    np.add.at(dense, (coors_zyx[:, 1], coors_zyx[:, 2]), 1.0)
    dense = dense.cumsum(0).cumsum(1)
    vs = np.asarray(voxel_size, np.float32)
    off = np.asarray(pc_range, np.float32)
    a = np.asarray(anchors_bv, np.float32)
    c0 = np.floor((a[:, 0] - off[0]) / vs[0]).astype(np.int32)
    c1 = np.floor((a[:, 1] - off[1]) / vs[1]).astype(np.int32)
    c2 = np.floor((a[:, 2] - off[0]) / vs[0]).astype(np.int32)
    c3 = np.floor((a[:, 3] - off[1]) / vs[1]).astype(np.int32)
    c0 = np.maximum(c0, 0); c1 = np.maximum(c1, 0)
    c2 = np.minimum(c2, W - 1); c3 = np.minimum(c3, H - 1)
    area = dense[c3, c2] - dense[c3, c0] - dense[c1, c2] + dense[c1, c0]
    return area > area_threshold


# --------------------------------------------------------------------------
# whole frame(s): SingleStageDetector.forward_test — single_stage.py:110-131
# (up to and excluding kitti_bbox2results, which is a "next" row)
# --------------------------------------------------------------------------
def forward_test(sd, points_list, cfg, num_class=1, stages=None):
    """cfg: dict(voxel_size, pc_range, max_points, max_voxels, sparse_shape,
    anchor_cfgs, grid_offsets, featmap_stride, score_thr, iou_thr).
    ``stages`` (dict) receives intermediate tensors when given."""
    vl, cl, nl = [], [], []
    for p in points_list:
        v, c, n = points_to_voxel(p, cfg["voxel_size"], cfg["pc_range"], cfg["max_points"], cfg["max_voxels"])
        vl.append(v); cl.append(c); nl.append(n)
    B = len(points_list)
    anchors, anchors_bv = make_anchors(cfg["anchor_cfgs"])
    vsz = np.asarray(cfg["voxel_size"], np.float32)
    rng = np.asarray(cfg["pc_range"], np.float32)
    grid = np.round((rng[3:] - rng[:3]) / vsz).astype(np.int64)
    masks = [anchors_mask(c, anchors_bv, vsz, rng, grid) for c in cl]
    voxels, coors, num = merge_batch(vl, cl, nl)
    vx = simple_voxel(voxels, num)
    feats, c3, shape3 = vxnet_forward(sd, vx, coors, cfg["sparse_shape"])
    bev = dense_bev(feats, c3, shape3, B)
    x, conv6 = bevnet_forward(sd, bev)
    box, cls, dirp = rpn_head_forward(sd, x, num_class)
    anc = torch.as_tensor(anchors).unsqueeze(0).expand(B, -1, -1)
    msk = torch.as_tensor(np.stack(masks, 0))
    guided, labels, index, rpn_scores = get_guided_anchors(box, cls, dirp, anc, msk, num_class, thr=0.1,
                                                           return_index=True)
    scores = pswarp_forward(sd, conv6, guided, cfg["grid_offsets"], cfg["featmap_stride"])
    det = get_rescore_bboxes(guided, scores, labels, cfg["score_thr"], cfg["iou_thr"])
    if stages is not None:
        stages.update(dict(voxels=vl, coors=cl, num_points=nl, anchors=anchors, anchors_mask=masks, vx=vx,
                           feats3=feats, coors3=c3, bev=bev, x=x, conv6=conv6, box=box, cls=cls, dir=dirp,
                           guided=guided, labels=labels, guided_index=index, rpn_scores=rpn_scores,
                           ps_scores=scores))
    return det
