"""``mmdet.models.necks`` mirror for the hot path: SpMiddleFHD = VxNet (sparse 3-D
backbone) + BEVNet (dense BEV convs) — mmdet/models/necks/cmn.py:12-29,102-119,138-282.

Parameter names and shapes equal the reference's (SURVEY.md §8b) so that its
checkpoints load; all arithmetic runs in the sm_90a kernels of csrc/gconv.cu
(BatchNorm folded into each conv's epilogue, eval mode).  The auxiliary point-wise network
(cmn.py:121-135, :175-189) runs in eval mode: ``forward(..., is_test=False)`` returns the reference's
``(x, conv6, (points_mean, point_cls, point_reg))`` through csrc/point_aux.cu.  Its loss and targets
(cmn.py:44-100) serve training only and are not built; in training mode ``forward`` raises.
"""
import torch
from torch import nn

from . import ops, spconv
from .spconv import fold_bn, _versions


def single_conv(in_channels, out_channels, indice_key=None):
    return spconv.SparseSequential(
        spconv.SubMConv3d(in_channels, out_channels, 1, bias=False, indice_key=indice_key),
        nn.BatchNorm1d(out_channels, eps=1e-3, momentum=0.01),
        nn.ReLU(),
    )


def _subm_block(n, in_channels, out_channels, indice_key):
    layers = []
    for i in range(n):
        layers += [spconv.SubMConv3d(in_channels if i == 0 else out_channels, out_channels, 3, bias=False,
                                     indice_key=indice_key),
                   nn.BatchNorm1d(out_channels, eps=1e-3, momentum=0.01), nn.ReLU()]
    return spconv.SparseSequential(*layers)


def double_conv(in_channels, out_channels, indice_key=None):
    return _subm_block(2, in_channels, out_channels, indice_key)


def triple_conv(in_channels, out_channels, indice_key=None):
    return _subm_block(3, in_channels, out_channels, indice_key)


def stride_conv(in_channels, out_channels, indice_key=None):
    return spconv.SparseSequential(
        spconv.SparseConv3d(in_channels, out_channels, 3, (2, 2, 2), padding=1, bias=False, indice_key=indice_key),
        nn.BatchNorm1d(out_channels, eps=1e-3, momentum=0.01),
        nn.ReLU(),
    )


class VxNet(nn.Module):
    """cmn.py:192-231."""

    def __init__(self, num_input_features):
        super().__init__()
        self.conv0 = double_conv(num_input_features, 16, "subm0")
        self.down0 = stride_conv(16, 32, "down0")
        self.conv1 = double_conv(32, 32, "subm1")
        self.down1 = stride_conv(32, 64, "down1")
        self.conv2 = triple_conv(64, 64, "subm2")
        self.down2 = stride_conv(64, 64, "down2")
        self.conv3 = triple_conv(64, 64, "subm3")
        self.extra_conv = spconv.SparseSequential(
            spconv.SparseConv3d(64, 64, (1, 1, 1), (1, 1, 1), bias=False),
            nn.BatchNorm1d(64, eps=1e-3, momentum=0.01),
            nn.ReLU(),
        )

    def forward(self, x):
        middle = []
        x = self.conv0(x)
        x = self.down0(x)
        x = self.conv1(x)
        middle.append(x)
        x = self.down1(x)
        x = self.conv2(x)
        middle.append(x)
        x = self.down2(x)
        x = self.conv3(x)
        middle.append(x)
        out = self.extra_conv(x)
        return out, middle

    def set_precision(self, precision):
        for m in self.modules():
            if isinstance(m, spconv._SparseConvBase):
                m.precision = precision

    def prebuild_rulebooks(self, x, side_stream, table_stream=None):
        """All seven rulebooks depend on coordinates only, never on features, so they are built beside the feature
        convolutions, which wait on each rulebook's event when they first use it.  Two chains: ``side_stream`` carries
        the coordinate chain - level-0 hash, then per strided conv "mark + single-pass compaction", which also hashes
        the next level's rows (7 kernels end to end); ``table_stream`` fills the seven neighbour tables, each as soon
        as the coordinates and the hash it probes exist.  Round 1 ran all 23 launches back to back on one stream and the
        last table arrived 0.3 ms into a 0.9 ms step - later than the convolutions needed it."""
        main = torch.cuda.current_stream()
        side_stream.wait_stream(main)
        tables = table_stream if table_stream is not None else side_stream
        dev = x.device
        coors, d_rows, shape, cap = x._indices, x.d_rows, x.spatial_shape, x.rows_cap
        with torch.cuda.stream(side_stream):
            index = ops.hash_build(ops.HashIndex(cap, dev), coors, d_rows, x.batch_size, shape, x.status)
        x._index = index
        for lvl in range(4):
            tables.wait_stream(side_stream)              # this level's coordinates and hash are queued
            with torch.cuda.stream(tables):
                nbr, tmask = ops.rulebook_subm(coors, d_rows, shape, index)
                ev = torch.cuda.Event(); ev.record(tables)
                x.indice_dict["subm%d" % lvl] = spconv.Rulebook(nbr, coors, d_rows, shape, index, ev, tmask)
            if lvl == 3:
                break
            D, H, W = ops.conv_out_shape(shape)
            cap = max(1, min(int(cap * x.row_cap_factor), x.batch_size * D * H * W))
            with torch.cuda.stream(side_stream):
                index_out = ops.HashIndex(cap, dev)
                co, dn, so = ops.rulebook_conv_outputs(coors, d_rows, x.batch_size, shape, cap, x.status,
                                                       ws_key="rbconv%d" % lvl, index_out=index_out)
            tables.wait_stream(side_stream)
            with torch.cuda.stream(tables):
                nbr2, tmask2 = ops.rulebook_conv_nbr(co, dn, shape, index)
                ev = torch.cuda.Event(); ev.record(tables)
                x.indice_dict["down%d" % lvl] = spconv.Rulebook(nbr2, co, dn, so, index_out, ev, tmask2)
            coors, d_rows, shape, index = co, dn, so, index_out
        if tables is not side_stream:
            side_stream.wait_stream(tables)              # one join point for the caller
        x._rulebook_stream = side_stream   # keep the stream (and its tensors) alive with the tensor


def pack_conv2d_weight(w, dc_order=None):
    """[Cout, Cin, kh, kw] -> [taps, Cin, Cout] (tap = ky*3+kx).  ``dc_order=(C, D)`` re-orders
    the input channels from the reference's dense() order c*D+d to the internal d*C+c."""
    cout, cin, kh, kw = w.shape
    p = w.detach().permute(2, 3, 1, 0).reshape(kh * kw, cin, cout)
    if dc_order is not None:
        C, D = dc_order
        p = p.reshape(kh * kw, C, D, cout).permute(0, 2, 1, 3).reshape(kh * kw, cin, cout)
    return p.contiguous().float()


def conv2d_nhwc(x, weight_packed, scale, shift, relu, cout, precision=ops.PREC_FP32, out=None, split_out=False,
                in_ready=None, out_ready=None):
    """x [B,H,W,Cin] NHWC contiguous -> [B,H,W,cout_stride]; 3x3 (pad 1) when taps == 9, 1x1 when 1.
    A ``ops.SplitMap`` input selects the TMA tensor-core kernel (csrc/conv2d_tma.cu); ``split_out`` then keeps
    the output in split form for the next such layer, and in_ready / out_ready are its tile counters
    (ops.conv2d_split)."""
    if isinstance(x, ops.SplitMap):
        sp, f32 = ops.conv2d_split(x, weight_packed, scale, shift, relu, cout, out_split=split_out,
                                   out_f32=not split_out, in_ready=in_ready, out_ready=out_ready)
        return sp if split_out else f32
    B, H, W, cin = x.shape
    taps = weight_packed.shape[0]
    stride = (cout + 3) // 4 * 4
    if out is None:
        out = torch.empty((B, H, W, stride), dtype=torch.float32, device=x.device)
        if stride != cout:
            out.zero_()
    ops.gconv(x.view(-1, cin), weight_packed, scale, shift, out.view(-1, out.shape[-1]), mode=ops.GCONV_CONV2D,
              taps=taps, cin=cin, cout=cout, relu=relu, rows_cap=B * H * W, batch=B, H=H, W=W, precision=precision)
    return out


class BEVNet(nn.Module):
    """cmn.py:233-282.  conv{i}/bn{i} hold the reference-named parameters; compute is NHWC."""

    def __init__(self, in_features, num_filters=256):
        super().__init__()
        for i in range(8):
            k = 1 if i == 7 else 3
            setattr(self, "conv%d" % i, nn.Conv2d(in_features if i == 0 else num_filters, num_filters, k,
                                                  padding=k // 2, bias=False))
            setattr(self, "bn%d" % i, nn.BatchNorm2d(num_filters, eps=1e-3, momentum=0.01))
        self.num_filters = num_filters
        self.precision = ops.DEFAULT_PRECISION
        self._packed = {}

    def _weights(self, i, dc_order):
        conv = getattr(self, "conv%d" % i)
        key = (i, dc_order)
        ver = _versions(conv.weight)
        c = self._packed.get(key)
        if c is None or c[0] != ver:
            c = (ver, pack_conv2d_weight(conv.weight, dc_order))
            self._packed[key] = c
        return c[1]

    def forward_nhwc(self, x, dc_order=None):
        """x [B,H,W,Cin] (channel order d*C+c when dc_order=(C,D)).  Returns (x, conv6) NHWC."""
        if self.training:
            raise NotImplementedError("sassd_b200 is inference-only: call .eval()")
        split = isinstance(x, ops.SplitMap)
        # conv1-conv7 start each tile once the tiles it reads of the previous map are stored: counters for the
        # outputs of conv0-conv6.  A layer may then still read its input while later layers write theirs, so every
        # map stays referenced until conv7 is queued: the allocator must not hand one to a later layer's output.
        # Every layer's weights and folded BatchNorm before the first conv: on a cache miss they queue work, which must
        # not come between a conv and the next (ops.conv2d_split, in_ready).
        params = [(self._weights(i, dc_order if i == 0 else None),) + fold_bn(getattr(self, "bn%d" % i))
                  for i in range(8)]
        ready = ops.tile_ready_arena(x, 7) if split and self.num_filters > 64 else None
        live = []
        for i, (weight, scale, shift) in enumerate(params):
            kw = {}
            if ready is not None:
                kw = dict(in_ready=ready[i - 1] if i > 0 else None, out_ready=ready[i] if i < 7 else None)
                live.append(x)
            x = conv2d_nhwc(x, weight, scale, shift, True, self.num_filters, self.precision, split_out=split, **kw)
            if i == 6:
                conv6 = x
        return x, conv6

    def forward(self, x):
        """Reference signature: x [B, Cin, H, W] -> (x, conv6), both [B, 256, H, W] (channels-last storage)."""
        ops.require_cuda()
        xh = x.permute(0, 2, 3, 1).contiguous()
        y, c6 = self.forward_nhwc(xh)
        return y.permute(0, 3, 1, 2), c6.permute(0, 3, 1, 2)


class SpMiddleFHD(nn.Module):
    """cmn.py:12-29,102-119.  Constructor kwargs as in configs/car_cfg.py:10-15."""

    def __init__(self, output_shape, num_input_features=4, num_hidden_features=128):
        super().__init__()
        self.sparse_shape = list(output_shape)
        self.backbone = VxNet(num_input_features)
        self.fcn = BEVNet(in_features=num_hidden_features, num_filters=256)
        # auxiliary point-wise network (cmn.py:27-29), run by forward_nhwc(point_outputs=True)
        self.point_fc = nn.Linear(160, 64, bias=False)
        self.point_cls = nn.Linear(64, 1, bias=False)
        self.point_reg = nn.Linear(64, 3, bias=False)
        self.row_cap_factor = 4
        self.dense_tma = True             # F16X3: keep the BEV maps as split fp16 planes and feed the convs by TMA
        self.overlap_rulebooks = True     # build the rulebook chain on a side stream, concurrently with the convs
        self._side = None
        self._point_packed = None

    def max_batch(self):
        """The most frames one step can hold: the level-0 hash keys each voxel by its flattened (b, z, y, x) cell in
        31 bits (sassd_hash_build refuses batch * D * H * W >= 2^31 - 1); 23 on the 40 x 1600 x 1408 grid."""
        D, H, W = self.sparse_shape
        return (2147483647 - 1) // (D * H * W)

    def _point_weights(self):
        """(point_fc.weight^T [160,64], [point_cls.weight; point_reg.weight] [4,64]) fp32, re-derived when a reload
        changes the parameters (the same version check as BEVNet._weights)."""
        ver = _versions(self.point_fc.weight, self.point_cls.weight, self.point_reg.weight)
        c = self._point_packed
        if c is None or c[0] != ver:
            with torch.no_grad():
                fc_t = self.point_fc.weight.detach().t().contiguous().float()
                out = torch.cat([self.point_cls.weight.detach(), self.point_reg.weight.detach()], 0).contiguous().float()
            c = self._point_packed = (ver, fc_t, out)
        return c[1], c[2]

    def point_head(self, mean, coors, d_rows, middle, neighbours=None):
        """The auxiliary network on the device (cmn.py:121-135): ``mean`` / ``coors`` [cap,4] are the voxel rows,
        ``middle`` the outputs of conv1, conv2, conv3.  Returns dict(points_mean [cap,4] (b, x, y, z), point_cls [cap],
        point_reg [cap,3], idx / dist2 [cap,3,3] of the three nearest centres per level); rows past d_rows are
        unwritten.  point_reg is what the reference regresses, the offset from the point to its box centre
        (points_op.cpp:107-144).  ``neighbours``: (idx, dist2, points_mean) of an earlier call over the same voxels and
        rulebooks; they depend on coordinates only, so the networks of a detectors.CheckpointSweep skip three_nn."""
        if neighbours is None:
            levels = [(m._indices, m.d_rows) for m in middle]
            neighbours = ops.three_nn(mean, coors, d_rows, levels, points_mean=True)
        idx, dist2, pm = neighbours
        feats = []
        for m, ch in zip(middle, ops._lib.POINT_LEVEL_CHANNELS):
            if m._features is not None:
                feats.append(ops.point_level(feat=m._features, channels=ch))
            else:
                feats.append(ops.point_level(split=m._split, channels=ch))
        fc_t, w_out = self._point_weights()
        cls, reg = ops.point_aux_head(idx, dist2, d_rows, feats, fc_t, w_out)
        return dict(points_mean=pm, point_cls=cls, point_reg=reg, idx=idx, dist2=dist2, middle=middle)

    def build_aux_target(self, nxyz, gt_boxes3d, enlarge=1.0):
        """cmn.py:44-70 on the device: nxyz [N,4] (b, x, y, z) voxel means, frames in row order; gt_boxes3d one [G_b,7]
        tensor per frame (x, y, z_bottom, w, l, h, ry).  Returns (pts_labels [N] uint8: inside any box of the point's
        frame, center_offsets [N,3]: point minus the centre of the last box containing it, 0 when none), as
        pts_in_boxes3d computes them (points_op.cpp:92-144, including its z centre from the box's fourth value).  A frame
        without boxes is all background (the reference never sees one)."""
        labels, offsets, _ = self._aux_targets(nxyz, gt_boxes3d, enlarge)
        return labels.to(torch.uint8), offsets

    def _aux_targets(self, nxyz, gt_boxes3d, enlarge=1.0):
        from .single_stage_heads import stage_gt
        ops.require_cuda()
        dev = nxyz.device if nxyz.is_cuda else torch.device("cuda")
        boxes = []
        for g in gt_boxes3d:
            g = torch.as_tensor(g, dtype=torch.float32).reshape(-1, 7).clone()
            g[:, 3:6] *= enlarge
            boxes.append(g)
        gt, _, _, d_ngt = stage_gt(boxes, None, None, dev)
        pm = nxyz.to(dev).float().contiguous()
        n = pm.shape[0]
        if n == 0:
            return torch.zeros(0, dtype=torch.int32, device=dev), torch.zeros((0, 3), device=dev), None
        status = torch.zeros((1,), dtype=torch.int32, device=dev)
        d_rows = torch.tensor([n], dtype=torch.int32, device=dev)
        labels, offsets, d_npos = ops.points_in_boxes(pm, d_rows, gt, d_ngt, status)
        ops._lib.raise_on_status(status)
        return labels, offsets, (d_rows, d_npos)

    def aux_loss(self, points, point_cls, point_reg, gt_bboxes):
        """cmn.py:72-100: dict(aux_loss_cls, aux_loss_reg), each a [1] tensor, from the auxiliary outputs of
        forward(is_test=False) and one GT tensor per frame."""
        labels, offsets, rows = self._aux_targets(points, gt_bboxes)
        dev = labels.device
        out = torch.zeros((2,), dtype=torch.float32, device=dev)
        if rows is not None:
            d_rows, d_npos = rows
            ops.aux_loss(point_cls.reshape(-1).float().contiguous(), point_reg.float().contiguous(), labels, offsets,
                         d_rows, len(gt_bboxes), d_npos, out)
        return dict(aux_loss_cls=out[0:1], aux_loss_reg=out[1:2])

    def set_precision(self, precision, sparse=None):
        """precision for the dense BEV convs; ``sparse`` (default: same) for the ruled sparse convs."""
        self.backbone.set_precision(precision if sparse is None else sparse)
        self.fcn.precision = precision

    def sparse_input(self, voxel_features, coors, batch_size, d_rows=None, status=None):
        """The backbone's level-0 tensor with its seven rulebooks queued (VxNet.prebuild_rulebooks on this neck's side
        streams; with ``overlap_rulebooks`` off the first conv of each level builds them).  The rulebooks depend on the
        coordinates only, so the members of a detectors.DetectorSet share one such tensor (forward_nhwc's
        ``sparse_in``)."""
        x = spconv.SparseConvTensor(voxel_features, coors, self.sparse_shape, batch_size, d_rows=d_rows, status=status)
        x.row_cap_factor = self.row_cap_factor
        if self.overlap_rulebooks:
            if self._side is None:
                self._side = torch.cuda.Stream(device=x.device)
                self._side2 = torch.cuda.Stream(device=x.device)
            self.backbone.prebuild_rulebooks(x, self._side, self._side2)
        return x

    def forward_nhwc(self, voxel_features, coors, batch_size, d_rows=None, status=None, point_outputs=False,
                     sparse_in=None, neighbours=None):
        """Device-side entry: capacity-sized inputs + row counter; returns NHWC (x, conv6) and the tensor.  With
        ``point_outputs`` the auxiliary network runs after conv3, before the dense neck, and its outputs
        (point_head) come fourth; ``neighbours`` as point_head takes them.  ``sparse_in``: a sparse_input() tensor
        over these voxels, whose rulebooks this call uses instead of building its own."""
        if self.training:
            raise NotImplementedError("sassd_b200 is inference-only: call .eval()")
        if sparse_in is None:
            x = self.sparse_input(voxel_features, coors, batch_size, d_rows, status)
        else:       # the shared rulebooks and hash, but this network's own feature chain
            x = sparse_in._derive(sparse_in._features)
        side = getattr(sparse_in if sparse_in is not None else x, "_rulebook_stream", None)
        x0_mean, x0_coors, rows0 = x._features, x._indices, x.d_rows     # level 0: the voxel means (SimpleVoxel)
        x, middle = self.backbone(x)
        if side is not None:
            torch.cuda.current_stream().wait_stream(side)   # join (also required to end a graph capture)
        pts = None
        if point_outputs:
            pts = self.point_head(x0_mean, x0_coors, rows0, middle, neighbours)
        C = x._channels
        D, H, W = x.spatial_shape
        if self.fcn.precision == ops.PREC_F16X3 and self.dense_tma:
            # split fp16 planes + TMA-fed tensor-core convs (conv2d_tma.cu); y / conv6 are ops.SplitMap
            if x._split is not None and x._split.shape[2] == C:
                bev = ops.split_rows_to_bev(x._split, x._indices, x.d_rows, C, D, H, W, batch_size, x.status)
            else:
                bev = ops.sparse_to_bev_split(x.features_cap(), x._indices, x.d_rows, C, D, H, W, batch_size,
                                              x.status)
        else:
            feats = x.features_cap()
            bev = torch.zeros((batch_size, H, W, D * C), dtype=torch.float32, device=feats.device)
            ops.sparse_to_bev(feats, x._indices, x.d_rows, C, D, H, W, bev)
        y, conv6 = self.fcn.forward_nhwc(bev, dc_order=(C, D))
        if point_outputs:
            return y, conv6, x, pts
        return y, conv6, x

    def forward(self, voxel_features, coors, batch_size, is_test=False, d_rows=None, status=None):
        """cmn.py:102-135.  Returns (x, conv6), both [B, 256, H, W]; with ``is_test=False`` (eval mode only) also the
        auxiliary outputs (points_mean [N,4] = (b, x, y, z), point_cls [N,1] foreground logits, point_reg [N,3]
        offsets to the box centre), N the voxel rows (aux_loss takes them).  Training mode raises: BatchNorm batch
        statistics are not built."""
        if not is_test and self.training:
            raise NotImplementedError("the auxiliary training branch (cmn.py:44-100) is out of scope: call .eval()")
        out = self.forward_nhwc(voxel_features, coors, batch_size, d_rows, status, point_outputs=not is_test)
        y, conv6 = out[0], out[1]
        if isinstance(y, ops.SplitMap):
            y, conv6 = y.float(), conv6.float()
        y, conv6 = y.permute(0, 3, 1, 2), conv6.permute(0, 3, 1, 2)
        if is_test:
            return y, conv6
        pts = out[3]
        n = voxel_features.shape[0] if d_rows is None else int(d_rows.reshape(-1)[0].item())
        return y, conv6, (pts["points_mean"][:n], pts["point_cls"][:n].unsqueeze(1), pts["point_reg"][:n])
