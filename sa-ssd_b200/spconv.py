"""Host-side mirror of the spconv v1.0 operator API that the reference neck uses
(call sites mmdet/models/necks/cmn.py:1,109,112,139-173,208-212): SparseConvTensor,
SubMConv3d, SparseConv3d, SparseSequential.  spconv itself is third-party and not
vendored by the reference; the semantics implemented here are those of SURVEY.md
§A.2 (and are tested by definition against dense conv3d).

Everything computes through the sm_90a kernels behind the C ABI
(rulebook.cu + gconv.cu); there is no torch fallback.  Tensors carry a capacity
and a device-side row count (``d_rows``) so that a chain of layers never
synchronises; ``features`` / ``indices`` properties trim to the exact row count
(one sync) for callers that want the reference's exact shapes.
"""
import torch
from torch import nn

from . import ops


SPLIT_ROWS = True   # F16X3 sparse layers keep their features as split fp16 rows (spconv_split.cu)


class Rulebook:
    """nbr [rows_cap, 27] + the output coordinate set of one indice_key."""

    def __init__(self, nbr, coors_out, d_rows_out, shape_out, index_out=None, event=None, tile_mask=None):
        self.nbr, self.coors_out, self.d_rows_out, self.shape_out = nbr, coors_out, d_rows_out, shape_out
        self.tile_mask = tile_mask   # int32 per 128-row output tile: taps that occur in the tile (tap skipping)
        self.index_out = index_out   # hash index over coors_out when it was prebuilt
        self.event = event           # recorded on the stream that built the rulebook (None = same stream)

    def indice_pairs(self):
        """spconv-v1 tables (indice_pairs [2,27,cap], indice_pair_num [27])."""
        return ops.rulebook_pairs(self.nbr, self.d_rows_out)


class SparseConvTensor:
    """spconv.SparseConvTensor(features [N,C], indices [N,4] int32 (b,z,y,x), spatial_shape, batch_size)."""

    def __init__(self, features, indices, spatial_shape, batch_size, d_rows=None, status=None):
        ops.require_cuda()
        self._features = features.contiguous()
        self._indices = indices.to(torch.int32).contiguous()
        self.spatial_shape = [int(s) for s in spatial_shape]
        self.batch_size = int(batch_size)
        dev = self._features.device
        self.d_rows = d_rows if d_rows is not None else torch.tensor([features.shape[0]], dtype=torch.int32, device=dev)
        self.status = status if status is not None else torch.zeros((1,), dtype=torch.int32, device=dev)
        self.indice_dict = {}
        self._index = None  # hash index over self._indices
        self.row_cap_factor = 8
        self._split = None  # fp16 hi/lo planes [2, cap, C8] when the layer chain runs in split form
        self._channels = self._features.shape[1]

    # exact-shape views (synchronise)
    def num_rows(self):
        return int(self.d_rows.item())

    @property
    def features(self):
        if self._features is None:      # split-row chain: reconstruct fp32 (hi + lo/2048) for API-compat consumers
            return ops.split_rows_float(self._split, self._channels)[: self.num_rows()]
        return self._features[: self.num_rows()]

    def features_cap(self):
        """capacity-sized fp32 feature matrix (no sync)."""
        if self._features is None:
            return ops.split_rows_float(self._split, self._channels)
        return self._features

    def split_planes(self):
        if self._split is None:
            self._split = ops.features_to_split(self._features, self.d_rows, self.status)
        return self._split

    @property
    def indices(self):
        return self._indices[: self.num_rows()]

    @property
    def rows_cap(self):
        return self._features.shape[0] if self._features is not None else self._split.shape[1]

    @property
    def device(self):
        return self._indices.device

    def hash_index(self):
        if self._index is None:
            self._index = ops.hash_build(ops.HashIndex(self.rows_cap, self.device), self._indices,
                                         self.d_rows, self.batch_size, self.spatial_shape, self.status)
        return self._index

    def _derive(self, features, indices=None, spatial_shape=None, d_rows=None, index=None, split=None, channels=None):
        t = SparseConvTensor.__new__(SparseConvTensor)
        t._features = features
        t._split = split
        t._channels = channels if channels is not None else (features.shape[1] if features is not None else None)
        t._indices = self._indices if indices is None else indices
        t.spatial_shape = self.spatial_shape if spatial_shape is None else spatial_shape
        t.batch_size = self.batch_size
        t.d_rows = self.d_rows if d_rows is None else d_rows
        t.status = self.status
        t.indice_dict = self.indice_dict
        t._index = index if indices is not None else self._index
        t.row_cap_factor = self.row_cap_factor
        return t

    def dense(self):
        """[B, C, D, H, W] like spconv's scatter_nd + permute (cmn.py:112)."""
        feats = self._features if self._features is not None else ops.split_rows_float(self._split, self._channels)
        C = feats.shape[1]
        D, H, W = self.spatial_shape
        bev = torch.zeros((self.batch_size, H, W, D * C), dtype=torch.float32, device=feats.device)
        ops.sparse_to_bev(feats, self._indices, self.d_rows, C, D, H, W, bev)
        # internal NHWC (d, c) order -> reference [B, C, D, H, W]
        return bev.view(self.batch_size, H, W, D, C).permute(0, 4, 3, 1, 2).contiguous()

    def check_status(self):
        ops._lib.raise_on_status(self.status)


class _SparseConvBase(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, bias, indice_key, subm):
        super().__init__()
        ks = (kernel_size,) * 3 if isinstance(kernel_size, int) else tuple(kernel_size)
        st = (stride,) * 3 if isinstance(stride, int) else tuple(stride)
        pd = (padding,) * 3 if isinstance(padding, int) else tuple(padding)
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride, self.padding = ks, st, pd
        self.indice_key, self.subm = indice_key, subm
        # spconv-v1.0 weight layout: (*kernel_size, in, out)
        self.weight = nn.Parameter(torch.empty(*ks, in_channels, out_channels))
        bound = 1.0 / (in_channels * ks[0] * ks[1] * ks[2]) ** 0.5
        nn.init.uniform_(self.weight, -bound, bound)
        self.bias = nn.Parameter(torch.zeros(out_channels)) if bias else None
        self.precision = ops.DEFAULT_PRECISION
        if not (ks in ((3, 3, 3), (1, 1, 1))):
            raise NotImplementedError("kernel sizes used by SA-SSD: 3x3x3 and 1x1x1")
        if ks == (3, 3, 3) and not subm and (st != (2, 2, 2) or pd != (1, 1, 1)):
            raise NotImplementedError("strided SparseConv3d: k=3, s=2, p=1 (cmn.py:170)")

    def _rulebook(self, x):
        key = self.indice_key
        if key is not None and key in x.indice_dict:
            rb = x.indice_dict[key]
            if rb.event is not None:      # built on a side stream: order this stream after it
                torch.cuda.current_stream().wait_event(rb.event)
            return rb
        if self.subm:
            nbr, tmask = ops.rulebook_subm(x._indices, x.d_rows, x.spatial_shape, x.hash_index())
            rb = Rulebook(nbr, x._indices, x.d_rows, x.spatial_shape, tile_mask=tmask)
        else:
            D, H, W = ops.conv_out_shape(x.spatial_shape)
            cap = min(int(x.rows_cap * x.row_cap_factor), x.batch_size * D * H * W)
            co, dn, nbr, so, tmask = ops.rulebook_conv(x._indices, x.d_rows, x.batch_size, x.spatial_shape,
                                                       x.hash_index(), max(cap, 1), x.status)
            rb = Rulebook(nbr, co, dn, so, tile_mask=tmask)
        if key is not None:
            x.indice_dict[key] = rb
        return rb

    def forward(self, x, scale=None, shift=None, relu=False):
        w = self.weight
        taps = self.kernel_size[0] * self.kernel_size[1] * self.kernel_size[2]
        wp = w.detach().reshape(taps, self.in_channels, self.out_channels).contiguous()
        if shift is None and self.bias is not None:
            shift = self.bias.detach()
        if self.precision == ops.PREC_F16X3 and SPLIT_ROWS and self.out_channels <= 64:
            # split-row chain: cp.async-fed tensor-core kernel (csrc/spconv_split.cu), output stays split
            planes = x.split_planes()
            if taps == 1:
                out, _ = ops.spconv_split(planes, wp, scale, shift, relu, self.out_channels, x.rows_cap,
                                          d_rows=x.d_rows, status=x.status)
                return x._derive(None, split=out, channels=self.out_channels)
            rb = self._rulebook(x)
            out, _ = ops.spconv_split(planes, wp, scale, shift, relu, self.out_channels, rb.nbr.shape[0], nbr=rb.nbr,
                                      d_rows=rb.d_rows_out, tile_mask=rb.tile_mask, status=x.status)
            if self.subm:
                return x._derive(None, split=out, channels=self.out_channels)
            return x._derive(None, indices=rb.coors_out, spatial_shape=rb.shape_out, d_rows=rb.d_rows_out,
                             index=rb.index_out, split=out, channels=self.out_channels)
        if x._features is None:
            x = x._derive(ops.split_rows_float(x._split, x._channels))
        if taps == 1:
            out = torch.empty((x.rows_cap, self.out_channels), dtype=torch.float32, device=wp.device)
            ops.gconv(x._features, wp, scale, shift, out, mode=ops.GCONV_ROWS, taps=1, cin=self.in_channels,
                      cout=self.out_channels, relu=relu, d_rows=x.d_rows, rows_cap=x.rows_cap,
                      precision=self.precision, status=x.status)
            return x._derive(out)
        rb = self._rulebook(x)
        cap = rb.nbr.shape[0]
        out = torch.empty((cap, self.out_channels), dtype=torch.float32, device=wp.device)
        ops.gconv(x._features, wp, scale, shift, out, mode=ops.GCONV_TABLE, taps=27, cin=self.in_channels,
                  cout=self.out_channels, relu=relu, nbr=rb.nbr, d_rows=rb.d_rows_out, rows_cap=cap,
                  precision=self.precision, status=x.status)
        if self.subm:
            return x._derive(out)
        return x._derive(out, indices=rb.coors_out, spatial_shape=rb.shape_out, d_rows=rb.d_rows_out,
                         index=rb.index_out)


class SubMConv3d(_SparseConvBase):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, bias=True, indice_key=None):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, bias, indice_key, subm=True)


class SparseConv3d(_SparseConvBase):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, bias=True, indice_key=None):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, bias, indice_key, subm=False)


def _versions(*tensors):
    return tuple((t.data_ptr(), t._version) for t in tensors)


def fold_bn(bn):
    """eval-mode BatchNorm -> (scale, shift): y = x*scale + shift.  Cached on the module and
    refreshed when any of its tensors changes (load_state_dict bumps the versions)."""
    ver = _versions(bn.weight, bn.bias, bn.running_mean, bn.running_var)
    cached = getattr(bn, "_sassd_fold", None)
    if cached is not None and cached[0] == ver:
        return cached[1], cached[2]
    with torch.no_grad():
        scale = (bn.weight.detach() / torch.sqrt(bn.running_var.detach() + bn.eps)).float().contiguous()
        shift = (bn.bias.detach() - bn.running_mean.detach() * scale).float().contiguous()
    bn._sassd_fold = (ver, scale, shift)
    return scale, shift


class SparseSequential(nn.Sequential):
    """spconv.SparseSequential: sparse modules get the tensor, dense modules are applied to
    ``.features``.  The conv -> BatchNorm1d(eval) -> ReLU pattern of cmn.py:145-173 is
    executed as one kernel (BN folded into the epilogue)."""

    def forward(self, x):
        mods = list(self._modules.values())
        i = 0
        while i < len(mods):
            m = mods[i]
            if isinstance(m, _SparseConvBase):
                bn = mods[i + 1] if i + 1 < len(mods) and isinstance(mods[i + 1], nn.BatchNorm1d) else None
                if bn is not None and not bn.training and m.bias is None:
                    relu = i + 2 < len(mods) and isinstance(mods[i + 2], nn.ReLU)
                    scale, shift = fold_bn(bn)
                    x = m(x, scale, shift, relu)
                    i += 3 if relu else 2
                    continue
                x = m(x)
            else:
                feats = x._features if x._features is not None else ops.split_rows_float(x._split, x._channels)
                x = x._derive(m(feats))
            i += 1
        return x
