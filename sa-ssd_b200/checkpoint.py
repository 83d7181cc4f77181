"""Checkpoint format of the reference + synthetic weights for offline work.

Reference format (tools/train_utils/__init__.py:125-180): ``torch.save`` of
``{'epoch','it','model_state','optimizer_state','version'}``; ``model_state``
keys carry an optional ``module.`` prefix (saved through the DataParallel
wrapper, tools/test.py:142-143) and are copied only where name and shape match.

Parameter names (SURVEY.md §8b): ``neck.backbone.{conv0,down0,...}.{0,3,6}.weight``
in spconv-v1 layout ``[kz,ky,kx,Cin,Cout]`` with BatchNorm1d at ``.{1,4,7}``;
``neck.fcn.conv{0..7}.weight`` / ``neck.fcn.bn{0..7}.*``; ``rpn_head.conv_{cls,box,
dir_cls}.{weight,bias}``; ``extra_head.convs.{0,1,3}.*``.  The aux-network keys
(``neck.point_fc/point_cls/point_reg``, cmn.py:27-29) are loaded like the others and used by
``SpMiddleFHD.forward(is_test=False)`` / ``forward_points(point_outputs=True)``;
``make_synthetic_state_dict`` does not set them.
"""
import math
import os

import torch

# (name, Cin, Cout, kernel, expected active taps used to scale the synthetic init)
_SPARSE_LAYERS = [
    ("conv0.0", 4, 16, 3, 4.0), ("conv0.3", 16, 16, 3, 4.0),
    ("down0.0", 16, 32, 3, 3.0),
    ("conv1.0", 32, 32, 3, 8.0), ("conv1.3", 32, 32, 3, 8.0),
    ("down1.0", 32, 64, 3, 5.0),
    ("conv2.0", 64, 64, 3, 9.0), ("conv2.3", 64, 64, 3, 9.0), ("conv2.6", 64, 64, 3, 9.0),
    ("down2.0", 64, 64, 3, 6.0),
    ("conv3.0", 64, 64, 3, 14.0), ("conv3.3", 64, 64, 3, 14.0), ("conv3.6", 64, 64, 3, 14.0),
    ("extra_conv.0", 64, 64, 1, 1.0),
]


def _bn(sd, prefix, c, g):
    sd[prefix + ".weight"] = torch.rand(c, generator=g) * 0.5 + 0.75
    sd[prefix + ".bias"] = torch.randn(c, generator=g) * 0.1
    sd[prefix + ".running_mean"] = torch.randn(c, generator=g) * 0.1
    sd[prefix + ".running_var"] = torch.rand(c, generator=g) + 0.5


_CALIB = os.path.join(os.path.dirname(os.path.abspath(__file__)), "synth_calib.npz")


def make_synthetic_state_dict(seed=0, num_class=1, num_filters=256, bev_in=320, num_parts=28,
                              cls_gain=2.5, cls_bias=-2.95, ps_gain=1.0, ps_offset=1.0, tap_decay=0.3,
                              calibrated=True):
    """Random-but-fixed weights in the reference's state_dict naming.

    No checkpoint is reachable offline, so benchmarks and parity tests use these.
    Scales follow a He-style rule on the *expected active* fan-in so activations
    stay O(1) through the 13 sparse + 8 dense layers; BatchNorm affine parameters are
    randomised and, for seed 0, the running statistics come from a calibration pass over
    synthetic frames (synth_calib.npz) so that BN is neither an identity nor a blow-up.  ``cls_gain``/``cls_bias``
    shape the RPN class logits so that, like a trained detector, only a few
    hundred anchors per frame pass the 0.1 guided-anchor threshold; ``ps_gain``/``ps_offset``
    centre the PSWarp logits on the 0.3 rescoring threshold (about half of the candidates pass)
    (constants picked by tests/tools/calibrate_synthetic_weights.py).  The head gains are kept
    moderate on purpose: a logit is a linear read-out of the neck map, whose two fp32 evaluation
    orders (CUDA kernel vs CPU oracle) already differ by ~1e-4 relative, so a logit spread of
    ~0.3-0.8 is what lets "class scores within 1e-4" be a statement about the kernels and not
    about the conditioning of random weights.
    """
    g = torch.Generator().manual_seed(int(seed))
    sd = {}
    p = "neck.backbone."
    for name, cin, cout, k, taps in _SPARSE_LAYERS:
        w = torch.randn(k, k, k, cin, cout, generator=g)
        if k == 3 and not name.startswith("down"):
            # Submanifold layers: a site with all 27 neighbours active sums three times the variance of a typical one
            # (~9 active), layer after layer, which gives untrained weights activations with a far heavier tail
            # (max / std ~ 80) than any trained, BatchNorm-regularised network has - and every absolute error of a
            # layer scales with that max.  The off-centre taps are therefore weaker than the centre tap
            # (tap_decay), like a trained 3x3x3 kernel's energy profile: dense and sparse neighbourhoods then differ
            # by ~1.2x per layer instead of 1.7x.
            decay = torch.full((3, 3, 3, 1, 1), tap_decay)
            decay[1, 1, 1] = 1.0
            w = w * decay
            eff = 1.0 + (taps - 1.0) * tap_decay ** 2
        else:
            eff = taps
        sd[p + name + ".weight"] = w * math.sqrt(2.0 / (cin * eff))
        blk, idx = name.split(".")
        _bn(sd, "%s%s.%d" % (p, blk, int(idx) + 1), cout, g)
    p = "neck.fcn."
    for i in range(8):
        cin = bev_in if i == 0 else num_filters
        k = 1 if i == 7 else 3
        eff = cin * k * k * (0.06 if i == 0 else 1.0)   # conv0 sees a ~4-6 % occupied map
        sd["%sconv%d.weight" % (p, i)] = torch.randn(num_filters, cin, k, k, generator=g) * math.sqrt(2.0 / eff)
        _bn(sd, "%sbn%d" % (p, i), num_filters, g)
    p = "rpn_head."
    na = 2 * num_class
    s = math.sqrt(1.0 / num_filters)
    sd[p + "conv_cls.weight"] = torch.randn(na * num_class, num_filters, 1, 1, generator=g) * s * cls_gain
    # three classes triple the anchors and take the max over classes: lower the bias so that the guided-anchor and
    # detection counts stay in the range of a trained model (and below the fixed result capacity)
    sd[p + "conv_cls.bias"] = torch.randn(na * num_class, generator=g) * 0.05 + cls_bias - (0.9 if num_class > 1 else 0.0)
    sd[p + "conv_box.weight"] = torch.randn(na * 7, num_filters, 1, 1, generator=g) * s * 1.0
    sd[p + "conv_box.bias"] = torch.randn(na * 7, generator=g) * 0.02
    sd[p + "conv_dir_cls.weight"] = torch.randn(na * 2, num_filters, 1, 1, generator=g) * s
    sd[p + "conv_dir_cls.bias"] = torch.randn(na * 2, generator=g) * 0.05
    p = "extra_head."
    sd[p + "convs.0.weight"] = torch.randn(num_parts, num_filters, 3, 3, generator=g) * math.sqrt(2.0 / (num_filters * 9))
    _bn(sd, p + "convs.1", num_parts, g)
    sd[p + "convs.3.weight"] = (torch.randn(num_parts, num_parts, 1, 1, generator=g) * ps_gain - ps_offset) * \
        math.sqrt(2.0 / num_parts)
    if calibrated and seed == 0 and num_filters == 256 and bev_in == 320 and os.path.isfile(_CALIB):
        # BatchNorm running statistics as training-mode BN would have recorded them on synthetic
        # frames (tests/tools/calibrate_synthetic_weights.py): keeps activations O(1) in all 22 layers
        import numpy as np
        with np.load(_CALIB) as z:
            for k in z.files:
                sd[k] = torch.from_numpy(z[k].copy())
    return sd


def save_checkpoint(state_dict, filename, epoch=0, it=0, module_prefix=False):
    """Write the reference's checkpoint dict (train_utils/__init__.py:125-152)."""
    ms = {("module." + k if module_prefix else k): v for k, v in state_dict.items()}
    torch.save({"epoch": epoch, "it": it, "model_state": ms, "optimizer_state": None,
                "version": "sassd_b200"}, filename)


def load_params_from_file(model, filename, to_cpu=False, verbose=False, allow_pickle=False):
    """Mirror of tools/train_utils/__init__.py:154-180: copy every key whose name
    (after stripping an optional ``module.`` prefix) and shape match; report the
    rest.  Returns (n_loaded, missing_keys).  The reference format holds tensors and plain scalars only, so the
    file is read with ``weights_only=True``; ``allow_pickle=True`` opts into arbitrary pickles for legacy files
    from a trusted source."""
    if not os.path.isfile(filename):
        raise FileNotFoundError(filename)
    ckpt = torch.load(filename, map_location="cpu" if to_cpu else None, weights_only=not allow_pickle)
    disk = ckpt["model_state"] if isinstance(ckpt, dict) and "model_state" in ckpt else ckpt
    return load_state_dict_into(model, disk, verbose=verbose)


def load_state_dict_into(model, disk, verbose=False):
    own = model.state_dict()
    update = {}
    for key, val in disk.items():
        k = key[7:] if key.startswith("module.") else key
        if k in own and tuple(own[k].shape) == tuple(val.shape):
            update[k] = val
    own.update(update)
    model.load_state_dict(own)
    missing = [k for k in own if k not in update]
    if verbose:
        for k in missing:
            print("Not updated weight %s: %s" % (k, str(tuple(own[k].shape))))
        print("==> Done (loaded %d/%d)" % (len(update), len(own)))
    if hasattr(model, "refresh_packed_weights"):
        model.refresh_packed_weights()
    return len(update), missing
