"""Distinct checkpoints of configs/car_cfg.py for the checkpoint-sweep tests and timing tools: seed 0's synthetic
weights (checkpoint.make_synthetic_state_dict, the only ones whose BatchNorm statistics are calibrated) with auxiliary
head weights (the draws of tests/test_point_aux.py's _aux_weights), every conv and linear weight then scaled element by
element by 1 + WEIGHT_NOISE * N(0, 1) under a generator seed of its own."""
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAR_CFG = os.path.join(ROOT, "configs", "car_cfg.py")
WEIGHT_NOISE = 0.1


def aux_weights(seed=7):
    import torch
    g = torch.Generator().manual_seed(seed)
    return {"neck.point_fc.weight": torch.randn(64, 160, generator=g) / np.sqrt(160.0),
            "neck.point_cls.weight": torch.randn(1, 64, generator=g) / 8.0,
            "neck.point_reg.weight": torch.randn(3, 64, generator=g) / 8.0}


def checkpoint_state_dict(seed):
    """The checkpoint of ``seed`` (a positive integer; each seed gives different weights)."""
    import torch
    from sassd_b200 import checkpoint
    sd = checkpoint.make_synthetic_state_dict(0, 1)
    sd.update(aux_weights())
    g = torch.Generator().manual_seed(int(seed))
    for k in sorted(sd):
        if k.endswith(".weight") and sd[k].dim() >= 2:
            sd[k] = sd[k] * (1.0 + WEIGHT_NOISE * torch.randn(sd[k].shape, generator=g))
    return sd


def build(device):
    """A car_cfg detector with its data pipeline, on ``device``."""
    import sassd_b200 as S
    model, _, _ = S.build_from_config(S.Config.fromfile(CAR_CFG), device=device)
    return model
