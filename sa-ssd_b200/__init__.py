"""sassd_b200 — H100 (sm_90a) implementation of the SA-SSD point-cloud inference
hot path (voxelize -> sparse 3D conv backbone -> BEV neck -> SSD rotate head ->
PSWarp rescoring -> rotated NMS) behind the reference's mmdet.models operator
API.  Hand-written sm_90a CUDA lives in ``csrc/`` behind the C ABI declared in
``include/sassd_b200.h``; this package is the host-side mirror of the reference
interface.  Import name: ``sassd_b200`` (alias of the ``sa-ssd_b200/`` directory).
"""
__version__ = "0.1.0"

from .config import Config, obj_from_dict  # noqa: F401
from .results import Calibration, kitti_bbox2results  # noqa: F401


def get_official_eval_result(gt_annos, dt_annos, current_classes, difficultys=(0, 1, 2)):
    """KITTI official evaluation table (kitti_eval.get_official_eval_result; imported on first use because it
    loads the native library)."""
    from .kitti_eval import get_official_eval_result as impl
    return impl(gt_annos, dt_annos, current_classes, list(difficultys))



def build_from_config(cfg, device="cuda", data_key="val"):
    """Build detector + data-side objects from a reference-style config
    (tools/test.py:128-139, mmdet/datasets/utils.py:95-121)."""
    from . import anchors as A
    from . import voxel_generator as V
    from .builder import build_detector
    model = build_detector(cfg.model, train_cfg=cfg.get("train_cfg"), test_cfg=cfg.test_cfg).to(device)
    d = cfg.data[data_key]
    vg = obj_from_dict(d["generator"], V, dict(device=device))
    gens = {k: obj_from_dict(v, A) for k, v in d["anchor_generator"].items()}
    aset = A.AnchorSet(gens, vg, out_size_factor=d.get("out_size_factor", 8),
                       anchor_area_threshold=d.get("anchor_area_threshold", 1), device=device)
    model.class_names = list(d.get("class_names", ["Car"]))
    model.attach_data_pipeline(vg, aset)
    return model, vg, aset
