"""Generate tests/golden/loss_edges.npz by running the REFERENCE's own create_target_torch (NearestIouSimilarity and
RotateIou3dSimilarity), SSDRotateHead.loss and PSWarpHead.loss on the constructed edge cases of
tests/test_targets_edges.py: IoUs exactly at f32(pos / neg threshold) and one ulp either side for every class and at
PSWarp's 0.7, duplicate GT, maxima shared by several anchors, anchors tied across GT, a GT overlapping nothing, a class
absent from a frame, a GT of no anchor class, a wholly masked class; head outputs at extreme logits, at the smooth-L1
knee and with yaws up to +-100 rad.  Run once where the original project is checked out and __graft_entry__.build()
made oracle/_ref/ (make_golden_loss.py's stubs); the fixture is committed.  The inputs are stored with their sha256
(tests/test_targets_edges.inputs_digest), so a test can tell that the constructions still produce them.

    python tests/golden/make_golden_loss_edges.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from make_golden_loss import cfg_dict, install_stubs  # noqa: E402
from tests import test_targets_edges as E  # noqa: E402


def main():
    inp = E.fixture_inputs()
    digest = E.inputs_digest(inp)
    install_stubs()
    from mmdet.core.bbox3d.target_ops import create_target_torch
    from mmdet.models.single_stage_heads import ssd_rotate_head as RH
    from mmdet.ops.iou3d import iou3d_utils
    rc, pc = E.rpn_case(), E.pswarp_case()
    B, classes, P = 2, E.CLASSES, E.P
    cfg = cfg_dict(classes)
    gt_t = [torch.from_numpy(g) for g in rc["gts"]]
    lb_t = [torch.from_numpy(l) for l in rc["gt_labels"]]
    anchors = {c: torch.from_numpy(rc["anchors"][:, i * P:(i + 1) * P].copy()) for i, c in enumerate(classes)}
    masks = {c: torch.from_numpy(rc["mask"][:, i * P:(i + 1) * P].copy()) for i, c in enumerate(classes)}
    out = dict(inp)
    L, T, M = [], [], []
    for c in classes:
        gt_mask = [torch.BoolTensor(t == c) for t in rc["gt_types"]]
        lab, tgt, iou = [], [], []
        for b in range(B):
            l_, t_, m_ = create_target_torch(anchors[c][b], masks[c][b], gt_t[b], lb_t[b], gt_mask[b],
                                             similarity_fn=iou3d_utils.NearestIouSimilarity(),
                                             box_encoding_fn=RH.second_box_encode,
                                             matched_threshold=E.THR[c][0], unmatched_threshold=E.THR[c][1],
                                             box_code_size=7)
            lab.append(l_.numpy()); tgt.append(t_.numpy())
            mm = np.zeros(P, np.float32)
            if len(m_) == int(masks[c][b].sum()):
                mm[masks[c][b].numpy()] = m_.numpy()
            iou.append(mm)
        L.append(np.stack(lab)); T.append(np.stack(tgt)); M.append(np.stack(iou))
    out.update(rpn_labels=np.concatenate(L, 1), rpn_targets=np.concatenate(T, 1), rpn_ious=np.concatenate(M, 1))
    head = RH.SSDRotateHead(num_class=len(classes), num_output_filters=8, num_anchor_per_loc=2, use_sigmoid_cls=True,
                            encode_rad_error_by_sin=True, use_direction_classifier=True, box_code_size=7)
    rpn = head.loss(torch.from_numpy(inp["box_preds"]), torch.from_numpy(inp["cls_preds"]),
                    torch.from_numpy(inp["dir_preds"]), gt_t, lb_t, list(rc["gt_types"]), anchors, masks, cfg.rpn)
    ps = RH.PSWarpHead(grid_offsets=(0., 40.), featmap_stride=.4, in_channels=8, num_class=1, num_parts=28)
    pgt = [torch.from_numpy(g) for g in pc["gts"]]
    ps_loss = ps.loss(torch.from_numpy(inp["ps_scores"]), pgt, None, [torch.from_numpy(x) for x in pc["guided"]],
                      cfg.extra)
    ps_lab, ps_iou = [], []
    for b in range(B):
        l_, _, m_ = create_target_torch(torch.from_numpy(pc["guided"][b]), None, pgt[b], None, None,
                                        similarity_fn=iou3d_utils.RotateIou3dSimilarity(),
                                        box_encoding_fn=RH.second_box_encode, matched_threshold=0.7,
                                        unmatched_threshold=0.7)
        ps_lab.append(l_.numpy()); ps_iou.append(m_.numpy())
    out.update(ps_labels=np.concatenate(ps_lab), ps_ious=np.concatenate(ps_iou))
    for k, v in list(rpn.items()) + list(ps_loss.items()):
        out["loss_" + k] = v.detach().numpy().astype(np.float32).reshape(1)
    out["inputs_sha256"] = np.array(digest)
    print({k: float(v) for k, v in list(rpn.items()) + list(ps_loss.items())},
          "labels:", np.unique(out["rpn_labels"], return_counts=True), np.unique(out["ps_labels"], return_counts=True))
    np.savez_compressed(os.path.join(HERE, "loss_edges.npz"), **out)


if __name__ == "__main__":
    main()
