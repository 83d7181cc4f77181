"""Cost of validation losses in the KITTI driver (python -m sassd_b200.test --losses) on a synthetic labelled tree.

    python tests/tools/val_loss_timing.py [--frames 256] [--reps 2] [--json FILE]

Writes a KITTI-layout tree of ``--frames`` full synthetic sweeps (32 distinct clouds, repeated), the two calibrations
of tests/golden/frustum.npz alternating, PNG headers of two sizes and label files of 1-6 cars per frame (synthetic
weights, including the auxiliary head's).  Reports, with the card's name and power limit read in the same run:
  * driver frames/s with and without ``--losses`` at batch 1 and 16 (full sweeps cropped on the device, KITTI
    formatter on the device), the two runs alternated ``--reps`` times;
  * the GPU time of one captured step of the loss kind against the plain crop + KITTI kind at the same batch (CUDA
    events around one slot's replay, median of 20, the slot's static inputs holding the first batch).
"""
import argparse
import gc
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    import sassd_b200 as S
    from sassd_b200 import checkpoint, kitti_data as K
    from sassd_b200 import test as T
    from sassd_b200.frustum import camera_frustum_planes
    from sassd_b200.results import annos_to_kitti_label, kitti_bbox2results
    from sassd_b200.synth import synth_cloud
    from tests.test_kitti_data import write_split
    from tests.test_kitti_format import _calib_txt, _calibs
    from tests.test_point_aux import _aux_weights
    from tests.tools.kitti_driver_timing import power_limit

    calibs = _calibs(os.path.join(ROOT, "tests", "golden"))
    shapes = [(375, 1242), (370, 1224)]
    clouds = [synth_cloud(2000 + k, fov_deg=180.0) for k in range(32)]
    out = dict(gpu=torch.cuda.get_device_name(0), power_limit=power_limit(), frames=args.frames)
    rng = np.random.default_rng(0)
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "kitti")
        ids = list(range(args.frames))
        write_split(root, ids, shapes, [_calib_txt(c) for c in calibs], [clouds[i % 32] for i in ids])
        split = K.KittiSplit(root, "val", "velodyne")
        for i in ids:
            n = int(rng.integers(1, 7))
            boxes = np.stack([rng.uniform(8, 40, n), rng.uniform(-6, 6, n), np.full(n, -1.7), np.full(n, 1.6),
                              np.full(n, 3.9), np.full(n, 1.56), rng.uniform(-3, 3, n)], 1).astype(np.float32)
            gt = kitti_bbox2results(boxes, np.ones(n, np.float32), np.zeros(n, np.int64), split.meta(i), ["Car"])
            with open(split.path("label_2", i, "txt"), "w") as fh:
                fh.write("".join(l + "\n" for l in annos_to_kitti_label(
                    dict(gt, dimensions=gt["dimensions"][:, [1, 2, 0]]))))
        sd = checkpoint.make_synthetic_state_dict(0, 1)
        sd.update(_aux_weights())
        ckpt = os.path.join(tmp, "w.pth")
        checkpoint.save_checkpoint(sd, ckpt)
        cfg = os.path.join(ROOT, "configs", "car_cfg.py")
        for B in (1, 16):
            for _ in range(args.reps):
                for losses in (False, True):
                    gc.collect()
                    torch.cuda.empty_cache()        # each run builds its own model and captured slots
                    res = T.run(T.parse_args([cfg, ckpt, "--data-root", root, "--batch", str(B)] +
                                             (["--losses"] if losses else [])), log=lambda *a, **k: None)
                    out.setdefault("driver_fps_b%d_%s" % (B, "losses" if losses else "plain"), []).append(
                        round(res["frames_per_s"], 1))

        gc.collect()
        torch.cuda.empty_cache()
        model, _, _ = S.build_from_config(S.Config.fromfile(cfg), device="cuda:0")
        checkpoint.load_params_from_file(model, ckpt)
        gsplit = K.KittiSplit(root, "val", "velodyne", gt_classes=["Car"])
        for B in (1, 16):
            frames = [gsplit.frame(i) for i in range(B)]
            pts, metas = [f[0] for f in frames], [f[1] for f in frames]
            planes = [camera_frustum_planes(m["calib"], m["img_shape"]) for m in metas]
            gts = ([f[2][0] for f in frames], [f[2][1] for f in frames])
            for losses in (False, True):
                item = (pts, planes, metas) + ((gts,) if losses else ())
                list(model.detect_stream([item] * 2, B, 131072, depth=1, crop=True, kitti=True, losses=losses))
                slot = model._stream_slots[0]
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                times = []
                for _ in range(20):
                    e0.record()
                    slot.graph.replay()
                    e1.record()
                    torch.cuda.synchronize()
                    times.append(e0.elapsed_time(e1))
                out["gpu_step_ms_b%d_%s" % (B, "losses" if losses else "plain")] = round(float(np.median(times)), 3)
    print(json.dumps(out))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
