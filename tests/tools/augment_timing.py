"""Time training-time augmentation on the GPU: ``python tests/tools/augment_timing.py [--frames 512]``.

Builds the synthetic root of tests/kitti_root.py, prepares it with sassd_b200.create_data, lists ``--frames`` train
frames (its labelled frames, cycled) and reports, at batch 1 and 16, with the card's name and power limit:
  * the driver's frame rate and read wait (python -m sassd_b200.augment on full sweeps, car_cfg);
  * the augment kernels' GPU time per frame (CUDA events around each launch, ops.PROFILE);
  * the host time per frame spent on the draws and box geometry (PointAugmentor.draw + finish_boxes).
"""
import argparse
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    args = ap.parse_args()
    import torch
    from sassd_b200 import augment as A
    from sassd_b200 import create_data as CD
    from sassd_b200 import ops
    from tests import kitti_root as KR
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)
    work = tempfile.mkdtemp(prefix="aug_timing_")
    try:
        root = os.path.join(work, "kitti")
        KR.write_tree(root)
        assert CD.main(["--data-root", root]) == 0
        ids = [KR.TRAIN[i % len(KR.TRAIN)] for i in range(args.frames)]
        with open(os.path.join(root, "ImageSets", "train.txt"), "w") as fh:
            fh.write("".join("%06d\n" % i for i in ids))
        cfg = os.path.join(ROOT, "configs", "car_cfg.py")
        for batch in (1, 16):
            A.main([cfg, "--data-root", root, "--seed", "0", "--batch", str(batch), "--frames", "64"])   # warm-up
            ops.PROFILE = []
            A.main([cfg, "--data-root", root, "--seed", "0", "--batch", str(batch)])
            torch.cuda.synchronize()
            per = {}
            for name, _label, e0, e1 in ops.PROFILE:
                per[name] = per.get(name, 0.0) + e0.elapsed_time(e1)
            ops.PROFILE = None
            print("batch %d kernels (ms per frame): %s" % (batch, {k: round(v / len(ids), 4) for k, v in per.items()}))
        # host draws and box geometry alone
        from sassd_b200.kitti_data import KittiSplit, labelled_boxes, read_label
        from sassd_b200.config import Config
        c = Config.fromfile(cfg)
        aug = A.build_augmentor(c, root, rng=np.random.RandomState(0), device=None)
        split = KittiSplit(root, "train", lidar="velodyne_reduced")
        gts = [labelled_boxes(read_label(split.path("label_2", i, "txt")), split.meta(i)["calib"]) for i in ids]
        t0 = time.perf_counter()
        for g in gts:
            plan = aug.draw(g[0], g[1], ["Car"])
            aug.finish_boxes(plan, -np.ones(len(plan["boxes"]), np.int64))
        print("host draws + box geometry: %.3f ms per frame" % ((time.perf_counter() - t0) * 1e3 / len(gts)))
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
