"""Time training-time augmentation with and without road planes on the GPU:
``python tests/tools/augment_plane_timing.py [--frames 512] [--reps 2]``.

Builds the synthetic root of tests/kitti_root.py with tests/kitti_planes.py's plane files, prepares it with
sassd_b200.create_data and lists ``--frames`` train frames (its labelled frames, cycled).  Then, ``--reps`` times,
alternating car_cfg without and with data.train.with_plane, at batch 1 and 16, with the card's name and power limit,
it reports:
  * the driver's frame rate (python -m sassd_b200.augment on full sweeps), after a 64-frame warm-up run;
  * sassd_augment_assemble's GPU time per frame (CUDA events around each launch, ops.PROFILE);
and once, the host time per frame of the plane correction alone (augment.plane_shift on each frame's sampled boxes).
"""
import argparse
import contextlib
import io
import os
import re
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def _driver(A, ops, cfg, root, batch, frames):
    """One driver run after a warm-up run: (its frames/s, sassd_augment_assemble ms per frame)."""
    with contextlib.redirect_stdout(io.StringIO()):
        A.main([cfg, "--data-root", root, "--seed", "0", "--batch", str(batch), "--frames", "64"])
    ops.PROFILE = []
    out = io.StringIO()
    with contextlib.redirect_stdout(out):
        A.main([cfg, "--data-root", root, "--seed", "0", "--batch", str(batch)])
    fps = float(re.search(r"([0-9.]+) frames/s", out.getvalue()).group(1))      # the driver's own rate
    asm = sum(e0.elapsed_time(e1) for name, _l, e0, e1 in ops.PROFILE if name == "sassd_augment_assemble")
    ops.PROFILE = None
    return fps, asm / frames


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    from sassd_b200 import augment as A
    from sassd_b200 import create_data as CD
    from sassd_b200 import ops
    from sassd_b200.config import Config
    from sassd_b200.kitti_data import KittiSplit, labelled_boxes, read_label, read_plane
    from tests import kitti_planes as KP
    from tests import kitti_root as KR
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)
    work = tempfile.mkdtemp(prefix="aug_plane_timing_")
    try:
        root = os.path.join(work, "kitti")
        KR.write_tree(root)
        KP.write_planes(root)
        with contextlib.redirect_stdout(io.StringIO()):
            assert CD.main(["--data-root", root]) == 0
        ids = [KR.TRAIN[i % len(KR.TRAIN)] for i in range(args.frames)]
        with open(os.path.join(root, "ImageSets", "train.txt"), "w") as fh:
            fh.write("".join("%06d\n" % i for i in ids))
        cfgs = {False: os.path.join(ROOT, "configs", "car_cfg.py"), True: os.path.join(work, "car_plane_cfg.py")}
        with open(cfgs[False]) as fh:
            text = fh.read()
        with open(cfgs[True], "w") as fh:
            fh.write(text + "\ndata['train']['with_plane'] = True\n")
        for rep in range(args.reps):
            for with_plane in (False, True):
                for batch in (1, 16):
                    fps, asm = _driver(A, ops, cfgs[with_plane], root, batch, len(ids))
                    print("run %d planes %-5s batch %2d: driver %.1f frames/s, sassd_augment_assemble %.4f ms per "
                          "frame" % (rep, with_plane, batch, fps, asm))
        # host plane correction alone, on the frames' sampled database boxes
        aug = A.build_augmentor(Config.fromfile(cfgs[False]), root, rng=np.random.RandomState(0), device=None)
        split = KittiSplit(root, "train", lidar="velodyne_reduced")
        work_items = []
        for i in ids:
            meta = split.meta(i)
            g = labelled_boxes(read_label(split.path("label_2", i, "txt")), meta["calib"])
            plan = aug.draw(g[0], g[1], ["Car"])
            if plan["records"]:
                work_items.append((np.stack([aug.records[r]["box3d_lidar"] for r in plan["records"]]),
                                   read_plane(split.path("planes", i, "txt")), meta["calib"]))
        t0 = time.perf_counter()
        for s, plane, calib in work_items:
            A.plane_shift(s, plane, calib)
        print("host plane correction: %.4f ms per frame" % ((time.perf_counter() - t0) * 1e3 / len(ids)))
    finally:
        shutil.rmtree(work, ignore_errors=True)


if __name__ == "__main__":
    main()
