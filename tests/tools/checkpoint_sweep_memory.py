"""Where a checkpoint sweep's device memory goes: one step eager and one captured step (a detect_stream slot) of
CheckpointSweep at K = 1, 2, 4 checkpoints, beside a single model's, at batch 16 of full sweeps with the losses (the
frustum-crop KITTI kind).

    python tests/tools/checkpoint_sweep_memory.py [--batch 16] [--ks 1 2 4]

Per case it prints torch.cuda.memory_allocated after each member's network (forward_voxels), the step's peak over
what was allocated before it, and for a captured step what it keeps: allocated and reserved memory after the capture,
split by allocator pool (the default pool and each CUDA graph's private pool, from torch.cuda.memory_snapshot).  The
card's name and power limit are read in the same run."""
import argparse
import gc
import os
import sys
import tempfile
import shutil

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

GB = float(1 << 30)


def release():
    import torch
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def pools():
    """{pool id: (reserved GB, allocated GB)} of the caching allocator's segments."""
    import torch
    out = {}
    for seg in torch.cuda.memory_snapshot():
        key = str(tuple(seg.get("segment_pool_id", (0, 0))))
        r, a = out.get(key, (0.0, 0.0))
        out[key] = (r + seg["total_size"] / GB, a + seg["allocated_size"] / GB)
    return {k: "%.2f/%.2f" % v for k, v in out.items()}


def main(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--batch", type=int, default=16)
    p.add_argument("--ks", type=int, nargs="+", default=[1, 2, 4])
    args = p.parse_args(argv)
    import torch
    from sassd_b200 import checkpoint, detectors as D
    from sassd_b200.kitti_data import KittiSplit
    from tests.checkpoint_weights import build, checkpoint_state_dict
    from tests.tools.checkpoint_sweep_timing import card, write_root
    print(card(), flush=True)
    tmp = tempfile.mkdtemp()
    try:
        write_root(os.path.join(tmp, "k"), args.batch)
        split = KittiSplit(os.path.join(tmp, "k"), "val", "velodyne", gt_classes=["Car"])
        frames = [split.frame(i) for i in split.ids]
        kw = dict(frustum_planes=[split.planes(m["calib"], m["img_shape"]) for _, m, _ in frames],
                  metas=[m for _, m, _ in frames], gt_bboxes=[g[0] for _, _, g in frames],
                  gt_labels=[g[1] for _, _, g in frames])
        pts = [f[0] for f in frames]
        models = []
        for seed in range(1, max(args.ks) + 1):
            m = build("cuda:0")
            checkpoint.load_state_dict_into(m, checkpoint_state_dict(seed))
            models.append(m)
        trace = []
        fv = D.SingleStageDetector.forward_voxels

        def traced(self, *a, **k):
            r = fv(self, *a, **k)
            trace.append(torch.cuda.memory_allocated() / GB)
            return r
        D.SingleStageDetector.forward_voxels = traced
        cases = [("single", models[0])] + [("sweep K=%d" % K, D.CheckpointSweep(models[:K])) for K in args.ks]
        for name, obj in cases:
            for captured in (False, True):
                release()
                trace.clear()
                torch.cuda.reset_peak_memory_stats()
                a0, r0 = torch.cuda.memory_allocated() / GB, torch.cuda.memory_reserved() / GB
                if captured:
                    run = D._run_step if obj is models[0] else D._sweep_step
                    slot = D._GraphedStep(obj, args.batch, 131072, crop=D.CROP_FRUSTUM, kitti=True, losses=True,
                                          run_step=run)
                else:
                    obj.forward_points(pts, **kw)
                torch.cuda.synchronize()
                a1, r1 = torch.cuda.memory_allocated() / GB, torch.cuda.memory_reserved() / GB
                peak = torch.cuda.max_memory_allocated() / GB
                print("%-10s %-8s before %.2f GB; peak +%.2f; after: allocated +%.2f, reserved +%.2f; "
                      "after each network %s; pools (reserved/allocated GB) %s" % (
                          name, "captured" if captured else "eager", a0, peak - a0, a1 - a0, r1 - r0,
                          " ".join("%.2f" % t for t in trace), pools()), flush=True)
                if captured:
                    del slot
    finally:
        shutil.rmtree(tmp, ignore_errors=True)


if __name__ == "__main__":
    main()
