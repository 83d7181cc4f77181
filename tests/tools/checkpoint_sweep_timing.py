"""Timing of a checkpoint sweep (python -m sassd_b200.test --checkpoints) against one driver run per checkpoint.

    python tests/tools/checkpoint_sweep_timing.py [--ks 4 10] [--frames 512] [--batches 1 16] [--losses both]
                                                  [--rounds 2] [--reps 20] [--json FILE]

Checkpoints: configs/car_cfg.py with seed 0's synthetic weights and the auxiliary head's, each scaled element by element
by 1 + 0.1 N(0, 1) under a seed of its own (tests/checkpoint_weights.py).  Frames: a synthetic labelled KITTI root
of ``--frames`` full sweeps (synth_cloud, 180 degrees, ~120 k points each) with the label rows of tests/kitti_root.py,
cropped on the device.  For each K, batch and loss setting, the sweep and the K single runs alternate in one process,
``--rounds`` times each, and every round reports:
  * wall: the driver's wall clock of the streamed detection (its own frames_per_s measure) and its read wait, summed
    over the K runs for the singles;
  * eval: the host time of the AP evaluation (official_eval_many for the sweep, official_eval per run);
  * memory: torch.cuda.max_memory_allocated over the run;
  * step: the GPU time of one captured step (CUDA events around ``reps`` back-to-back replays of the frustum-crop
    KITTI kind, with the losses when asked), for the sweep and summed over K single models.
The card's name and power limit are read in the same run (nvidia-smi --query-gpu)."""
import argparse
import gc
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
CFG = os.path.join(ROOT, "configs", "car_cfg.py")


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def write_root(root, n):
    """A labelled root of n full sweeps: ImageSets/val.txt, training/{velodyne,calib,image_2,label_2}."""
    from sassd_b200.synth import synth_cloud
    from tests.kitti_root import SHAPES, _rig, calib_text, label_lines, png_bytes
    os.makedirs(os.path.join(root, "ImageSets"))
    with open(os.path.join(root, "ImageSets", "val.txt"), "w") as fh:
        fh.write("".join("%06d\n" % i for i in range(n)))
    sub = os.path.join(root, "training")
    for d in ("velodyne", "calib", "image_2", "label_2"):
        os.makedirs(os.path.join(sub, d))
    for i in range(n):
        synth_cloud(1000 + i, fov_deg=180.0).tofile(os.path.join(sub, "velodyne", "%06d.bin" % i))
        with open(os.path.join(sub, "calib", "%06d.txt" % i), "w") as fh:
            fh.write(calib_text(i % 2))
        with open(os.path.join(sub, "image_2", "%06d.png" % i), "wb") as fh:
            fh.write(png_bytes(*SHAPES[(i // 2) % 2]))
        rows = label_lines(5 + i, _rig(i % 2), np.random.default_rng(1000 + i))
        with open(os.path.join(sub, "label_2", "%06d.txt" % i), "w") as fh:
            fh.write("".join(r + "\n" for r in rows))


class EvalClock:
    """Host time spent in kitti_eval.official_eval / official_eval_many during a driver run."""

    def __init__(self):
        from sassd_b200 import kitti_eval as KE
        self.s, self.inside = 0.0, False
        for name in ("official_eval", "official_eval_many"):
            fn = getattr(KE, name)
            setattr(KE, name, self._timed(fn))

    def _timed(self, fn):
        def run(*a, **k):          # official_eval calls official_eval_many: count the outer call only
            if self.inside:
                return fn(*a, **k)
            self.inside = True
            t0 = time.perf_counter()
            try:
                return fn(*a, **k)
            finally:
                self.s += time.perf_counter() - t0
                self.inside = False
        run.__wrapped__ = fn
        return run


def release():
    import torch
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def driver_run(argv, clock):
    import torch
    from sassd_b200 import test as T
    release()
    torch.cuda.reset_peak_memory_stats()
    clock.s = 0.0
    res = T.run(T.parse_args(argv), log=lambda *a, **k: None)
    return dict(wall_s=res["wall_s"], read_wait_s=res["read_wait_s"], eval_s=clock.s,
                max_memory_gb=torch.cuda.max_memory_allocated() / 2 ** 30)


def step_ms(obj, frames, planes, metas, gts, losses, reps):
    """GPU time of one captured step of the frustum-crop KITTI kind (with the losses when asked)."""
    import torch
    import sassd_b200 as S
    B = len(frames)
    obj.enable_cuda_graph(B, 131072)
    kw = dict(frustum_planes=planes, metas=metas)
    if losses:
        kw.update(gt_bboxes=[g[0] for g in gts], gt_labels=[g[1] for g in gts])
    obj.forward_points(frames, **kw)
    # a SingleStageDetector's kinds are (crop, kitti, point_outputs[, losses]), a CheckpointSweep's (crop, kitti, losses)
    g = obj._graph_for(1, True, losses) if isinstance(obj, S.CheckpointSweep) else obj._graph_for(1, True, False, losses)
    g.graph.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.graph.replay()
    e1.record()
    e1.synchronize()
    obj.disable_cuda_graph()
    return e0.elapsed_time(e1) / reps


def main(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--ks", type=int, nargs="+", default=[4, 10])
    p.add_argument("--frames", type=int, default=512)
    p.add_argument("--batches", type=int, nargs="+", default=[1, 16])
    p.add_argument("--losses", choices=("both", "on", "off"), default="both")
    p.add_argument("--rounds", type=int, default=2)
    p.add_argument("--reps", type=int, default=20)
    p.add_argument("--json", default=None)
    args = p.parse_args(argv)
    import torch
    assert torch.cuda.is_available(), "the timing needs a CUDA device"
    out = dict(card=card(), frames=args.frames, runs=[])
    print("%s; %d frames" % (out["card"], args.frames), flush=True)
    tmp = tempfile.mkdtemp()
    try:
        run_all(args, out, tmp)
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


def run_all(args, out, tmp):
    import sassd_b200 as S
    from sassd_b200 import checkpoint
    from sassd_b200.kitti_data import KittiSplit
    from tests.checkpoint_weights import checkpoint_state_dict
    root = os.path.join(tmp, "kitti")
    write_root(root, args.frames)
    ckpts = []
    for seed in range(1, max(args.ks) + 1):
        ckpts.append(os.path.join(tmp, "epoch_%d.pth" % (2 * seed)))
        checkpoint.save_checkpoint(checkpoint_state_dict(seed), ckpts[-1])
    clock = EvalClock()
    split = KittiSplit(root, "val", "velodyne", gt_classes=["Car"])
    loss_modes = dict(both=(False, True), on=(True,), off=(False,))[args.losses]
    for K in args.ks:
        for B in args.batches:
            frames = [split.frame(i) for i in split.ids[:B]]
            pts, metas, gts = [f[0] for f in frames], [f[1] for f in frames], [f[2] for f in frames]
            planes = [split.planes(m["calib"], m["img_shape"]) for m in metas]
            for losses in loss_modes:
                base = ["--data-root", root, "--batch", str(B), "--workers", "4"] + (["--losses"] if losses else [])
                rounds = []
                for r in range(2 * args.rounds):                  # sweep, singles, sweep, singles, ...
                    if r % 2 == 0:
                        x = driver_run([CFG, ckpts[0], "--checkpoints"] + ckpts[1:K] + base, clock)
                        models = []
                        for c in ckpts[:K]:
                            m, _, _ = S.build_from_config(S.Config.fromfile(CFG), device="cuda:0")
                            checkpoint.load_params_from_file(m, c)
                            models.append(m)
                        x.update(what="sweep", step_ms=step_ms(S.CheckpointSweep(models), pts, planes, metas, gts,
                                                               losses, args.reps))
                    else:
                        each = [driver_run([CFG, c] + base, clock) for c in ckpts[:K]]
                        x = {k: sum(e[k] for e in each) for k in ("wall_s", "read_wait_s", "eval_s")}
                        x.update(what="singles", max_memory_gb=max(e["max_memory_gb"] for e in each))
                        m, _, _ = S.build_from_config(S.Config.fromfile(CFG), device="cuda:0")
                        steps = []
                        for c in ckpts[:K]:
                            checkpoint.load_params_from_file(m, c)
                            steps.append(step_ms(m, pts, planes, metas, gts, losses, args.reps))
                        x["step_ms"] = sum(steps)
                    models = m = None
                    release()
                    x.update(K=K, batch=B, losses=losses)
                    rounds.append(x)
                    print("K %2d batch %2d losses %-5s %-7s wall %7.2f s  read wait %7.2f s  eval %6.2f s  "
                          "step %8.3f ms  max memory %6.2f GB" % (K, B, losses, x["what"], x["wall_s"],
                                                                   x["read_wait_s"], x["eval_s"], x["step_ms"],
                                                                   x["max_memory_gb"]), flush=True)
                out["runs"] += rounds


if __name__ == "__main__":
    main()
