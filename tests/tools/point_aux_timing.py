"""Timing of the auxiliary point-wise network (csrc/point_aux.cu) on synthetic ~20 k-point clouds.

    python tests/tools/point_aux_timing.py [--batches 1 16] [--steps 50] [--json FILE]

Reports, with the card's name and power limit read in the same run, per batch size:
  * the kernel time of sassd_three_nn and sassd_point_aux_head on the step's own voxel rows and levels: a CUDA graph of
    KERNEL_REPS back-to-back launches, timed between one pair of events and divided by KERNEL_REPS;
  * the captured forward_points step (enable_cuda_graph; host staging, H2D, replay, D2H and unpacking) with and
    without ``point_outputs``, alternating, median of ``--steps`` calls each.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

KERNEL_REPS = 100

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def graph_ms(fn):
    """Kernel time of fn's launches: KERNEL_REPS of them captured in one graph, timed with events."""
    import torch
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(KERNEL_REPS):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / KERNEL_REPS


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[1, 16])
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    import sassd_b200 as S
    from sassd_b200 import checkpoint, ops
    from sassd_b200.synth import synth_cloud
    if not torch.cuda.is_available():
        raise SystemExit("point_aux_timing needs a CUDA device")
    dev = torch.device("cuda:0")
    card = torch.cuda.get_device_name(0)
    plim = power_limit()
    cfg = S.Config.fromfile(os.path.join(ROOT, "configs", "car_cfg.py"))
    model, _, _ = S.build_from_config(cfg, device="cuda:0")
    sd = checkpoint.make_synthetic_state_dict(0, 1)
    g = __import__("torch").Generator().manual_seed(7)
    sd.update({"neck.point_fc.weight": torch.randn(64, 160, generator=g) / 160 ** 0.5,
               "neck.point_cls.weight": torch.randn(1, 64, generator=g) / 8,
               "neck.point_reg.weight": torch.randn(3, 64, generator=g) / 8})
    checkpoint.load_state_dict_into(model, sd)
    clouds = [synth_cloud(s) for s in range(16)]
    out = dict(card=card, power_limit=plim, kernel_reps=KERNEL_REPS, batches={})
    for B in args.batches:
        pts = [clouds[b % len(clouds)] for b in range(B)]
        hp, ho, counts = model.stage_points(pts)
        det, nd, status, aux = model.forward_device(hp.to(dev), ho.to(dev), B, max(counts), point_outputs=True)
        torch.cuda.synchronize()
        n0 = int(aux["frame_rows"][-1].item())
        levels = [(m._indices, m.d_rows) for m in aux["middle"]]
        rows0 = aux["frame_rows"][B:B + 1]
        nn_ms = graph_ms(lambda: ops.three_nn(aux["mean"], aux["coors"], rows0, levels, points_mean=True))
        feats = [ops.point_level(feat=m._features, channels=c) if m._features is not None
                 else ops.point_level(split=m._split, channels=c) for m, c in zip(aux["middle"], (32, 64, 64))]
        fc_t, w_out = model.neck._point_weights()
        head_ms = graph_ms(lambda: ops.point_aux_head(aux["idx"], aux["dist2"], rows0, feats, fc_t, w_out))
        lvl_rows = [int(m.d_rows.item()) for m in aux["middle"]]
        model.enable_cuda_graph(B, 32768)
        for flag in (False, True):          # capture + warm both graphs
            model.forward_points(pts, point_outputs=flag)
        t = {False: [], True: []}
        for _ in range(args.steps):
            for flag in (False, True):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                model.forward_points(pts, point_outputs=flag)
                t[flag].append((time.perf_counter() - t0) * 1e3)
        model.disable_cuda_graph()
        r = dict(points=n0, level_rows=lvl_rows, three_nn_ms=nn_ms, point_aux_head_ms=head_ms,
                 step_ms=float(np.median(t[False])), step_point_outputs_ms=float(np.median(t[True])))
        out["batches"][B] = r
        print("%s, power limit %s | B=%d: %d voxel rows, level rows %s | three_nn %.3f ms, point_aux_head %.3f ms | "
              "captured forward_points %.2f ms, with point_outputs %.2f ms (median of %d, alternating)"
              % (card, plim, B, n0, lvl_rows, nn_ms, head_ms, r["step_ms"], r["step_point_outputs_ms"], args.steps))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
