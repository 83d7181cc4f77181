"""Timing of the camera-frustum crop of full sweeps (needs an H100).

    python tests/tools/crop_timing.py [--iters 200] [--steps 40]

  * crop kernel (ops.frustum_crop) time per frame from CUDA events over --iters launches replayed from a captured
    graph (eager calls are bounded by the host, and are reported apart), at batch 1 and 16, on synthetic 360-degree
    sweeps (synth_cloud(seed, fov_deg=180), ~123 k points each), with the bytes it must move (16 B per input point +
    16 B per kept point) over that time;
  * detect_stream frames/s on the same full sweeps with crop=True (the crop runs inside every captured step), against
    the same stream fed the clouds cropped beforehand on the host (what the reference's velodyne_reduced files give).
Prints the card name and power limit first, then one JSON line per measurement."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import sassd_b200 as S  # noqa: E402
from oracle.frustum import inside_frustum  # noqa: E402
from sassd_b200 import checkpoint, ops  # noqa: E402
from sassd_b200.frustum import camera_frustum_planes  # noqa: E402
from sassd_b200.synth import synth_cloud  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else "unavailable")


def kitti_planes():
    z = np.load(os.path.join(ROOT, "tests", "golden", "frustum.npz"))
    calib = S.Calibration({"P2": z["calib0_P2"], "Tr_velo_to_cam": z["calib0_Tr"], "R0_rect": z["calib0_R0"]})
    return camera_frustum_planes(calib, (375, 1242))


def time_crop(sweeps, planes, B, iters):
    dev = torch.device("cuda:0")
    frames = [sweeps[b % len(sweeps)] for b in range(B)]
    counts = [f.shape[0] for f in frames]
    pts = torch.from_numpy(np.concatenate(frames, 0)).to(dev)
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)).to(dev)
    d_planes = torch.from_numpy(np.stack([planes] * B)).to(dev)
    ws = ops.Workspace()
    for _ in range(10):
        out, off_out = ops.frustum_crop(pts, off, B, d_planes, ws=ws)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    # eager calls: bounded by the host (ctypes call + output allocation), as when the crop runs outside a graph
    e0.record()
    for _ in range(iters):
        ops.frustum_crop(pts, off, B, d_planes, ws=ws)
    e1.record()
    torch.cuda.synchronize()
    ms_eager = e0.elapsed_time(e1) / iters
    # device time: PER_GRAPH launches (descriptor memset + kernel each) captured in one graph, replayed back to back
    per_graph = 20
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(per_graph):
            ops.frustum_crop(pts, off, B, d_planes, ws=ws)
    g.replay()
    torch.cuda.synchronize()
    reps = max(1, iters // per_graph)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / (reps * per_graph)
    kept = int(off_out[-1])
    nbytes = 16 * (sum(counts) + kept)
    return dict(what="crop_kernel", batch=B, points_in=sum(counts), points_kept=kept, ms_per_launch=round(ms, 5),
                us_per_frame=round(1e3 * ms / B, 3), achieved_GBps=round(nbytes / (ms * 1e-3) / 1e9, 1),
                ms_per_eager_call=round(ms_eager, 5))


def time_stream(model, batches, B, maxpts, depth, steps, crop):
    pool = len(batches)
    for _ in model.detect_stream([batches[i % pool] for i in range(2 * depth)], B, maxpts, depth=depth, crop=crop):
        pass
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n = 0
    for _ in model.detect_stream((batches[i % pool] for i in range(steps)), B, maxpts, depth=depth, crop=crop):
        n += 1
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return dict(what="detect_stream", crop_on_gpu=crop, batch=B, max_points_per_frame=maxpts, depth=depth, steps=n,
                frames_per_s=round(n * B / dt, 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--depth", type=int, default=4)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "crop_timing.py needs a CUDA device"
    print(json.dumps(dict(what="card", **card())))
    planes = kitti_planes()
    sweeps = [synth_cloud(s, fov_deg=180.0) for s in range(4)]
    reduced = [s[inside_frustum(s, planes)] for s in sweeps]
    for B in (1, 16):
        print(json.dumps(time_crop(sweeps, planes, B, args.iters)))
    cfg = S.Config.fromfile(os.path.join(ROOT, "configs", "car_cfg.py"))
    model, _, _ = S.build_from_config(cfg, device="cuda:0")
    checkpoint.load_state_dict_into(model, checkpoint.make_synthetic_state_dict(0, 1))
    red_cap = ops.next_pow2(max(r.shape[0] for r in reduced))
    for B in (1, 16):
        idx = [[(i * B + b) % len(sweeps) for b in range(B)] for i in range(4)]
        full = [([sweeps[j] for j in ix], np.stack([planes] * B)) for ix in idx]
        pre = [[reduced[j] for j in ix] for ix in idx]
        for _ in range(2):                 # alternate the two arms
            print(json.dumps(time_stream(model, full, B, 131072, args.depth, args.steps, True)))
            print(json.dumps(time_stream(model, pre, B, red_cap, args.depth, args.steps, False)))
    print(json.dumps(dict(what="card_after", **card())))


if __name__ == "__main__":
    main()
