"""Timing of KITTI root preparation (python -m sassd_b200.create_data; needs an H100).

    python tests/tools/create_data_timing.py [--frames 512] [--iters 400] [--json FILE]

  * driver frames/s on a synthetic root of --frames training frames (full sweeps synth_cloud(seed, fov_deg=180),
    ~123 k points, 15 labelled objects and a DontCare row each; tests/kitti_root.py's rows), with the seconds spent
    waiting on reads and on writes, at batch 16 and 1, each run twice (the second on a warm page cache);
  * kernel time per batch of ops.frustum_crop and ops.points_in_rbboxes on 16 of those frames, from CUDA events over
    --iters launches replayed from a captured graph.
Prints the card name and power limit read in the same run, then one JSON line per measurement."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from sassd_b200 import create_data as CD  # noqa: E402
from sassd_b200 import ops  # noqa: E402
from sassd_b200.synth import synth_cloud  # noqa: E402
from tests import kitti_root as KR  # noqa: E402

PER_GRAPH = 20
N_CLOUDS = 8


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else "unavailable")


def write_root(root, n):
    """n training frames (ids 0..n-1 in train), empty val and test lists."""
    os.makedirs(os.path.join(root, "ImageSets"))
    for name, ids in (("train", range(n)), ("val", []), ("test", [])):
        with open(os.path.join(root, "ImageSets", name + ".txt"), "w") as fh:
            fh.write("".join("%06d\n" % i for i in ids))
    sub = os.path.join(root, "training")
    for d in ("velodyne", "calib", "image_2", "label_2"):
        os.makedirs(os.path.join(sub, d))
    clouds = [os.path.join(root, "cloud%d.bin" % k) for k in range(N_CLOUDS)]
    for k, path in enumerate(clouds):
        synth_cloud(1000 + k, fov_deg=180.0).tofile(path)
    pngs = [KR.png_bytes(h, w) for h, w in KR.SHAPES]
    for idx in range(n):
        shutil.copyfile(clouds[idx % N_CLOUDS], os.path.join(sub, "velodyne", "%06d.bin" % idx))
        rig = idx % 2
        with open(os.path.join(sub, "calib", "%06d.txt" % idx), "w") as fh:
            fh.write(KR.calib_text(rig))
        with open(os.path.join(sub, "image_2", "%06d.png" % idx), "wb") as fh:
            fh.write(pngs[(idx // 2) % 2])
        rows = KR.label_lines(5, KR._rig(rig), np.random.default_rng(idx))
        with open(os.path.join(sub, "label_2", "%06d.txt" % idx), "w") as fh:
            fh.write("".join(r + "\n" for r in rows))


def clean_outputs(root):
    for d in ("training/velodyne_reduced", "gt_database"):
        shutil.rmtree(os.path.join(root, d), ignore_errors=True)


def time_kernels(root, B, iters):
    """ms per launch of the frustum crop and of points_in_rbboxes on B frames of the root."""
    from sassd_b200.kitti_data import PlaneCache
    from sassd_b200.results import Calibration
    dev = torch.device("cuda:0")
    planes = PlaneCache()
    pts, fpl, bpl, cen, nbox = [], [], [], [], []
    for idx in range(B):
        info, p = CD.frame_info(root, idx, True)
        boxes = CD.lidar_boxes(info["annos"], info["calib/R0_rect"], info["calib/Tr_velo_to_cam"])
        calib = Calibration({"P2": info["calib/P2"][:3], "Tr_velo_to_cam": info["calib/Tr_velo_to_cam"][:3],
                             "R0_rect": info["calib/R0_rect"][:3, :3]})
        pts.append(p); fpl.append(planes(calib, info["img_shape"]))
        bpl.append(CD.box_planes(boxes)); cen.append(boxes[:, :3]); nbox.append(len(boxes))
    box_cap = max(nbox)
    P, C = np.zeros((B, box_cap, 6, 4)), np.zeros((B, box_cap, 3))
    for b in range(B):
        P[b, :nbox[b]], C[b, :nbox[b]] = bpl[b], cen[b]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)    # noqa: E731
    d_pts = t(np.concatenate(pts, 0))
    d_off = t(np.concatenate([[0], np.cumsum([len(p) for p in pts])]).astype(np.int32))
    d_fpl, d_P, d_C, d_n = t(np.stack(fpl)), t(P), t(C), t(np.array(nbox, np.int32))
    ws = ops.Workspace()
    status = torch.zeros((1,), dtype=torch.int32, device=dev)
    crop, crop_off = ops.frustum_crop(d_pts, d_off, B, d_fpl, ws=ws)
    gcap = d_pts.shape[0]
    out = {}
    for name, fn in (("frustum_crop", lambda: ops.frustum_crop(d_pts, d_off, B, d_fpl, ws=ws)),
                     ("points_in_rbboxes", lambda: ops.points_in_rbboxes(crop, crop_off, B, d_P, d_C, d_n, gcap,
                                                                          status=status, ws=ws))):
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                fn()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(PER_GRAPH):
                res = fn()
        g.replay()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        reps = max(1, iters // PER_GRAPH)
        e0.record()
        for _ in range(reps):
            g.replay()
        e1.record()
        torch.cuda.synchronize()
        out[name] = e0.elapsed_time(e1) / (reps * PER_GRAPH)
        if name == "points_in_rbboxes":
            assert int(status.item()) == 0
            out["gathered_rows"] = int(res[1][-1])
    return dict(what="kernels", batch=B, points_in=int(d_off[-1]), points_cropped=int(crop_off[-1]),
                boxes=int(sum(nbox)), gathered_rows=out["gathered_rows"],
                frustum_crop_ms_per_batch=round(out["frustum_crop"], 4),
                points_in_rbboxes_ms_per_batch=round(out["points_in_rbboxes"], 4))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--iters", type=int, default=400)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    results = [dict(what="card", **card())]
    print(json.dumps(results[-1]))
    work = tempfile.mkdtemp(prefix="create_data_timing_")
    try:
        root = os.path.join(work, "kitti")
        t0 = time.perf_counter()
        write_root(root, args.frames)
        print("wrote %d frames in %.1f s" % (args.frames, time.perf_counter() - t0))
        results.append(time_kernels(root, 16, args.iters))
        print(json.dumps(results[-1]))
        for batch in (16, 1, 16, 1):
            clean_outputs(root)
            r = CD.create_data(root, batch=batch, log=lambda *a: None)
            results.append(dict(what="driver", batch=batch, frames=r["frames"],
                                frames_per_s=round(r["frames"] / r["seconds"], 1), seconds=round(r["seconds"], 3),
                                read_wait_s=round(r["read_wait"], 3), write_wait_s=round(r["write_wait"], 3)))
            print(json.dumps(results[-1]))
    finally:
        shutil.rmtree(work, ignore_errors=True)
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
