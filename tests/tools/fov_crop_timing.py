"""Timing of the image-FOV crop of raw-drive sweeps (needs an H100).

    python tests/tools/fov_crop_timing.py [--iters 400] [--frames 512] [--json FILE]

  * crop kernel time per frame (ops.image_fov_crop, and ops.frustum_crop on the same sweeps) from CUDA events over
    --iters launches replayed from a captured graph, at batch 1 and 16, on synthetic 360-degree sweeps
    (synth_cloud(seed, fov_deg=180), ~123 k points each), with the bytes each must move (16 B per input point + 16 B
    per kept point) over that time;
  * driver frames/s (python -m sassd_b200.test) on a --frames synthetic raw drive (``--drive``, image-FOV crop on the
    device) at batch 1 and 16, next to the frustum-crop driver on the same clouds (a ``testing/`` tree read with
    ``--split test``), alternating the two.
Prints the card name and power limit read in the same run, then one JSON line per measurement."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from sassd_b200 import ops  # noqa: E402
from sassd_b200.frustum import camera_frustum_planes  # noqa: E402
from sassd_b200.results import meta_block  # noqa: E402
from sassd_b200.synth import synth_cloud  # noqa: E402

PER_GRAPH = 20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else "unavailable")


def time_kernel(kind, sweeps, calib, shape, B, iters):
    dev = torch.device("cuda:0")
    frames = [sweeps[b % len(sweeps)] for b in range(B)]
    counts = [f.shape[0] for f in frames]
    pts = torch.from_numpy(np.concatenate(frames, 0)).to(dev)
    off = torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)).to(dev)
    if kind == "image_fov":
        arg = torch.from_numpy(np.stack([meta_block(calib, shape)] * B)).to(dev)
        fn = ops.image_fov_crop
    else:
        arg = torch.from_numpy(np.stack([camera_frustum_planes(calib, shape)] * B)).to(dev)
        fn = ops.frustum_crop
    ws = ops.Workspace()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            out, off_out = fn(pts, off, B, arg, ws=ws)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):                 # descriptor memset + kernel, PER_GRAPH times
        for _ in range(PER_GRAPH):
            out, off_out = fn(pts, off, B, arg, ws=ws)
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = max(1, iters // PER_GRAPH)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / (reps * PER_GRAPH)
    kept = int(off_out[-1])
    nbytes = 16 * (sum(counts) + kept)
    return dict(what="crop_kernel", crop=kind, batch=B, points_in=sum(counts), points_kept=kept,
                ms_per_launch=round(ms, 5), us_per_frame=round(1e3 * ms / B, 3),
                achieved_GBps=round(nbytes / (ms * 1e-3) / 1e9, 1))


def _link_or_copy(src, dst):
    try:
        os.link(src, dst)
    except OSError:
        shutil.copyfile(src, dst)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=400)
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "fov_crop_timing.py needs a CUDA device"
    from sassd_b200 import checkpoint
    from sassd_b200 import test as T
    from tests.test_image_fov import _calib, write_drive, write_testing
    from tests.test_kitti_format import _calib_txt
    results = [dict(what="card", **card())]
    print(json.dumps(results[-1]))
    z = np.load(os.path.join(ROOT, "tests", "golden", "fov.npz"))
    calib, shape = _calib(z, 0), (375, 1242, 3)
    sweeps = [synth_cloud(s, fov_deg=180.0) for s in range(4)]
    for B in (1, 16):
        for kind in ("image_fov", "frustum"):
            results.append(time_kernel(kind, sweeps, calib, shape, B, args.iters))
            print(json.dumps(results[-1]))

    clouds = [synth_cloud(4000 + k, fov_deg=180.0) for k in range(32)]
    cfg = os.path.join(ROOT, "configs", "car_cfg.py")
    with tempfile.TemporaryDirectory() as tmp:
        stems = list(range(args.frames))
        drive = write_drive(os.path.join(tmp, "2011_09_26"), stems, [shape[:2]], clouds, z, ci=0)
        root = os.path.join(tmp, "kitti")
        write_testing(root, [], [shape[:2]], [_calib_txt(calib)], clouds)
        with open(os.path.join(root, "ImageSets", "test.txt"), "w") as fh:
            fh.write("".join("%06d\n" % i for i in stems))
        for i in stems:             # the same clouds, image sizes and calibration as the drive
            _link_or_copy(os.path.join(drive, "velodyne_points", "data", "%010d.bin" % i),
                          os.path.join(root, "testing", "velodyne", "%06d.bin" % i))
            _link_or_copy(os.path.join(drive, "image_02", "data", "%010d.png" % i),
                          os.path.join(root, "testing", "image_2", "%06d.png" % i))
            with open(os.path.join(root, "testing", "calib", "%06d.txt" % i), "w") as fh:
                fh.write(_calib_txt(calib))
        ckpt = os.path.join(tmp, "w.pth")
        checkpoint.save_checkpoint(checkpoint.make_synthetic_state_dict(0, 1), ckpt)
        import gc
        for B in (1, 16):
            for rep in range(2):            # alternate the two arms
                for arm, src in (("image_fov", ["--drive", drive]), ("frustum", ["--data-root", root, "--split", "test"])):
                    gc.collect()
                    torch.cuda.empty_cache()            # each run builds its own model and captured slots
                    out = os.path.join(tmp, "out_%s_%d_%d" % (arm, B, rep))
                    res = T.run(T.parse_args([cfg, ckpt] + src + ["--batch", str(B), "--out", out]),
                                log=lambda *a, **k: None)
                    results.append(dict(what="driver", crop=arm, batch=B, frames=res["frames"],
                                        frames_per_s=round(res["frames_per_s"], 1),
                                        read_wait_ms_per_frame=round(1e3 * res["read_wait_s"] / res["frames"], 4)))
                    print(json.dumps(results[-1]))
    results.append(dict(what="card_after", **card()))
    print(json.dumps(results[-1]))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(results, fh, indent=1)


if __name__ == "__main__":
    main()
