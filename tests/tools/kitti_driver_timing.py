"""Timing of KITTI split evaluation (python -m sassd_b200.test) on a synthetic tree of full sweeps.

    python tests/tools/kitti_driver_timing.py [--frames 512] [--batch 16] [--json FILE]

Writes a KITTI-layout tree to a temporary directory: ``--frames`` full synthetic 360-degree sweeps (32 distinct clouds,
repeated), the same frames cropped to the camera frustum on the host as ``velodyne_reduced``, the two calibrations of
tests/golden/frustum.npz alternating, PNG headers of two sizes and empty label files.  Reports, with the card's name
and power limit read in the same run:
  * driver frames/s with ``--lidar velodyne`` (cropped on the device) and ``--lidar velodyne_reduced``;
  * per frame: the driver's wall clock, its time waiting on reads, and the GPU time of one captured crop + format step
    run alone (CUDA events around one slot's replay).  Host time is not separated from these: in the stream it
    overlaps the GPU work of the steps in flight;
  * the device formatter for a batch: its kernel time (a CUDA graph of KERNEL_REPS back-to-back launches, timed
    between one pair of events and divided by KERNEL_REPS) and the time of one ``ops.kitti_format`` call from Python
    (allocation, ctypes call and launch included), against host ``kitti_bbox2results`` per frame.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    import torch
    from oracle.frustum import inside_frustum
    from sassd_b200 import checkpoint, ops
    from sassd_b200 import test as T
    from sassd_b200.frustum import camera_frustum_planes
    from sassd_b200.results import Calibration, kitti_bbox2results, meta_block
    from sassd_b200.synth import synth_cloud
    from tests.test_kitti_data import write_split
    from tests.test_kitti_format import _calib_txt

    z = np.load(os.path.join(ROOT, "tests", "golden", "frustum.npz"))
    calibs = [Calibration({"P2": z["calib%d_P2" % c], "Tr_velo_to_cam": z["calib%d_Tr" % c],
                           "R0_rect": z["calib%d_R0" % c]}) for c in range(2)]
    shapes = [(375, 1242), (370, 1224)]
    clouds = [synth_cloud(2000 + k, fov_deg=180.0) for k in range(32)]
    out = dict(gpu=torch.cuda.get_device_name(0), power_limit=power_limit(), frames=args.frames, batch=args.batch)
    with tempfile.TemporaryDirectory() as tmp:
        root = os.path.join(tmp, "kitti")
        ids = list(range(args.frames))
        pts = [clouds[i % 32] for i in ids]
        write_split(root, ids, shapes, [_calib_txt(c) for c in calibs], pts)
        for i in ids:       # velodyne_reduced: the frames cropped to their frustum on the host
            p = camera_frustum_planes(calibs[i % 2], shapes[i % 2])
            c = pts[i][inside_frustum(pts[i], p)]
            c.tofile(os.path.join(root, "training", "velodyne_reduced", "%06d.bin" % i))
            open(os.path.join(root, "training", "label_2", "%06d.txt" % i), "w").close()
        ckpt = os.path.join(tmp, "w.pth")
        checkpoint.save_checkpoint(checkpoint.make_synthetic_state_dict(0, 1), ckpt)
        cfg = os.path.join(ROOT, "configs", "car_cfg.py")
        import gc
        for lidar in ("velodyne", "velodyne_reduced"):
            gc.collect()
            torch.cuda.empty_cache()            # each run builds its own model and captured slots
            res = T.run(T.parse_args([cfg, ckpt, "--data-root", root, "--batch", str(args.batch), "--lidar", lidar]),
                        log=lambda *a, **k: None)
            key = "driver_" + lidar
            out.setdefault(key, []).append(dict(frames_per_s=round(res["frames_per_s"], 1),
                                                read_wait_ms_per_frame=round(1e3 * res["read_wait_s"] / args.frames, 4),
                                                wall_ms_per_frame=round(1e3 * res["wall_s"] / args.frames, 4)))

        # GPU time of one captured formatting step (crop slot), per frame
        gc.collect()
        torch.cuda.empty_cache()
        import sassd_b200 as S
        model, _, _ = S.build_from_config(S.Config.fromfile(cfg), device="cuda:0")
        checkpoint.load_state_dict_into(model, checkpoint.make_synthetic_state_dict(0, 1))
        B = args.batch
        batch = [(pts[i], camera_frustum_planes(calibs[i % 2], shapes[i % 2]),
                  dict(calib=calibs[i % 2], img_shape=shapes[i % 2] + (3,), sample_idx=i)) for i in range(B)]
        item = ([b[0] for b in batch], [b[1] for b in batch], [b[2] for b in batch])
        list(model.detect_stream([item] * 2, B, 131072, depth=1, crop=True, kitti=True))
        slot = model._stream_slots[0]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for _ in range(20):
            e0.record()
            slot.graph.replay()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        out["gpu_step_ms_per_frame"] = round(float(np.median(times)) / B, 4)

        # the formatter alone: device kernel for a batch vs host per frame, on this step's detections
        dets = model.forward_points(item[0], frustum_planes=item[1])
        rng = np.random.default_rng(0)
        det = np.zeros((B, 512, 9), np.float32)
        nd = np.zeros(B, np.int32)
        for b in range(B):
            n = int(rng.integers(5, 51))
            src = dets[b]["boxes_lidar"]
            boxes = np.tile(src, (n // max(len(src), 1) + 1, 1))[:n] if src is not None else \
                np.tile([[20, 0, -1, 1.6, 3.9, 1.56, 0.3]], (n, 1))
            det[b, :n, :7] = boxes
            det[b, :n, 7] = 0.5
            nd[b] = n
        dev = torch.device("cuda:0")
        d_det, d_nd = torch.from_numpy(det).to(dev), torch.from_numpy(nd).to(dev)
        d_meta = torch.from_numpy(np.stack([meta_block(m["calib"], m["img_shape"]) for m in item[2]])).to(dev)
        ops.kitti_format(d_det, d_nd, d_meta)
        times = []
        for _ in range(50):
            e0.record()
            ops.kitti_format(d_det, d_nd, d_meta)
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1))
        out["device_format_call_us_per_batch"] = round(1e3 * float(np.median(times)), 2)
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            ops.kitti_format(d_det, d_nd, d_meta)
        torch.cuda.current_stream().wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(KERNEL_REPS):
                ops.kitti_format(d_det, d_nd, d_meta)
        g.replay()
        torch.cuda.synchronize()
        times = []
        for _ in range(10):
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / KERNEL_REPS)
        out["device_format_kernel_us_per_batch"] = round(1e3 * float(np.median(times)), 2)
        t = []
        for _ in range(5):
            t0 = time.perf_counter()
            for b in range(B):
                n = int(nd[b])
                kitti_bbox2results(det[b, :n, :7].copy(), det[b, :n, 7], det[b, :n, 8].astype(np.int64), item[2][b],
                                   ["Car"])
            t.append((time.perf_counter() - t0) / B)
        out["host_format_us_per_frame"] = round(1e6 * float(np.median(t)), 1)
    print(json.dumps(out, indent=1))
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
