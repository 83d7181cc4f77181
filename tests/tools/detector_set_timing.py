"""Timing of a DetectorSet of three single-class models against its members run one after another.

    python tests/tools/detector_set_timing.py [--reps 50] [--json FILE]

Members: the Car model of configs/car_cfg.py (seed 0's synthetic weights) and single-class Pedestrian and Cyclist models
built from the same config with configs/multi_cfg.py's anchor sizes, each with weights of its own
(member_state_dict), as tests/test_detector_set.py builds them.  Frames: synthetic full sweeps (synth_cloud, 180 degrees, ~120 k points), cropped on the device to the
camera frustums of tests/golden/frustum.npz's two calibrations.  At batch 1 and 16, with every step captured
(enable_cuda_graph, the frustum-crop kind), it reports:
  * step: the GPU time of one captured step (CUDA events around ``reps`` back-to-back replays, divided by ``reps``),
    for the set and for each member; the members' sum is what three separate runs spend;
  * call: the wall clock of one forward_points call (staging, H2D, replay, D2H, unpacking; the host clock around work
    that ends in a stream synchronise), median of ``reps`` calls, for the set and for each member.
The set and the members are measured alternately, twice each, and every round is printed.  The card's name and power
limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)


def power_limit():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def step_ms(graph, reps):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    graph.replay()
    e0.record()
    for _ in range(reps):
        graph.replay()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def call_ms(obj, frames, planes, reps):
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        obj.forward_points(frames, frustum_planes=planes)
        t.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(t))


def main(argv=None):
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=50)
    p.add_argument("--json", default=None)
    args = p.parse_args(argv)
    import torch
    from sassd_b200 import checkpoint
    from sassd_b200.detectors import CROP_FRUSTUM, DetectorSet
    from sassd_b200.frustum import camera_frustum_planes
    from sassd_b200.results import Calibration
    from sassd_b200.synth import synth_cloud
    from tests.test_detector_set import MEMBERS, SHAPES, build_member, member_state_dict
    assert torch.cuda.is_available(), "the timing needs a CUDA device"
    card = torch.cuda.get_device_name(0)
    limit = power_limit()
    tmp = tempfile.mkdtemp()
    members = []
    for name, seed, sizes in MEMBERS:
        m = build_member(tmp, name, sizes, "cuda:0")
        checkpoint.load_state_dict_into(m, member_state_dict(seed))
        members.append(m)
    dset = DetectorSet(members)
    z = np.load(os.path.join(ROOT, "tests", "golden", "frustum.npz"))
    calibs = [Calibration({"P2": z["calib%d_P2" % c], "Tr_velo_to_cam": z["calib%d_Tr" % c],
                           "R0_rect": z["calib%d_R0" % c]}) for c in range(2)]
    clouds = [synth_cloud(500 + i, fov_deg=180.0) for i in range(16)]
    all_planes = [camera_frustum_planes(calibs[i % 2], SHAPES[i % 2]) for i in range(16)]
    maxpts = 131072
    out = dict(card=card, power_limit=limit, reps=args.reps, members=[n for n, _, _ in MEMBERS], batches={})
    print("%s, power limit %s; %d reps per measurement" % (card, limit, args.reps))
    for B in (1, 16):
        frames, planes = clouds[:B], all_planes[:B]
        objs = members + [dset]
        graphs = []
        for o in objs:
            o.enable_cuda_graph(B, maxpts)
            o.forward_points(frames, frustum_planes=planes)       # captures the crop kind and loads its inputs
            graphs.append(o._graph_for(CROP_FRUSTUM, False) if o is dset else o._graph_for(CROP_FRUSTUM, False, False))
        torch.cuda.synchronize()
        rounds = []
        for r in range(4):                                          # set, members, set, members
            if r % 2 == 0:
                rounds.append(dict(what="set", step_ms=step_ms(graphs[-1], args.reps),
                                   call_ms=call_ms(dset, frames, planes, args.reps)))
            else:
                steps = [step_ms(g, args.reps) for g in graphs[:-1]]
                calls = [call_ms(m, frames, planes, args.reps) for m in members]
                rounds.append(dict(what="members", step_ms=sum(steps), call_ms=sum(calls), step_each=steps,
                                   call_each=calls))
            x = rounds[-1]
            print("batch %2d  %-7s  step %8.3f ms  call %8.3f ms%s" % (
                B, x["what"], x["step_ms"], x["call_ms"],
                "  (each step %s)" % ", ".join("%.3f" % s for s in x["step_each"]) if "step_each" in x else ""))
        for o in objs:
            o.disable_cuda_graph()
        out["batches"][B] = rounds
    if args.json:
        with open(args.json, "w") as fh:
            json.dump(out, fh, indent=1)


if __name__ == "__main__":
    main()
