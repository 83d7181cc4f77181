"""Wall time of the KITTI evaluation on a val-split-sized synthetic set (3769 frames, classes 0, 1, 2), device
evaluator against the host path, for K = 1 and K = 10 detection sets, official tables (R11) alone and official + COCO.

    python tests/tools/coco_eval_timing.py [--out FILE.json]

The host path is given the device's rotated overlaps: one batched launch per criterion computes them for every
(set, frame), and its ``overlap_fn`` looks each frame's matrix up, so the two paths differ in cleaning and matching only
(the host still computes the 2-D and height overlaps in numpy).  The two paths alternate, twice, and their texts must
agree.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
from make_golden_eval import synth_annos  # noqa: E402
from sassd_b200 import kitti_eval as K  # noqa: E402


def detection_sets(dts, n, seed=3):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        s = []
        for d in dts:
            keep = rng.uniform(size=len(d["name"])) < 0.85
            e = {k: np.asarray(v)[keep] for k, v in d.items()}
            e["score"] = np.clip(e["score"] + rng.normal(0, 0.05, len(e["score"])), 0.0, 1.0)
            s.append(e)
        out.append(s)
    return out


def lookup_overlap_fn(gts, sets):
    """An overlap_fn answering from one batched device launch per criterion over every (set, frame)."""
    import torch
    bev = [0, 2, 3, 5, 6]

    def cam(a):
        return np.concatenate([np.asarray(a["location"], np.float64).reshape(-1, 3),
                               np.asarray(a["dimensions"], np.float64).reshape(-1, 3),
                               np.asarray(a["rotation_y"], np.float64).reshape(-1, 1)], 1)[:, bev].astype(np.float32)
    dts = [cam(d) for s in sets for d in s]
    gs = [cam(g) for g in gts] * len(sets)
    table = {}
    for criterion in (-1, 2):
        for b, q, o in zip(dts, gs, K._rotated_overlaps(dts, gs, criterion)):
            table[criterion, b.tobytes(), q.tobytes()] = o
    torch.cuda.synchronize()
    return lambda b, q, criterion: table[criterion, np.asarray(b, np.float32).tobytes(),
                                         np.asarray(q, np.float32).tobytes()]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--frames", type=int, default=3769)
    args = ap.parse_args()
    import torch
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    card = dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=smi[0] if smi else None)
    print("card:", card)
    gts, dts = synth_annos(np.random.default_rng(5), nframes=args.frames)
    all_sets = detection_sets(dts, 10)
    K.eval_many(gts[:50], [s[:50] for s in all_sets[:2]], [0, 1, 2], (11, "coco"))      # warm-up (context, library)
    rows = []
    for nsets in (1, 10):
        sets = all_sets[:nsets]
        fn = lookup_overlap_fn(gts, sets)
        for tables in ((11,), (11, "coco")):
            times = {"device": [], "host": []}
            texts = {}
            for rep in range(2):
                for path in ("device", "host"):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    res = K.eval_many(gts, sets, [0, 1, 2], tables, overlap_fn=None if path == "device" else fn)
                    torch.cuda.synchronize()
                    times[path].append(time.perf_counter() - t0)
                    texts[path] = [[r[t][0] for t in tables] for r in res]
            assert texts["device"] == texts["host"], "device and host texts differ"
            row = dict(frames=len(gts), sets=nsets, tables=[str(t) for t in tables], device_s=times["device"],
                       host_s=times["host"])
            rows.append(row)
            print("K=%2d %-14s device %s s   host %s s" % (nsets, "+".join(row["tables"]),
                                                         " ".join("%.3f" % t for t in times["device"]),
                                                         " ".join("%.3f" % t for t in times["host"])))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(dict(card=card, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
