"""Wall time of the KITTI evaluation with and without range bins on a val-split-sized synthetic set (3769 frames,
classes 0, 1, 2, the official R11 table), device evaluator against the host path, for K = 1 and K = 10 detection
sets.  "bins" is eval_many(ranges=(0, 20, 40, inf), match=True): three bins on top of the whole range and the match
table, what the drivers' --ranges runs.

    python tests/tools/kitti_eval_ranges_timing.py [--out FILE.json] [--frames 3769]

The host path is given the device's rotated overlaps (coco_eval_timing.lookup_overlap_fn), so the two paths differ in
cleaning and matching only.  The two paths alternate, twice each, and their texts must agree.  The card's name and
power limit are read in the same run."""
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
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
from coco_eval_timing import detection_sets, lookup_overlap_fn  # noqa: E402
from make_golden_eval import synth_annos  # noqa: E402
from sassd_b200 import kitti_eval as K  # noqa: E402

EDGES = (0.0, 20.0, 40.0, np.inf)


def _texts(res):
    return [[r[11][0]] + [b[2][11][0] for b in r.get("ranges", [])] for r in res]


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
    K.eval_many(gts[:50], [s[:50] for s in all_sets[:2]], [0, 1, 2], (11,), ranges=EDGES, match=True)   # warm-up
    rows = []
    for nsets in (1, 10):
        sets = all_sets[:nsets]
        fn = lookup_overlap_fn(gts, sets)
        for binned in (False, True):
            kw = dict(ranges=EDGES, match=True) if binned else {}
            times = {"device": [], "host": []}
            texts = {}
            for rep in range(2):
                for path in ("device", "host"):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    res = K.eval_many(gts, sets, [0, 1, 2], (11,), None if path == "device" else fn, **kw)
                    torch.cuda.synchronize()
                    times[path].append(time.perf_counter() - t0)
                    texts[path] = _texts(res)
            assert texts["host"] == texts["device"], "host and device texts differ"
            rows.append(dict(frames=len(gts), sets=nsets, bins=len(EDGES) - 1 if binned else 0, device_s=times["device"],
                             host_s=times["host"]))
            print("K=%2d bins=%d device %s host %s" % (nsets, rows[-1]["bins"], ", ".join("%.3f" % t for t in
                                                                                         times["device"]),
                                                     ", ".join("%.2f" % t for t in times["host"])))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(dict(card=card, edges=[e if np.isfinite(e) else None for e in EDGES], rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
