"""Wall time and peak device memory of the KITTI evaluation with R = 1000 bootstrap replicates on a val-split-sized
synthetic set (3769 frames, classes Car, Pedestrian, Cyclist), for K = 1 and K = 10 detection sets, the R11 table alone
and with COCO.  For comparison, a loop of plain eval_many over the first 50 replicates' resampled lists, reported per
replicate.

    python tests/tools/kitti_eval_bootstrap_timing.py [--out FILE.json] [--frames 3769] [--replicates 1000]

The bootstrap and the loop alternate, twice each; the loop's AP must equal the bootstrap's replicates bit for bit.  The
card's name and power limit are read in the same run."""
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
from coco_eval_timing import detection_sets  # noqa: E402
from make_golden_eval import synth_annos  # noqa: E402
from sassd_b200 import kitti_eval as K  # noqa: E402

CLASSES = ["Car", "Pedestrian", "Cyclist"]
LOOP = 50


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--frames", type=int, default=3769)
    ap.add_argument("--replicates", type=int, default=1000)
    args = ap.parse_args()
    import torch
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    card = dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=smi[0] if smi else None)
    print("card:", card)
    gts, dts = synth_annos(np.random.default_rng(5), nframes=args.frames)
    all_sets = detection_sets(dts, 10)
    idx = K.bootstrap_indices(len(gts), args.replicates, seed=0)
    K.eval_many(gts[:50], [s[:50] for s in all_sets[:2]], CLASSES, (11,), bootstrap=idx[:4, :50] % 50)   # warm-up
    rows = []
    for nsets in (1, 10):
        sets = all_sets[:nsets]
        for tables in ((11,), (11, "coco")):
            boot_s, loop_s, peak = [], [], []
            for rep in range(2):
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                res = K.eval_many(gts, sets, CLASSES, tables, bootstrap=idx)
                torch.cuda.synchronize()
                boot_s.append(time.perf_counter() - t0)
                peak.append(torch.cuda.max_memory_allocated())
                t0 = time.perf_counter()
                for r in range(LOOP):
                    one = K.eval_many([gts[i] for i in idx[r]], [[d[i] for i in idx[r]] for d in sets], CLASSES, tables)
                    for ev, o in zip(res, one):
                        for t in tables:
                            for key in ("bbox", "bev", "d3"):
                                assert ev["bootstrap"][t][key][r].tobytes() == o[t][1][key].tobytes(), (r, t, key)
                torch.cuda.synchronize()
                loop_s.append((time.perf_counter() - t0) / LOOP)
            rows.append(dict(frames=len(gts), sets=nsets, tables=[str(t) for t in tables], replicates=len(idx),
                             bootstrap_s=boot_s, peak_bytes=peak, loop_per_replicate_s=loop_s))
            print("K=%2d tables=%-12s R=%d bootstrap %s s (peak %.2f GB), plain eval_many per replicate %s s" % (
                nsets, "+".join(map(str, tables)), len(idx), ", ".join("%.3f" % t for t in boot_s), max(peak) / 1e9,
                ", ".join("%.3f" % t for t in loop_s)))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(dict(card=card, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
