"""Wall time of the KITTI evaluation with R = 1000 bootstrap replicates on a val-split-sized synthetic set (3769 frames,
classes Car, Pedestrian, Cyclist, one detection set), frame-level (bootstrap_indices) against drive-level
(bootstrap_groups over synthetic drives of consecutive frames), for the R11 table alone and with COCO.

    python tests/tools/kitti_eval_bootstrap_drive_timing.py [--out FILE.json] [--frames 3769] [--replicates 1000]

The two kinds alternate, twice each.  The first few drive-level replicates are checked bit for bit against plain
eval_many on their lists.  The card's name and power limit are read in the same run."""
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

CLASSES = ["Car", "Pedestrian", "Cyclist"]
CHECK = 3


def synthetic_drives(nframes, seed=0):
    """Drive labels of consecutive runs of 20..180 frames."""
    rs = np.random.RandomState(seed)
    out, d = [], 0
    while len(out) < nframes:
        out += [d] * int(rs.randint(20, 181))
        d += 1
    return np.array(out[:nframes])


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
    drives = synthetic_drives(len(gts))
    kinds = dict(frame=K.bootstrap_indices(len(gts), args.replicates, seed=0),
                 drive=K.bootstrap_groups(drives, args.replicates, seed=0))
    lengths = kinds["drive"].lengths
    print("drives: %d, drive-level list lengths min %d median %g max %d" % (
        len(np.unique(drives)), lengths.min(), np.median(lengths), lengths.max()))
    K.eval_many(gts[:50], [dts[:50]], CLASSES, (11,), bootstrap=K.bootstrap_indices(50, 4))     # warm-up
    rows = []
    for tables in ((11,), (11, "coco")):
        times = {k: [] for k in kinds}
        for rep in range(2):
            for kind, boot in kinds.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res = K.eval_many(gts, [dts], CLASSES, tables, bootstrap=boot)[0]
                torch.cuda.synchronize()
                times[kind].append(time.perf_counter() - t0)
                if kind == "drive" and rep == 0:
                    lists = boot
                    for r in range(CHECK):
                        one = K.eval_many([gts[i] for i in lists[r]], [[dts[i] for i in lists[r]]], CLASSES,
                                          tables)[0]
                        for t in tables:
                            for key in ("bbox", "bev", "d3"):
                                assert res["bootstrap"][t][key][r].tobytes() == one[t][1][key].tobytes(), (r, t, key)
        rows.append(dict(frames=len(gts), drives=int(len(np.unique(drives))), tables=[str(t) for t in tables],
                         replicates=args.replicates, frame_level_s=times["frame"], drive_level_s=times["drive"],
                         drive_lengths=dict(min=int(lengths.min()), median=float(np.median(lengths)),
                                            max=int(lengths.max()))))
        print("tables=%-10s R=%d frame-level %s s, drive-level %s s" % (
            "+".join(map(str, tables)), args.replicates, ", ".join("%.3f" % t for t in times["frame"]),
            ", ".join("%.3f" % t for t in times["drive"])))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(dict(card=card, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
