"""Wall time of evaluating KITTI result directories on a val-split-sized synthetic set (3769 frames, classes 0, 1, 2,
the official R11 table): the host path (kitti_data.read_labels of the label directory and every result directory,
then eval_many on the dicts, which runs the device evaluator) against kitti_eval.eval_dirs (the files parsed on the
device into AnnoBlocks, then the same eval_many), for K = 1 and K = 10 result directories.

    python tests/tools/kitti_eval_dirs_timing.py --out FILE.json [--frames 3769]

The label files are written with KITTI's %.2f fields (annos_to_kitti_label), the result directories by
test.write_results (%.4f and a score).  The two paths alternate, twice each, and their texts must agree.  eval_dirs
reports reading (files into pinned memory), parsing (copy to the device, scan, parse, synchronised) and evaluation
separately; the host path reports read_labels (reading and parsing together) and evaluation.  The page cache is warm
for both.  The card's name and power limit are read in the same run."""
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
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
sys.path.insert(0, os.path.join(ROOT, "tests", "tools"))
from coco_eval_timing import detection_sets  # noqa: E402
from make_golden_eval import synth_annos  # noqa: E402
from sassd_b200 import kitti_eval as K  # noqa: E402
from sassd_b200 import test as T  # noqa: E402
from sassd_b200.kitti_data import read_labels  # noqa: E402
from sassd_b200.results import annos_to_kitti_label  # noqa: E402


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
    sets = detection_sets(dts, 10)
    ids = list(range(args.frames))
    classes, tables = [0, 1, 2], (11,)
    rows = []
    with tempfile.TemporaryDirectory() as tmp:
        gt_dir = os.path.join(tmp, "label_2")
        os.makedirs(gt_dir)
        for i, g in zip(ids, gts):
            with open(os.path.join(gt_dir, "%06d.txt" % i), "w") as fh:
                lines = annos_to_kitti_label(dict(g, dimensions=np.asarray(g["dimensions"])[:, [1, 2, 0]]))
                fh.write("".join(l + "\n" for l in lines))
        dirs = []
        for k, s in enumerate(sets):
            dirs.append(os.path.join(tmp, "set%d" % k))
            T.write_results(dirs[-1], ids, s)
        K.eval_dirs(gt_dir, dirs[:2], ids[:50], classes, tables)        # warm-up (context, library, page cache)
        read_labels(gt_dir, ids)
        for nsets in (1, 10):
            times = {"host": [], "device": []}
            texts = {}
            for rep in range(2):
                for path in ("host", "device"):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    if path == "host":
                        gt = read_labels(gt_dir, ids)
                        dt = [read_labels(d, ids) for d in dirs[:nsets]]
                        t1 = time.perf_counter()
                        res = K.eval_many(gt, dt, classes, tables)
                        t = dict(read_labels=t1 - t0, eval=time.perf_counter() - t1)
                    else:
                        t = {}
                        res = K.eval_dirs(gt_dir, dirs[:nsets], ids, classes, tables, t)
                    torch.cuda.synchronize()
                    t["total"] = time.perf_counter() - t0
                    times[path].append(t)
                    texts[path] = [r[11][0] for r in res]
            assert texts["host"] == texts["device"], "host and device texts differ"
            rows.append(dict(frames=len(ids), dirs=nsets, host_s=times["host"], device_s=times["device"]))
            for path in ("host", "device"):
                print("K=%2d %-6s %s" % (nsets, path, "   ".join(
                    " ".join("%s %.3f" % kv for kv in t.items()) for t in times[path])))
    if args.out:
        with open(args.out, "w") as fh:
            json.dump(dict(card=card, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
