"""Time the loss path on the GPU: the target and loss kernels alone (CUDA events around each C-ABI call), and
SingleStageDetector.loss_points against forward_points(point_outputs=True) at batch 1 and 16, on synthetic clouds with
their cars as ground truth.

    python tests/tools/loss_timing.py [--iters 20] [--out DIR]

Prints one JSON object (with the card's name and power limit) and writes it to DIR/loss_timing.json."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    from sassd_b200 import ops
    from tests.test_losses import _frames, _model
    assert torch.cuda.is_available(), "loss_timing needs a CUDA device"
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    model = _model()
    res = dict(gpu=smi, iters=args.iters)
    for B in (1, 16):
        pts, gts, labels = _frames(B)
        model.enable_cuda_graph(B, 32768)

        def wall(fn):
            for _ in range(3):
                fn()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(args.iters):
                fn()
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) / args.iters * 1e3

        res["B%d_forward_points_point_outputs_ms" % B] = wall(lambda: model.forward_points(pts, point_outputs=True))
        res["B%d_loss_points_ms" % B] = wall(lambda: model.loss_points(pts, gts, labels))
        # the target and loss kernels alone
        model.loss_points(pts, gts, labels)
        ops.PROFILE = []
        for _ in range(args.iters):
            model.loss_points(pts, gts, labels)
        torch.cuda.synchronize()
        names = ("sassd_points_in_boxes", "sassd_aux_loss", "sassd_assign_rpn", "sassd_rpn_loss", "sassd_assign_pswarp",
                 "sassd_pswarp_loss")
        per = {n: 0.0 for n in names}
        for name, _, e0, e1 in ops.PROFILE:
            if name in per:
                per[name] += e0.elapsed_time(e1) / args.iters
        ops.PROFILE = None
        res["B%d_kernels_ms" % B] = {k: round(v, 4) for k, v in per.items()}
        res["B%d_targets_and_losses_ms" % B] = round(sum(per.values()), 4)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "loss_timing.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
