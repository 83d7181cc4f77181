"""GPU dev tool: kernel time of the dense BEV convs (conv2d_tma_kernel) on full 200 x 176 maps, every tile computed,
with CUDA events over many launches, and the fp32 output's error against an fp64 restatement.

    python tests/tools/dense_conv_timing.py [--root TREE] [--iters N]

--root imports the package from another checkout, so two builds can be timed alternately in one session.  Prints the
card's name, power limit and SM clock beside the numbers."""
import argparse
import os
import subprocess
import sys

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__)))))
ap.add_argument("--iters", type=int, default=50)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import torch  # noqa: E402
from sassd_b200 import ops  # noqa: E402

dev = torch.device("cuda:0")
ops.TILE_OCCUPANCY = False


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def layer(B, cin, cout, taps, iters):
    g = torch.Generator(device=dev).manual_seed(B * 1000 + cin + cout + taps)
    x = torch.randn(B, 200, 176, cin, device=dev, generator=g)
    w = torch.randn(taps, cin, cout, device=dev, generator=g) * 0.05
    scale = torch.rand(cout, device=dev, generator=g) + 0.5
    shift = torch.randn(cout, device=dev, generator=g) * 0.1
    xs = ops.SplitMap.from_float(x)
    _, f32 = ops.conv2d_split(xs, w, scale, shift, True, cout, out_split=False, out_f32=True)
    k = 3 if taps == 9 else 1
    f0 = x[:1].double().permute(0, 3, 1, 2)
    wk = w.double().view(k, k, cin, cout).permute(3, 2, 0, 1)
    ref = torch.nn.functional.conv2d(f0, wk, padding=k // 2).permute(0, 2, 3, 1)
    ref = (ref * scale.double() + shift.double()).clamp_min(0)
    err = ((f32[:1, ..., :cout].double() - ref).abs().max() / ref.abs().max()).item()
    for _ in range(3):
        ops.conv2d_split(xs, w, scale, shift, True, cout)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        ops.conv2d_split(xs, w, scale, shift, True, cout)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    flop = 2.0 * B * 200 * 176 * cin * cout * taps
    print("dense %dx%d %3d->%3d B=%-2d  %.4f ms  %.0f TFLOP/s algorithmic (x3 executed: %.0f)  rel err vs fp64 %.2e" %
          (k, k, cin, cout, B, ms, flop / ms / 1e9, 3 * flop / ms / 1e9, err), flush=True)
    return ms


print("root", os.path.abspath(args.root))
print("card", card())
for B in (1, 16):
    layer(B, 256, 256, 9, args.iters)
    layer(B, 320, 256, 9, args.iters)
    layer(B, 256, 256, 1, args.iters)
print("card", card())
