"""GPU dev tool: check the tensor-core (3xTF32 / 3xFP16) gathered-GEMM kernels against the FFMA path and fp64,
smallest cases first, printing diagnostics instead of asserting."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import numpy as np, torch
from sassd_b200 import ops

dev = torch.device("cuda:0")
torch.manual_seed(0)


def run(mode, M, cin, cout, taps, relu, H=0, W=0, B=0, nbr=None, d_rows=None, tag="", pattern=None, time_it=False):
    x = torch.randn(M, cin, device=dev)
    w = torch.randn(taps, cin, cout, device=dev) * 0.1
    if pattern == "ones":
        x.fill_(1.0); w.fill_(0.0); w[:, :, :] = 0.0
        for n in range(cout):
            w[0, n % cin, n] = 1.0 + n
    scale = torch.rand(cout, device=dev) + 0.5
    shift = torch.randn(cout, device=dev) * 0.1
    stride = (cout + 3) // 4 * 4
    outs = []
    for prec in (ops.PREC_FP32, ops.PREC_TF32X3, ops.PREC_F16X3):
        out = torch.zeros(M, stride, device=dev)
        ops.gconv(x, w, scale, shift, out, mode=mode, taps=taps, cin=cin, cout=cout, relu=relu, nbr=nbr, d_rows=d_rows,
                  rows_cap=M, batch=B, H=H, W=W, precision=prec)
        torch.cuda.synchronize()
        outs.append(out[:, :cout].clone())
    # fp64 reference
    xd, wd = x.double().cpu(), w.double().cpu()
    ref = torch.zeros(M, cout, dtype=torch.float64)
    if mode == ops.GCONV_ROWS or (mode == ops.GCONV_CONV2D and taps == 1):
        ref = xd @ wd[0]
    elif mode == ops.GCONV_CONV2D:
        img = xd.view(B, H, W, cin).permute(0, 3, 1, 2)
        wk = wd.view(3, 3, cin, cout).permute(3, 2, 0, 1)
        ref = torch.nn.functional.conv2d(img, wk, padding=1).permute(0, 2, 3, 1).reshape(M, cout)
    else:
        nb = nbr.cpu().long()
        for t in range(taps):
            o = torch.nonzero(nb[:, t] >= 0).view(-1)
            ref.index_add_(0, o, xd[nb[o, t]] @ wd[t])
    ref = ref * scale.double().cpu() + shift.double().cpu()
    if relu:
        ref = ref.clamp_min(0)
    e32 = (outs[0].double().cpu() - ref).abs().max().item()
    etc = (outs[1].double().cpu() - ref).abs().max().item()
    e16 = (outs[2].double().cpu() - ref).abs().max().item()
    sc = ref.abs().max().item()
    bad16 = e16 > 20 * max(e32, 1e-6 * sc)
    print("%-34s M=%-6d cin=%-3d cout=%-3d taps=%-2d  |ref|max %.3g  err ffma %.2e  tf32x3 %.2e  f16x3 %.2e  %s" %
          (tag, M, cin, cout, taps, sc, e32, etc, e16,
           "OK" if etc <= 20 * max(e32, 1e-6 * sc) and not bad16 else "MISMATCH"), flush=True)
    if bad16:
        d = (outs[2].double().cpu() - ref)
        bad = torch.nonzero(d.abs() > 1e-3 * max(sc, 1)).cpu()
        print("   f16 first bad (row, col):", bad[:8].tolist(), " n_bad", bad.shape[0])
        print("   f16 row0[:8]", outs[2][0, :8].tolist())
        print("   ref row0[:8]", ref[0, :8].tolist())
    if etc > 20 * max(e32, 1e-6 * sc):
        d = (outs[1].double().cpu() - ref)
        bad = torch.nonzero(d.abs() > 1e-3 * max(sc, 1)).cpu()
        print("   first bad (row, col):", bad[:8].tolist(), " n_bad", bad.shape[0])
        print("   tc  row0[:8]", outs[1][0, :8].tolist())
        print("   ref row0[:8]", ref[0, :8].tolist())
    if time_it:
        for prec, name in ((ops.PREC_FP32, "ffma"), (ops.PREC_TF32X3, "tf32x3"), (ops.PREC_F16X3, "f16x3")):
            out = torch.zeros(M, stride, device=dev)
            for _ in range(2):
                ops.gconv(x, w, scale, shift, out, mode=mode, taps=taps, cin=cin, cout=cout, relu=relu, nbr=nbr,
                          d_rows=d_rows, rows_cap=M, batch=B, H=H, W=W, precision=prec)
            torch.cuda.synchronize()
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(5):
                ops.gconv(x, w, scale, shift, out, mode=mode, taps=taps, cin=cin, cout=cout, relu=relu, nbr=nbr,
                          d_rows=d_rows, rows_cap=M, batch=B, H=H, W=W, precision=prec)
            e1.record(); torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / 5
            fl = 2.0 * M * cin * cout * taps
            print("   %-6s %.3f ms  %.1f TFLOP/s (algorithmic fp32)" % (name, ms, fl / ms / 1e9), flush=True)


stage = sys.argv[1] if len(sys.argv) > 1 else "all"
if stage in ("tiny", "all"):
    run(ops.GCONV_ROWS, 128, 32, 16, 1, False, tag="rows tiny pattern", pattern="ones")
    run(ops.GCONV_ROWS, 128, 32, 16, 1, False, tag="rows tiny")
    run(ops.GCONV_ROWS, 128, 32, 64, 1, True, tag="rows 1 tile N64")
    run(ops.GCONV_ROWS, 128, 64, 256, 1, True, tag="rows 1 tile N256 2 chunks")
    run(ops.GCONV_ROWS, 1000, 256, 256, 1, True, tag="rows multi-tile")
    run(ops.GCONV_ROWS, 1000, 28, 28, 1, False, tag="rows cin=28 (K tail) cout=28")
    run(ops.GCONV_ROWS, 777, 256, 20, 1, False, tag="rows 256->20")
if stage in ("conv", "all"):
    run(ops.GCONV_CONV2D, 2 * 12 * 10, 32, 16, 9, True, H=12, W=10, B=2, tag="conv2d small")
    run(ops.GCONV_CONV2D, 1 * 40 * 36, 256, 256, 9, True, H=40, W=36, B=1, tag="conv2d 256->256 40x36")
    run(ops.GCONV_CONV2D, 1 * 40 * 36, 320, 256, 9, True, H=40, W=36, B=1, tag="conv2d 320->256 40x36")
    run(ops.GCONV_CONV2D, 1 * 40 * 36, 256, 28, 9, True, H=40, W=36, B=1, tag="conv2d 256->28 40x36")
if stage in ("table", "all"):
    rs = np.random.RandomState(0)
    for cin, cout in ((4, 16), (16, 16), (16, 32), (32, 64), (64, 64)):
        M = 3000
        nbr = torch.from_numpy(np.where(rs.rand(M, 27) < 0.3, rs.randint(0, M, (M, 27)), -1).astype(np.int32)).to(dev)
        d_rows = torch.tensor([M - 37], dtype=torch.int32, device=dev)
        run(ops.GCONV_TABLE, M, cin, cout, 27, True, nbr=nbr, d_rows=None, tag="table %d->%d" % (cin, cout))
if stage in ("perf", "all"):
    run(ops.GCONV_CONV2D, 200 * 176, 256, 256, 9, True, H=200, W=176, B=1, tag="BEV 3x3 256->256 B=1", time_it=True)
    run(ops.GCONV_CONV2D, 4 * 200 * 176, 256, 256, 9, True, H=200, W=176, B=4, tag="BEV 3x3 256->256 B=4", time_it=True)


def run_tma(B, H, W, cin, cout, taps, relu, tag, time_it=False):
    x = torch.randn(B, H, W, cin, device=dev)
    w = torch.randn(taps, cin, cout, device=dev) * 0.05
    scale = torch.rand(cout, device=dev) + 0.5
    shift = torch.randn(cout, device=dev) * 0.1
    xs = ops.SplitMap.from_float(x)
    sp, f32 = ops.conv2d_split(xs, w, scale, shift, relu, cout, out_split=True, out_f32=True)
    torch.cuda.synchronize()
    img = x.double().cpu().permute(0, 3, 1, 2)
    k = 3 if taps == 9 else 1
    wk = w.double().cpu().view(k, k, cin, cout).permute(3, 2, 0, 1)
    ref = torch.nn.functional.conv2d(img, wk, padding=k // 2).permute(0, 2, 3, 1)
    ref = ref * scale.double().cpu() + shift.double().cpu()
    if relu:
        ref = ref.clamp_min(0)
    sc = ref.abs().max().item()
    e1 = (f32[..., :cout].double().cpu() - ref).abs().max().item()
    e2 = (sp.float().double().cpu() - ref).abs().max().item()
    ok = e1 < 2e-5 * max(sc, 1) and e2 < 2e-5 * max(sc, 1)
    print("%-30s B=%d %dx%d cin=%-3d cout=%-3d taps=%d |ref|max %.3g  err f32-out %.2e  err split-out %.2e  %s" %
          (tag, B, H, W, cin, cout, taps, sc, e1, e2, "OK" if ok else "MISMATCH"), flush=True)
    if not ok:
        d = (f32[..., :cout].double().cpu() - ref).abs()
        bad = torch.nonzero(d > 1e-3 * max(sc, 1))
        print("   n_bad", bad.shape[0], "first", bad[:6].tolist())
        print("   got", f32[0, 0, 0, :6].tolist(), "ref", ref[0, 0, 0, :6].tolist())
    if time_it:
        for _ in range(2):
            ops.conv2d_split(xs, w, scale, shift, relu, cout, out_split=True, out_f32=False)
        torch.cuda.synchronize()
        e0 = torch.cuda.Event(enable_timing=True); e1_ = torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            ops.conv2d_split(xs, w, scale, shift, relu, cout, out_split=True, out_f32=False)
        e1_.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1_) / 5
        print("   tma f16x3 %.3f ms  %.1f TFLOP/s (algorithmic fp32)" % (ms, 2.0 * B * H * W * cin * cout * taps / ms / 1e9), flush=True)


if stage in ("tma", "all"):
    run_tma(1, 8, 16, 64, 32, 1, False, "tma 1 tile 1x1")
    run_tma(1, 8, 16, 64, 32, 9, True, "tma 1 tile 3x3")
    run_tma(2, 24, 20, 256, 256, 9, True, "tma 256->256 partial tiles")
    run_tma(1, 40, 36, 320, 256, 9, True, "tma 320->256")
    run_tma(1, 40, 36, 256, 28, 9, True, "tma 256->28")
    run_tma(1, 40, 36, 28, 28, 1, False, "tma 28->28 1x1")
    run_tma(1, 40, 36, 256, 20, 1, False, "tma 256->20 1x1")
if stage in ("tmaperf", "all"):
    run_tma(1, 200, 176, 256, 256, 9, True, "tma BEV 3x3 B=1", time_it=True)
    run_tma(4, 200, 176, 256, 256, 9, True, "tma BEV 3x3 B=4", time_it=True)
if stage in ("tmaperf1",):
    run_tma(1, 200, 176, 256, 256, 9, True, "tma BEV 3x3 B=1", time_it=True)
    run_tma(1, 200, 176, 256, 256, 1, True, "tma BEV 1x1 B=1", time_it=True)
    run_tma(4, 200, 176, 256, 256, 1, True, "tma BEV 1x1 B=4", time_it=True)
print("done")
if stage in ("tmafull",):
    run_tma(1, 200, 176, 256, 28, 9, True, "tma full 256->28")
    run_tma(1, 200, 176, 28, 28, 1, False, "tma full 28->28 1x1")
    run_tma(1, 200, 176, 256, 20, 1, False, "tma full 256->20 1x1")
    run_tma(2, 200, 176, 256, 20, 1, False, "tma full B=2 256->20 1x1")
    run_tma(1, 200, 176, 256, 64, 9, True, "tma full 256->64")
    run_tma(1, 200, 176, 256, 128, 9, True, "tma full 256->128")


def tile_masks(nb, n_rows):
    """What the rulebook kernels record: per 128-row tile, the taps that occur among its first n_rows rows."""
    M, taps = nb.shape
    nt = (M + 127) // 128
    pad = np.full((nt * 128, taps), -1, np.int64)
    pad[:n_rows] = nb[:n_rows]
    present = (pad.reshape(nt, 128, taps) >= 0).any(1)
    return (present * (1 << np.arange(taps))[None, :]).sum(1).astype(np.int32)


def run_split(M, cin, cout, taps, relu, tag, density=0.3, masks=False, absent=0.0):
    """masks: pass the per-tile tap masks (tap skipping); absent: fraction of (tile, tap) combinations with no
    neighbour at all, so that whole chunks really are skipped."""
    rs = np.random.RandomState(cin * 100 + cout)
    x = torch.randn(M, cin, device=dev)
    w = torch.randn(taps, cin, cout, device=dev) * 0.1
    scale = torch.rand(cout, device=dev) + 0.5
    shift = torch.randn(cout, device=dev) * 0.1
    nbr = tm = None
    if taps > 1:
        nb = np.where(rs.rand(M, taps) < density, rs.randint(0, M, (M, taps)), -1).astype(np.int32)
        if absent > 0:
            gone = rs.rand((M + 127) // 128, taps) < absent
            gone[0, :] = True        # a tile with no pair at all must still produce act(shift)
            nb[np.repeat(gone, 128, axis=0)[:M]] = -1
        nbr = torch.from_numpy(nb).to(dev)
        if masks:
            tm = torch.from_numpy(tile_masks(nb, M - 5)).to(dev)
    d_rows = torch.tensor([M - 5], dtype=torch.int32, device=dev)
    planes = ops.features_to_split(x)
    out, of = ops.spconv_split(planes, w, scale, shift, relu, cout, M, nbr=nbr, d_rows=d_rows, want_f32=True,
                               tile_mask=tm)
    torch.cuda.synchronize()
    xd, wd = x.double().cpu(), w.double().cpu()
    ref = torch.zeros(M, cout, dtype=torch.float64)
    if taps == 1:
        ref = xd @ wd[0]
    else:
        nb = nbr.cpu().long()
        for t in range(taps):
            o = torch.nonzero(nb[:, t] >= 0).view(-1)
            ref.index_add_(0, o, xd[nb[o, t]] @ wd[t])
    ref = ref * scale.double().cpu() + shift.double().cpu()
    if relu:
        ref = ref.clamp_min(0)
    n = M - 5
    sc = ref.abs().max().item()
    e1 = (of[:n, :cout].double().cpu() - ref[:n]).abs().max().item()
    e2 = (ops.split_rows_float(out, cout)[:n].double().cpu() - ref[:n]).abs().max().item()
    ok = e1 < 2e-5 * max(sc, 1) and e2 < 2e-5 * max(sc, 1)
    print("%-26s M=%-6d cin=%-3d cout=%-3d taps=%-2d |ref|max %.3g  err f32 %.2e  err split %.2e  %s" %
          (tag, M, cin, cout, taps, sc, e1, e2, "OK" if ok else "MISMATCH"), flush=True)
    if not ok:
        d = (of[:n, :cout].double().cpu() - ref[:n]).abs()
        bad = torch.nonzero(d > 1e-3 * max(sc, 1))
        print("   n_bad", bad.shape[0], "first", bad[:6].tolist())
        print("   got", of[0, :6].tolist(), "ref", ref[0, :6].tolist())


if stage in ("split",):
    run_split(128, 8, 16, 1, False, "split rows 1 tile")
    run_split(300, 4, 16, 27, True, "split table 4->16")
    run_split(3000, 16, 16, 27, True, "split table 16->16")
    run_split(3000, 16, 32, 27, True, "split table 16->32")
    run_split(3000, 32, 64, 27, True, "split table 32->64")
    run_split(3000, 64, 64, 27, True, "split table 64->64")
    run_split(20000, 64, 64, 27, True, "split table 64->64 big")
    run_split(3000, 64, 64, 1, True, "split rows 64->64")
    # tap skipping (tile masks) with whole (tile, tap) combinations absent; <= 74 tiles also take the cluster tap split
    run_split(300, 4, 16, 27, True, "skip 4->16", masks=True, absent=0.5)
    run_split(3000, 16, 32, 27, True, "skip 16->32", masks=True, absent=0.5)
    run_split(3000, 32, 32, 27, True, "skip 32->32", masks=True, absent=0.4)
    run_split(3000, 64, 64, 27, True, "skip 64->64 (tap split)", masks=True, absent=0.4)
    run_split(9400, 64, 64, 27, True, "skip 64->64 74 tiles", masks=True, absent=0.4)
    run_split(9500, 64, 64, 27, True, "skip 64->64 75 tiles", masks=True, absent=0.4)
    run_split(20000, 64, 64, 27, True, "skip 64->64 big", masks=True, absent=0.4)
    run_split(20000, 64, 64, 27, True, "skip 64->64 big sparse", masks=True, absent=0.9, density=0.5)
    print("done split")
if stage in ("splitperf",):
    M, cin, cout, taps = 120000, 64, 64, 27
    rs = np.random.RandomState(1)
    x = torch.randn(M, cin, device=dev)
    w = torch.randn(taps, cin, cout, device=dev) * 0.1
    # spatially coherent-ish neighbours: mostly nearby rows
    nb = np.where(rs.rand(M, taps) < 0.35, np.clip(np.arange(M)[:, None] + rs.randint(-300, 300, (M, taps)), 0, M - 1), -1).astype(np.int32)
    nbr = torch.from_numpy(nb).to(dev)
    d_rows = torch.tensor([M], dtype=torch.int32, device=dev)
    planes = ops.features_to_split(x)
    P = int((nb >= 0).sum())

    def timed(tag, nbr_t, tm, n_chunks):
        for _ in range(2):
            ops.spconv_split(planes, w, None, None, True, cout, M, nbr=nbr_t, d_rows=d_rows, tile_mask=tm)
        torch.cuda.synchronize()
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            ops.spconv_split(planes, w, None, None, True, cout, M, nbr=nbr_t, d_rows=d_rows, tile_mask=tm)
        e1.record(); torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 5
        pairs = int((nbr_t.cpu().numpy() >= 0).sum())
        print("splitperf %s: %.3f ms  pair-model %.0f GB/s  (%.0f clk per executed chunk)" % (
            tag, ms, pairs * (4 * cin + 4 * cout + 8) / ms / 1e6,
            ms * 1e-3 * 1.98e9 / (n_chunks / torch.cuda.get_device_properties(0).multi_processor_count)), flush=True)

    timed("all taps", nbr, None, 27 * (M / 128))
    # 30 % of the (tile, tap) combinations absent, like the level-2 SubM rulebook of a KITTI-shaped cloud
    nb2 = nb.copy()
    gone = rs.rand((M + 127) // 128, taps) < 0.3
    nb2[np.repeat(gone, 128, axis=0)[:M]] = -1
    tm = tile_masks(nb2, M)
    timed("30% tile-taps absent, masks", torch.from_numpy(nb2).to(dev), torch.from_numpy(tm).to(dev),
          float(sum(bin(int(v) & 0x7ffffff).count("1") for v in tm)))
    timed("30% tile-taps absent, no masks", torch.from_numpy(nb2).to(dev), None, 27 * (M / 128))
    # one-frame layer sizes: 7 500 rows (59 tiles, tap split) and 14 000 rows (110 tiles)
    for rows in (5300, 7500, 14000):
        sub = torch.from_numpy(np.where(nb[:rows] >= rows, -1, nb[:rows])).to(dev)
        d_rows = torch.tensor([rows], dtype=torch.int32, device=dev)
        M_full, M = M, rows
        timed("%d rows" % rows, sub, torch.from_numpy(tile_masks(sub.cpu().numpy(), rows)).to(dev), 27 * (rows / 128))
        M = M_full
        d_rows = torch.tensor([M], dtype=torch.int32, device=dev)

