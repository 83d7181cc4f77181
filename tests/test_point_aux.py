"""SA-SSD's auxiliary point-wise network in eval mode (csrc/point_aux.cu, ops.three_nn / ops.point_aux_head,
SpMiddleFHD.forward(is_test=False), forward_points(point_outputs=True)).

* sassd_three_nn is checked bit for bit against the reference's own pointnet2 kernel (interpolate_gpu.cu, compiled
  unmodified into oracle/_ref/libpointnet2_ref.so by build()), on a forward pass's level coordinates and on
  constructed sets: ties, frames with one or two centres, an empty frame.
* The oracle (oracle/point_aux.py) is checked on the CPU against a literal transcription of the reference loop.
* The whole branch is checked against the CPU oracle chain: voxelize -> vxnet_middle -> aux head."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import point_aux as PA

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _aux_weights(seed=7):
    g = torch.Generator().manual_seed(seed)
    return {"neck.point_fc.weight": torch.randn(64, 160, generator=g) / np.sqrt(160.0),
            "neck.point_cls.weight": torch.randn(1, 64, generator=g) / 8.0,
            "neck.point_reg.weight": torch.randn(3, 64, generator=g) / 8.0}


def _reference_loop(unknown, known):
    """interpolate_gpu.cu:9-56 transcribed: per unknown row, every known row in order, other batches skipped, double
    bests initialised to 1e40, strict <.  d as the kernel's SASS computes it (fma(dz, dz, fma(dx, dx, dy * dy)))."""
    n = unknown.shape[0]
    dist2 = np.zeros((n, 3), np.float32)
    idx = np.zeros((n, 3), np.int32)
    for i in range(n):
        ub = unknown[i, 0]
        d_all = PA.sq_dist32(np.broadcast_to(unknown[i, 1:], (known.shape[0], 3)), known[:, 1:])
        best1 = best2 = best3 = 1e40
        besti1 = besti2 = besti3 = 0
        for k in range(known.shape[0]):
            if known[k, 0] != ub:
                continue
            d = float(d_all[k])
            if d < best1:
                best3, besti3 = best2, besti2
                best2, besti2 = best1, besti1
                best1, besti1 = d, k
            elif d < best2:
                best3, besti3 = best2, besti2
                best2, besti2 = d, k
            elif d < best3:
                best3, besti3 = d, k
        with np.errstate(over="ignore"):            # 1e40 -> +inf, as the kernel stores it
            dist2[i] = np.array([best1, best2, best3], np.float64).astype(np.float32)
        idx[i] = (besti1, besti2, besti3)
    return idx, dist2


def _tie_sets(rng):
    """Known / unknown (b, x, y, z) sets on a coarse grid (duplicate centres, equidistant points), over four frames:
    frame 1 has a single centre, frame 2 two, frame 3 none."""
    grid = np.float32(0.25)
    k0 = rng.integers(0, 6, (40, 3)).astype(np.float32) * grid
    k0 = np.concatenate([k0, k0[:8]])                                    # duplicate centres
    known = [np.concatenate([np.zeros((len(k0), 1), np.float32), k0], 1),
             np.array([[1, 0.5, 0.5, 0.5]], np.float32),
             np.array([[2, 0.0, 0.0, 0.0], [2, 1.0, 0.0, 0.0]], np.float32)]
    known = np.concatenate(known)[rng.permutation(len(k0) + 3)]         # frames interleaved: the loop skips
    u0 = rng.integers(0, 12, (60, 3)).astype(np.float32) * (grid / 2)    # midpoints: equidistant from centres
    u0 = np.concatenate([u0, k0[:5], rng.random((20, 3)).astype(np.float32)])
    unknown = np.concatenate([np.concatenate([np.zeros((len(u0), 1), np.float32), u0], 1),
                              np.array([[1, 0, 0, 0], [1, 3, 2, 1]], np.float32),
                              np.array([[2, 0.5, 0, 0], [2, 0.5, 1, 1], [2, 7, 0, 0]], np.float32),
                              np.array([[3, 1, 1, 1]], np.float32)])
    return unknown, known


# ------------------------------------------------------------------------------------------------------------ CPU
def test_oracle_three_nn_matches_the_reference_loop():
    rng = np.random.default_rng(0)
    unknown, known = _tie_sets(rng)
    want = _reference_loop(unknown, known)
    got = PA.three_nn(unknown, known)
    assert np.array_equal(got[0], want[0])
    assert np.array_equal(got[1].view(np.int32), want[1].view(np.int32))
    assert np.isinf(want[1][unknown[:, 0] == 1][:, 1:]).all() and np.isinf(want[1][unknown[:, 0] == 3]).all()
    # continuous random sets over several frames, including a small k-d tree query (ball fallback)
    for seed in range(3):
        r = np.random.default_rng(10 + seed)
        known = np.concatenate([r.integers(0, 3, (300, 1)), r.random((300, 3)) * 4], 1).astype(np.float32)
        unknown = np.concatenate([r.integers(0, 3, (150, 1)), r.random((150, 3)) * 4], 1).astype(np.float32)
        want = _reference_loop(unknown, known)
        for kq in (3, 8):
            got = PA.three_nn(unknown, known, k_query=kq)
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def test_oracle_fma_is_correctly_rounded():
    r = np.random.default_rng(1)
    a, b, c = (r.standard_normal(20000).astype(np.float32) for _ in range(3))
    got = PA.fma32(a, b, c)
    from fractions import Fraction
    for i in range(0, 20000, 97):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(exact))
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(np.float32(v).view(np.int32)) & 1))
        assert got[i] == best, i


def test_oracle_tensor2points_matches_torch_fp32():
    rng = np.random.default_rng(2)
    coords = np.concatenate([rng.integers(0, 4, (5000, 1)), rng.integers(0, 11, (5000, 1)),
                             rng.integers(0, 400, (5000, 1)), rng.integers(0, 352, (5000, 1))], 1).astype(np.int32)
    for vs in PA.LEVEL_VOXEL_SIZES:
        # transforms.py:218-223 verbatim, fp32 torch on the CPU
        indices = torch.from_numpy(coords).float()
        offset = torch.Tensor((0, -40., -3.))
        voxel_size = torch.Tensor(vs)
        indices[:, 1:] = indices[:, [3, 2, 1]] * voxel_size + offset + .5 * voxel_size
        got = PA.tensor2points(coords, vs)
        assert np.array_equal(got.view(np.int32), indices.numpy().view(np.int32)), vs


def test_training_mode_raises_and_aux_weights_load():
    from sassd_b200 import checkpoint
    from sassd_b200.necks import SpMiddleFHD

    class Holder(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.neck = SpMiddleFHD([40, 1600, 1408], 4)

    m = Holder()
    m.neck.train()
    with pytest.raises(NotImplementedError):
        m.neck(torch.zeros((1, 4)), torch.zeros((1, 4), dtype=torch.int32), 1, is_test=False)
    sd = _aux_weights()
    n, missing = checkpoint.load_state_dict_into(m, sd)
    assert n == 3 and not any(k.startswith("neck.point_") for k in missing)
    for k, v in sd.items():
        assert torch.equal(m.state_dict()[k], v)


# ------------------------------------------------------------------------------------------------------------ GPU
def _ref_lib():
    from oracle import pointnet2_ref
    path = pointnet2_ref.path()
    assert os.path.isfile(path), ("%s is missing: __graft_entry__.build() compiles the reference's interpolate_gpu.cu "
                                  "into it" % path)
    L = ctypes.CDLL(path)
    fn = L._Z29three_nn_kernel_launcher_fastiiPKfS0_PfPiP11CUstream_st
    fn.restype = None
    fn.argtypes = [ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 5
    return fn


def _ref_three_nn(fn, unknown, known):
    """The reference kernel on (b, x, y, z) rows (device tensors)."""
    n = unknown.shape[0]
    dist2 = torch.empty((n, 3), dtype=torch.float32, device="cuda")
    idx = torch.empty((n, 3), dtype=torch.int32, device="cuda")
    fn(n, known.shape[0], unknown.data_ptr(), known.data_ptr(), dist2.data_ptr(), idx.data_ptr(),
       torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return idx.cpu().numpy(), dist2.cpu().numpy()


def _compare_with_reference(fn, points_mean, levels, idx, dist2):
    """points_mean [n,4] (b,x,y,z) host; levels: three coords [M,4] host; idx / dist2 [n,3,3] host from ops.three_nn."""
    u = torch.from_numpy(np.ascontiguousarray(points_mean)).cuda()
    for l, (coords, vs) in enumerate(zip(levels, PA.LEVEL_VOXEL_SIZES)):
        known = torch.from_numpy(PA.tensor2points(coords, vs)).cuda()
        ri, rd = _ref_three_nn(fn, u, known)
        assert np.array_equal(idx[:, l], ri), "level %d: idx differs from the reference kernel" % (l + 1)
        assert np.array_equal(dist2[:, l].view(np.int32), rd.view(np.int32)), "level %d: dist2 differs" % (l + 1)


def _model(precision=None):
    import sassd_b200 as S
    from sassd_b200 import checkpoint
    cfg = S.Config.fromfile(os.path.join(ROOT, "configs", "car_cfg.py"))
    model, _, _ = S.build_from_config(cfg, device="cuda:0")
    sd = checkpoint.make_synthetic_state_dict(0, 1)
    sd.update(_aux_weights())
    checkpoint.load_state_dict_into(model, sd)
    if precision is not None:
        model.set_precision(precision)
    return model, sd


def _clouds(B):
    from sassd_b200.synth import synth_cloud
    return [synth_cloud(b % 4) if b < 4 else synth_cloud(b) for b in range(B)]


def _step(model, pts, point_outputs=True):
    from sassd_b200 import ops
    dev = torch.device("cuda:0")
    hp, ho, counts = model.stage_points(pts)
    det, nd, status, aux = model.forward_device(hp.to(dev), ho.to(dev), len(pts), max(counts), point_outputs=point_outputs)
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    n0 = int(aux["frame_rows"][-1].item())
    return det, nd, aux, n0, ops


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 2, 16])
def test_three_nn_bit_identical_to_reference_on_forward_levels(B):
    fn = _ref_lib()
    model, _ = _model()
    _, _, aux, n0, _ = _step(model, _clouds(B))
    levels = [m.indices.cpu().numpy() for m in aux["middle"]]
    pm = aux["points_mean"][:n0].cpu().numpy()
    assert np.array_equal(pm[:, 0], aux["coors"][:n0, 0].float().cpu().numpy())
    _compare_with_reference(fn, pm, levels, aux["idx"][:n0].cpu().numpy(), aux["dist2"][:n0].cpu().numpy())
    print("B=%d: %d points, level rows %s" % (B, n0, [len(c) for c in levels]))


def _grid_sets(rng):
    """Constructed level-0 rows and level coordinates over four frames: frame 0 dense with ties (means on centre
    midpoints and on centres), frame 1 one centre per level, frame 2 two, frame 3 empty (no rows anywhere)."""
    lv_coords = []
    for l, vs in enumerate(PA.LEVEL_VOXEL_SIZES):
        rows = []
        c0 = np.unique(rng.integers(0, 6, (60, 3)), axis=0)
        rows.append(np.concatenate([np.zeros((len(c0), 1), np.int64), c0], 1))
        rows.append(np.array([[1, 2, 3, 4]]))
        rows.append(np.array([[2, 1, 1, 1], [2, 1, 1, 3]]))
        c = np.concatenate(rows).astype(np.int32)
        lv_coords.append(c)
    # unknown points: frame 0 on level-1 centres and midpoints between them, frames 1-2 a few points
    cen = PA.tensor2points(lv_coords[0], PA.LEVEL_VOXEL_SIZES[0])
    f0 = cen[cen[:, 0] == 0][:, 1:]
    mids = ((f0[:-1] + f0[1:]) * np.float32(0.5)).astype(np.float32)
    u0 = np.concatenate([f0, mids, f0 + rng.random(f0.shape).astype(np.float32) * 0.3])
    pts = [np.concatenate([np.zeros((len(u0), 1), np.float32), u0], 1),
           np.array([[1, 0.3, -39.5, -2.5], [1, 5, 5, 5]], np.float32),
           np.array([[2, 0.35, -39.85, -2.7], [2, 0.15, -39.8, -2.6], [2, 9, -30, 0]], np.float32)]
    pm = np.concatenate(pts)
    return pm, lv_coords


@pytest.mark.gpu
def test_three_nn_bit_identical_to_reference_on_constructed_sets():
    from sassd_b200 import ops
    fn = _ref_lib()
    pm, lv = _grid_sets(np.random.default_rng(3))
    dev = torch.device("cuda:0")
    n0 = pm.shape[0]
    cap0 = n0 + 37                                             # capacity beyond the row count, as in the step
    mean = torch.zeros((cap0, 4), dtype=torch.float32, device=dev)
    mean[:n0, :3] = torch.from_numpy(pm[:, 1:]).to(dev)
    coors0 = torch.zeros((cap0, 4), dtype=torch.int32, device=dev)
    coors0[:n0, 0] = torch.from_numpy(pm[:, 0].astype(np.int32)).to(dev)
    levels = []
    for c in lv:
        t = torch.full((len(c) + 5, 4), -7, dtype=torch.int32, device=dev)
        t[:len(c)] = torch.from_numpy(c).to(dev)
        levels.append((t, torch.tensor([len(c)], dtype=torch.int32, device=dev)))
    idx, dist2, got_pm = ops.three_nn(mean, coors0, torch.tensor([n0], dtype=torch.int32, device=dev), levels,
                                      points_mean=True)
    torch.cuda.synchronize()
    assert np.array_equal(got_pm[:n0].cpu().numpy(), pm)
    idx, dist2 = idx[:n0].cpu().numpy(), dist2[:n0].cpu().numpy()
    _compare_with_reference(fn, pm, lv, idx, dist2)
    f1, f2 = pm[:, 0] == 1, pm[:, 0] == 2
    assert np.isinf(dist2[f1][:, :, 1:]).all() and (idx[f1][:, :, 1:] == 0).all()
    assert np.isinf(dist2[f2][:, :, 2]).all() and np.isfinite(dist2[f2][:, :, :2]).all()
    # the oracle agrees too (it is what the end-to-end checks below use)
    for l, (c, vs) in enumerate(zip(lv, PA.LEVEL_VOXEL_SIZES)):
        oi, od = PA.three_nn(pm, PA.tensor2points(c, vs))
        assert np.array_equal(oi, idx[:, l]) and np.array_equal(od, dist2[:, l])


@pytest.mark.gpu
def test_point_aux_head_matches_the_oracle():
    from sassd_b200 import ops
    model, sd = _model()
    _, _, aux, n0, _ = _step(model, _clouds(2))
    idx, dist2 = aux["idx"], aux["dist2"]
    g = torch.Generator().manual_seed(5)
    feats = [torch.randn(m.rows_cap, c, generator=g) for m, c in zip(aux["middle"], (32, 64, 64))]
    fc_t, w_out = model.neck._point_weights()
    ih, dh = idx[:n0].cpu().numpy(), dist2[:n0].cpu().numpy()
    for split in (False, True):
        dev_f = [f.cuda() for f in feats]
        if split:
            planes = [ops.features_to_split(f) for f in dev_f]
            levels = [ops.point_level(split=p, channels=f.shape[1]) for p, f in zip(planes, dev_f)]
            host_f = [ops.split_rows_float(p, f.shape[1]).cpu().numpy() for p, f in zip(planes, dev_f)]
        else:
            levels = [ops.point_level(feat=f) for f in dev_f]
            host_f = [f.numpy() for f in feats]
        cls, reg = ops.point_aux_head(idx, dist2, aux["frame_rows"][-1:], levels, fc_t, w_out)
        torch.cuda.synchronize()
        ps = [PA.three_interpolate(f, ih[:, l], PA.interpolate_weights(dh[:, l])) for l, f in enumerate(host_f)]
        x = torch.from_numpy(np.concatenate(ps, 1))
        pw = x @ sd["neck.point_fc.weight"].t()
        want_cls = (pw @ sd["neck.point_cls.weight"].t()).numpy()[:, 0]
        want_reg = (pw @ sd["neck.point_reg.weight"].t()).numpy()
        # fp32 sums of 160 and 64 products in another order (torch's CPU matmul): about 1e-6 of the output scale
        for got, want in ((cls[:n0].cpu().numpy(), want_cls), (reg[:n0].cpu().numpy(), want_reg)):
            scale = float(np.abs(want).max())
            err = float(np.abs(got - want).max())
            assert err <= 2e-6 * scale, "split=%s: max error %g at scale %g" % (split, err, scale)


def _oracle_chain(sd, pts, points_mean):
    """voxelize -> SimpleVoxel -> vxnet_middle -> aux head, unknown points = the step's own means."""
    from oracle import ref_pipeline as O
    vl, cl, nl = [], [], []
    for p in pts:
        v, c, n = O.points_to_voxel(p, [0.05, 0.05, 0.1], [0, -40., -3., 70.4, 40., 1.], 5, 20000)
        vl.append(v); cl.append(c); nl.append(n)
    voxels, coors, num = O.merge_batch(vl, cl, nl)
    vx = O.simple_voxel(voxels, num)
    middle = PA.vxnet_middle(sd, vx, coors, [40, 1600, 1408])
    out = PA.point_head(sd, points_mean, [(f.numpy(), c) for f, c in middle])
    return vx.numpy(), coors, middle, out


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 2, 16])
@pytest.mark.parametrize("precision", ["f16x3", "fp32"])
def test_forward_points_point_outputs_match_the_oracle(B, precision):
    from sassd_b200 import ops
    model, sd = _model(ops.PREC_FP32 if precision == "fp32" else None)
    pts = _clouds(B)
    res, points, aux = model.forward_points(pts, point_outputs=True, return_aux=True)
    fr = aux["frame_rows"].cpu().numpy()
    n0 = int(fr[-1])
    pm = aux["points_mean"][:n0].cpu().numpy()
    vx, coors, middle, want = _oracle_chain(sd, pts, pm)
    assert np.array_equal(aux["coors"][:n0].cpu().numpy(), coors)
    for (f, c), m in zip(middle, aux["middle"]):
        assert np.array_equal(m.indices.cpu().numpy(), c)
    assert np.array_equal(aux["idx"][:n0].cpu().numpy(), want["idx"]), "nearest centres differ from the oracle"
    xyz = np.concatenate([p["xyz"] for p in points])
    assert np.array_equal(xyz, aux["mean"][:n0, :3].cpu().numpy()), "xyz must be the step's mean rows"
    assert np.abs(xyz - vx[:, :3]).max() <= 1e-6 * max(1.0, float(np.abs(vx[:, :3]).max()))
    cls = np.concatenate([p["cls"] for p in points])
    reg = np.concatenate([p["reg"] for p in points])
    for b in range(B):
        assert len(points[b]["cls"]) == fr[b + 1] - fr[b]
    # head quantities: 1e-4 of their scale, the bar the detection heads are held to
    for got, exp, what in ((cls, want["cls"][:, 0], "cls"), (reg, want["reg"], "reg")):
        scale = max(1.0, float(np.abs(exp).max()))
        err = float(np.abs(got - exp).max())
        assert err <= 1e-4 * scale, "%s: max error %g at scale %g" % (what, err, scale)
    print("B=%d %s: %d points, cls err %.2e, reg err %.2e" % (B, precision, n0, np.abs(cls - want["cls"][:, 0]).max(),
                                                           np.abs(reg - want["reg"]).max()))


def _same_detections(a, b):
    for x, y in zip(a, b):
        for k in ("boxes_lidar", "scores", "label_preds"):
            assert (x[k] is None) == (y[k] is None)
            if x[k] is not None:
                assert np.array_equal(x[k], y[k]), k


@pytest.mark.gpu
def test_neck_is_test_false_and_unchanged_detections():
    model, _ = _model()
    pts = _clouds(2)
    det0, nd0, aux0, n0, _ = _step(model, pts, point_outputs=False)
    det1, nd1, aux1, n1, _ = _step(model, pts, point_outputs=True)
    assert n0 == n1 and torch.equal(nd0, nd1)
    for b in range(2):
        k = int(nd0[b])
        assert torch.equal(det0[b, :k], det1[b, :k]), "detections change with point_outputs"
    # the reference signature on the same capacity-sized inputs
    fr = aux1["frame_rows"]
    x, conv6, (pm, cls, reg) = model.neck(aux1["mean"], aux1["coors"], 2, is_test=False, d_rows=fr[2:3])
    assert pm.shape == (n1, 4) and cls.shape == (n1, 1) and reg.shape == (n1, 3)
    assert torch.equal(pm, aux1["points_mean"][:n1])
    assert torch.equal(cls[:, 0], aux1["point_cls"][:n1]) and torch.equal(reg, aux1["point_reg"][:n1])
    # exact-shape inputs, as a reference caller passes them
    _, _, (pm2, cls2, reg2) = model.neck(aux1["mean"][:n1], aux1["coors"][:n1], 2, is_test=False)
    torch.cuda.synchronize()
    assert torch.equal(pm2, pm)
    assert np.abs((cls2 - cls).cpu().numpy()).max() <= 1e-5 and np.abs((reg2 - reg).cpu().numpy()).max() <= 1e-5
    assert x.shape[1] == 256 and conv6.shape[1] == 256


@pytest.mark.gpu
def test_forward_points_with_crop_metas_and_graph_table(golden_dir):
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from test_kitti_format import _sweeps_and_metas
    model, _ = _model()
    pts, metas, planes = _sweeps_and_metas(golden_dir, [0, 1])
    for kw in ({}, dict(frustum_planes=planes), dict(metas=metas), dict(frustum_planes=planes, metas=metas)):
        plain = model.forward_points(pts, **kw)
        res, points = model.forward_points(pts, point_outputs=True, **kw)
        if "metas" in kw:
            for a, b in zip(plain, res):
                assert set(a) == set(b) and all(np.array_equal(a[k], b[k]) for k in a)
        else:
            _same_detections(plain, res)
        assert len(points) == 2 and all(len(p["cls"]) > 0 for p in points)
    # captured: replay == eager, bit for bit (points), and a reload of point_fc is picked up by a re-capture
    model.enable_cuda_graph(2, 131072)
    for kw in ({}, dict(frustum_planes=planes), dict(metas=metas)):
        eager = model.forward_points(pts, point_outputs=True, return_aux=True, **kw)
        graph = model.forward_points(pts, point_outputs=True, **kw)
        for e, g in zip(eager[1], graph[1]):
            for k in ("xyz", "cls", "reg"):
                assert np.array_equal(e[k], g[k]), (kw, k)
    assert {k for k in model._graphs if k[2]} == {(False, False, True), (True, False, True), (False, True, True)}
    before = model.forward_points(pts, point_outputs=True)[1]
    from sassd_b200 import checkpoint
    w = model.neck.point_fc.weight.detach().cpu() * 2.0
    checkpoint.load_state_dict_into(model, {"neck.point_fc.weight": w})
    assert not model._graphs
    after = model.forward_points(pts, point_outputs=True)[1]
    for a, b in zip(before, after):
        assert np.array_equal(a["xyz"], b["xyz"])
        assert np.allclose(b["cls"], 2.0 * a["cls"], rtol=1e-5, atol=1e-6)
    model.disable_cuda_graph()
