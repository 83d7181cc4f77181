"""Camera-frustum crop of full sweeps (csrc/frustum.cu, sassd_b200/frustum.py, the ``frustum_planes`` / ``crop``
arguments of forward_points and detect_stream) against tests/golden/frustum.npz, produced by the reference's own
remove_outside_points (tests/golden/make_golden_frustum.py).

Bar: the planes to 1e-12 relative; kept rows, their order and the frame offsets bit-identical; detections of a cropped
full sweep bit-identical to those of the reference's reduced cloud of it."""
import ctypes
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle.frustum import inside_frustum
from sassd_b200.synth import synth_cloud

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "frustum.npz"))


def _digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        a = np.ascontiguousarray(a)
        h.update(str(a.dtype).encode()); h.update(str(a.shape).encode()); h.update(a.tobytes())
    return h.hexdigest()


def _calib(z, ci):
    from sassd_b200.results import Calibration
    return Calibration({"P2": z["calib%d_P2" % ci], "Tr_velo_to_cam": z["calib%d_Tr" % ci],
                        "R0_rect": z["calib%d_R0" % ci]})


def _mask(bits, n):
    return np.unpackbits(bits)[:n].astype(bool)


_SWEEPS = {}


def _sweep(z, si):
    seed = int(z["sweep_seed"][si])
    if seed not in _SWEEPS:
        _SWEEPS[seed] = synth_cloud(seed, fov_deg=180.0)
    return _SWEEPS[seed]


def _kept(z, si, pi):
    """The reference's kept indices of sweep si under plane set pi."""
    return np.flatnonzero(_mask(z["kept_s%d_p%d" % (si, pi)], int(z["sweep_npts"][si])))


# ------------------------------------------------------------------ CPU
def test_camera_frustum_planes_match_the_reference(gold):
    from sassd_b200.frustum import camera_frustum_planes
    for pi in range(gold["planes"].shape[0]):
        p = camera_frustum_planes(_calib(gold, int(gold["planeset_calib"][pi])), tuple(gold["planeset_shape"][pi]))
        g = gold["planes"][pi]
        assert p.dtype == np.float64 and p.shape == (6, 4)
        # per face, relative to the face's largest coefficient (LAPACK builds may differ in the last bits)
        assert np.all(np.abs(p - g).max(axis=1) <= 1e-12 * np.abs(g).max(axis=1)), pi


def test_synthetic_full_sweeps_regenerate(gold):
    for si in range(len(gold["sweep_seed"])):
        pts = _sweep(gold, si)
        assert pts.shape[0] == int(gold["sweep_npts"][si])
        assert _digest(pts) == str(gold["sweep_sha"][si]), "synthetic cloud generator drifted"


def test_oracle_reproduces_the_reference_kept_indices(gold):
    n_sets = gold["planes"].shape[0]
    for pi in range(n_sets):
        planes = gold["planes"][pi]
        for si in range(len(gold["sweep_seed"])):
            assert np.array_equal(np.flatnonzero(inside_frustum(_sweep(gold, si), planes)), _kept(gold, si, pi))
        bnd = gold["boundary_points"]
        assert np.array_equal(inside_frustum(bnd, planes), _mask(gold["boundary_kept_p%d" % pi], bnd.shape[0]))
    # the boundary cloud really straddles the faces: some points of each triple are kept, some are not
    m = _mask(gold["boundary_kept_p0"], gold["boundary_points"].shape[0])
    assert 0.2 < m.mean() < 0.8


def test_crop_symbols_and_argument_validation():
    from sassd_b200 import lib as L
    lib = L.load()
    assert "sassd_frustum_crop" in L.exported_symbols() and "sassd_frustum_crop_workspace_bytes" in L.exported_symbols()
    assert lib.sassd_frustum_crop_workspace_bytes(0, 1) == 8
    assert lib.sassd_frustum_crop_workspace_bytes(2048, 1) == 8
    assert lib.sassd_frustum_crop_workspace_bytes(16 * 131072, 16) == 8 * 1024
    a, b, c = ctypes.c_void_p(8), ctypes.c_void_p(16), ctypes.c_void_p(24)   # never dereferenced on these paths
    ws = 1 << 20
    assert lib.sassd_frustum_crop(None, a, 100, 1, a, b, c, a, ws, None) == -1
    assert lib.sassd_frustum_crop(a, None, 100, 1, a, b, c, a, ws, None) == -1
    assert lib.sassd_frustum_crop(a, a, 100, 1, None, b, c, a, ws, None) == -1
    assert lib.sassd_frustum_crop(a, a, 100, 1, a, None, c, a, ws, None) == -1
    assert lib.sassd_frustum_crop(a, a, 100, 1, a, b, None, a, ws, None) == -1
    assert lib.sassd_frustum_crop(a, a, 100, 1, a, b, c, None, ws, None) == -1
    assert lib.sassd_frustum_crop(a, a, 100, 0, a, b, c, a, ws, None) == -1          # batch < 1
    assert lib.sassd_frustum_crop(a, a, 100, 257, a, b, c, a, ws, None) == -1        # batch > 256
    assert lib.sassd_frustum_crop(a, a, -1, 1, a, b, c, a, ws, None) == -1           # negative capacity
    assert lib.sassd_frustum_crop(a, a, 100, 1, a, a, c, a, ws, None) == -1          # in place
    assert lib.sassd_frustum_crop(a, a, 1 << 20, 1, a, b, c, a, 8, None) == -3       # workspace too small


def test_frame_planes_shape_is_checked():
    from sassd_b200.detectors import _frame_planes
    assert _frame_planes([np.zeros((6, 4))] * 2, 2).shape == (2, 6, 4)
    with pytest.raises(ValueError):
        _frame_planes([np.zeros((6, 4))], 2)
    with pytest.raises(ValueError):
        _frame_planes([np.zeros((4, 6))], 1)


# ------------------------------------------------------------------ GPU: the kernel
def _frames_case(z, B):
    """B frames with their plane sets and the reference's kept indices: full sweeps under every plane set, the boundary
    cloud, an empty frame and a frame entirely outside the frustum (the points behind the camera)."""
    n_sets = z["planes"].shape[0]
    pool = []
    for si in range(len(z["sweep_seed"])):
        for pi in range(n_sets):
            pool.append((_sweep(z, si), pi, _kept(z, si, pi)))
    bnd = z["boundary_points"]
    for pi in range(n_sets):
        pool.append((bnd, pi, np.flatnonzero(_mask(z["boundary_kept_p%d" % pi], bnd.shape[0]))))
    sw = _sweep(z, 0)
    behind = np.flatnonzero(sw[:, 0] < -1.0)
    assert not np.isin(behind, _kept(z, 0, 0)).any()
    pool.append((sw[behind], 0, np.zeros(0, np.int64)))
    pool.append((np.zeros((0, 4), np.float32), 1, np.zeros(0, np.int64)))
    if B == 1:
        return [pool[0]]
    if B == 2:
        return [pool[-3], pool[-2]]                 # boundary cloud + the frame outside the frustum
    return [pool[(5 * b + 3) % len(pool)] for b in range(B - 2)] + [pool[-1], pool[-2]]


def _run_crop(frames, planes, dev, cap_extra=0):
    from sassd_b200 import ops
    counts = [f.shape[0] for f in frames]
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    pts = np.concatenate([f[:, :4] for f in frames] + [np.zeros((max(cap_extra, 1), 4), np.float32)], 0)
    d_pts = torch.from_numpy(pts).to(dev)
    d_off = torch.from_numpy(off).to(dev)
    d_planes = torch.from_numpy(np.ascontiguousarray(planes, np.float64)).to(dev)
    out, off_out = ops.frustum_crop(d_pts, d_off, len(frames), d_planes)
    torch.cuda.synchronize()
    return out.cpu().numpy(), off_out.cpu().numpy()


def _check_rows(frames, kept, out, off_out):
    exp_off = np.concatenate([[0], np.cumsum([len(k) for k in kept])])
    np.testing.assert_array_equal(off_out, exp_off)
    for b, (f, k) in enumerate(zip(frames, kept)):
        got = out[off_out[b]:off_out[b + 1]]
        # bit patterns: the boundary cloud keeps its NaN rows
        assert np.array_equal(got.view(np.uint32), np.ascontiguousarray(f[k, :4]).view(np.uint32)), "frame %d" % b


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 2, 16])
def test_kernel_keeps_the_reference_rows_in_order(gold, B):
    dev = torch.device("cuda:0")
    case = _frames_case(gold, B)
    frames = [f for f, _, _ in case]
    planes = np.stack([gold["planes"][pi] for _, pi, _ in case])
    out, off_out = _run_crop(frames, planes, dev, cap_extra=4099)
    _check_rows(frames, [k for _, _, k in case], out, off_out)


@pytest.mark.gpu
def test_kernel_with_product_planes_equals_the_oracle(gold):
    from sassd_b200.frustum import camera_frustum_planes
    dev = torch.device("cuda:0")
    n_sets = gold["planes"].shape[0]
    planes = np.stack([camera_frustum_planes(_calib(gold, int(gold["planeset_calib"][pi])),
                                             tuple(gold["planeset_shape"][pi])) for pi in range(n_sets)])
    frames = [_sweep(gold, pi % 3) for pi in range(n_sets)] + [gold["boundary_points"]] * n_sets
    fplanes = np.concatenate([planes, planes])
    kept = [np.flatnonzero(inside_frustum(f, p)) for f, p in zip(frames, fplanes)]
    out, off_out = _run_crop(frames, fplanes, dev)
    _check_rows(frames, kept, out, off_out)


@pytest.mark.gpu
def test_captured_crop_replays_like_the_eager_launch(gold):
    from sassd_b200 import ops
    dev = torch.device("cuda:0")
    B, cap = 4, 4 * 131072
    pts = torch.zeros((cap, 4), dtype=torch.float32, device=dev)
    off = torch.zeros((B + 1,), dtype=torch.int32, device=dev)
    planes = torch.zeros((B, 6, 4), dtype=torch.float64, device=dev)
    ws = ops.Workspace()

    def load(si_list):
        frames = [_sweep(gold, si) for si in si_list]
        counts = [f.shape[0] for f in frames]
        pts.zero_()
        pts[:sum(counts)].copy_(torch.from_numpy(np.concatenate(frames, 0)))
        off.copy_(torch.from_numpy(np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)))
        planes.copy_(torch.from_numpy(np.stack([gold["planes"][(si + 1) % 4] for si in si_list])))

    load([0, 1, 2, 0])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.frustum_crop(pts, off, B, planes, ws=ws)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        g_out, g_off = ops.frustum_crop(pts, off, B, planes, ws=ws)
    for si_list in ([2, 0, 1, 1], [0, 1, 2, 0]):
        load(si_list)
        g.replay()
        e_out, e_off = ops.frustum_crop(pts, off, B, planes)
        torch.cuda.synchronize()
        assert torch.equal(g_off, e_off)
        n = int(e_off[-1])
        assert n == sum(len(_kept(gold, si, (si + 1) % 4)) for si in si_list)
        assert torch.equal(g_out[:n], e_out[:n])


# ------------------------------------------------------------------ GPU: end to end
def _model(prec):
    import sassd_b200 as S
    from sassd_b200 import checkpoint, ops
    cfg = S.Config.fromfile(os.path.join(ROOT, "configs", "car_cfg.py"))
    model, _, _ = S.build_from_config(cfg, device="cuda:0")
    checkpoint.load_state_dict_into(model, checkpoint.make_synthetic_state_dict(0, 1))
    if prec != ops.PREC_F16X3:
        model.set_precision(prec)
    return model


def _e2e_batches(z):
    """Two batches of two full sweeps each, under plane sets of both calibrations, and the reference's reduced clouds."""
    full, planes, reduced = [], [], []
    for sis, pis in (((0, 1), (0, 2)), ((2, 0), (3, 1))):
        full.append([_sweep(z, si) for si in sis])
        planes.append(np.stack([z["planes"][pi] for pi in pis]))
        reduced.append([_sweep(z, si)[_kept(z, si, pi)] for si, pi in zip(sis, pis)])
    return full, planes, reduced


def _same(got, exp):
    n = 0
    for g, e in zip(got, exp):
        assert (g["boxes_lidar"] is None) == (e["boxes_lidar"] is None)
        if e["boxes_lidar"] is not None:
            n += len(e["boxes_lidar"])
            np.testing.assert_array_equal(g["boxes_lidar"], e["boxes_lidar"])
            np.testing.assert_array_equal(g["scores"], e["scores"])
            np.testing.assert_array_equal(g["label_preds"], e["label_preds"])
    return n


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["f16x3", "fp32"])
def test_cropped_full_sweeps_detect_like_the_reduced_clouds_eager_captured_and_streamed(gold, prec):
    from sassd_b200 import ops
    model = _model(ops.PREC_F16X3 if prec == "f16x3" else ops.PREC_FP32)
    full, planes, reduced = _e2e_batches(gold)
    dets = 0
    # eager
    for f, p, r in zip(full, planes, reduced):
        dets += _same(model.forward_points(f, frustum_planes=list(p)), model.forward_points(r))
    assert dets > 0, "no detection to compare"
    # captured: the crop graph against the plain graph fed the reduced clouds
    model.enable_cuda_graph(2, 131072)
    for f, p, r in zip(full, planes, reduced):
        _same(model.forward_points(f, frustum_planes=p), model.forward_points(r))
    assert set(model._graphs) == {(False, False, False), (True, False, False)}
    model.disable_cuda_graph()
    # detect_stream: crop slots against plain slots fed the reduced clouds
    order = [0, 1, 1, 0, 1]
    got = list(model.detect_stream([(full[i], planes[i]) for i in order], 2, 131072, depth=4, crop=True))
    exp = list(model.detect_stream([reduced[i] for i in order], 2, 131072, depth=4))
    assert len(got) == len(exp) == len(order)
    for g, e in zip(got, exp):
        _same(g, e)
