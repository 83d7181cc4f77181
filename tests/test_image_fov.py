"""Detection on unlabelled KITTI data: the image-FOV crop of raw-drive sweeps (csrc/frustum.cu sassd_image_fov_crop,
ops.image_fov_crop, the ``image_fov`` arguments of forward_points and detect_stream), the raw-drive calibration and
reader (results.Calibration.from_video, kitti_data.KittiDrive), the ``testing/`` split and the driver's unlabelled runs
(``--drive``, ``--split test``), against tests/golden/fov.npz, produced by the reference's own Calibration(from_video=
True) and get_lidar_in_image_fov (tests/golden/make_golden_fov.py).

Bar: calibration matrices equal; kept rows, their order and the frame offsets bit-identical; detections and KITTI rows
of a device-cropped sweep bit-identical to those of the same sweep cropped on the host by the reference's mask."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle.image_fov import in_image_fov, project
from sassd_b200 import kitti_data as K
from sassd_b200.results import Calibration
from sassd_b200.synth import synth_cloud
from tests.test_kitti_data import _header_only

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["Car"]


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "fov.npz"))


def _mask(bits, n):
    return np.unpackbits(bits)[:n].astype(bool)


_SWEEPS = {}


def _sweep(z, si):
    seed = int(z["sweep_seed"][si])
    if seed not in _SWEEPS:
        _SWEEPS[seed] = synth_cloud(seed, fov_deg=180.0)
    return _SWEEPS[seed]


def _kept(z, si, k):
    """The reference's kept mask of sweep si under crop set k."""
    return _mask(z["kept_s%d_k%d" % (si, k)], int(z["sweep_npts"][si]))


def _boundary_kept(z, k):
    return _mask(z["boundary_kept_k%d" % k], z["boundary_points"].shape[0])


def _write_calib(d, z, ci):
    os.makedirs(d, exist_ok=True)
    for name in ("cam_to_cam", "velo_to_cam"):
        with open(os.path.join(d, "calib_%s.txt" % name), "w") as fh:
            fh.write(str(z["calib%d_%s" % (ci, name)]))


def _calib(z, ci):
    return Calibration({"P2": z["calib%d_P2" % ci], "Tr_velo_to_cam": z["calib%d_Tr" % ci],
                        "R0_rect": z["calib%d_R0" % ci]})


def _set(z, k):
    """Crop set k: (calibration, image shape (h, w, 3))."""
    return _calib(z, int(z["set_calib"][k])), tuple(int(v) for v in z["set_shape"][k]) + (3,)


def write_drive(day_dir, stems, shapes, clouds, z, ci=0, name="2011_09_26_drive_0001_sync"):
    """A raw drive: the day's calibration files, IHDR-only PNGs and sweeps named by the %010d stems."""
    _write_calib(day_dir, z, ci)
    drive = os.path.join(day_dir, name)
    os.makedirs(os.path.join(drive, "image_02", "data"), exist_ok=True)
    os.makedirs(os.path.join(drive, "velodyne_points", "data"), exist_ok=True)
    for j, s in enumerate(stems):
        _header_only(os.path.join(drive, "image_02", "data", "%010d.png" % s), *shapes[j % len(shapes)])
        clouds[j % len(clouds)].astype(np.float32).tofile(os.path.join(drive, "velodyne_points", "data",
                                                                       "%010d.bin" % s))
    return drive


def write_testing(root, ids, shapes, calib_txts, clouds):
    """A KITTI ``testing/`` tree: ImageSets/test.txt, velodyne, calib, image_2 PNG headers; no labels."""
    os.makedirs(os.path.join(root, "ImageSets"), exist_ok=True)
    with open(os.path.join(root, "ImageSets", "test.txt"), "w") as fh:
        fh.write("".join("%06d\n" % i for i in ids))
    t = os.path.join(root, "testing")
    for sub in ("velodyne", "calib", "image_2"):
        os.makedirs(os.path.join(t, sub), exist_ok=True)
    for j, i in enumerate(ids):
        clouds[j % len(clouds)].astype(np.float32).tofile(os.path.join(t, "velodyne", "%06d.bin" % i))
        with open(os.path.join(t, "calib", "%06d.txt" % i), "w") as fh:
            fh.write(calib_txts[j % len(calib_txts)])
        _header_only(os.path.join(t, "image_2", "%06d.png" % i), *shapes[j % len(shapes)])


# ------------------------------------------------------------------ CPU
def test_calibration_from_video_matches_the_reference(gold, tmp_path):
    for ci in range(2):
        d = str(tmp_path / ("c%d" % ci))
        _write_calib(d, gold, ci)
        assert "calib_time" in str(gold["calib%d_cam_to_cam" % ci])          # the date lines are there, and skipped
        c = Calibration.from_video(d)
        assert np.array_equal(c.P2, gold["calib%d_P2" % ci])
        assert np.array_equal(c.V2C, gold["calib%d_Tr" % ci])
        assert np.array_equal(c.R0, gold["calib%d_R0" % ci])
    with pytest.raises(FileNotFoundError):
        Calibration.from_video(str(tmp_path))


def test_synthetic_sweeps_regenerate(gold):
    from tests.test_frustum_crop import _digest
    for si in range(len(gold["sweep_seed"])):
        pts = _sweep(gold, si)
        assert pts.shape[0] == int(gold["sweep_npts"][si])
        assert _digest(pts) == str(gold["sweep_sha"][si]), "synthetic cloud generator drifted"


def test_oracle_reproduces_every_stored_mask(gold):
    bnd = gold["boundary_points"]
    for k in range(len(gold["set_calib"])):
        c, shape = _set(gold, k)
        for si in range(len(gold["sweep_seed"])):
            assert np.array_equal(in_image_fov(_sweep(gold, si), c.P2, c.V2C, c.R0, shape), _kept(gold, si, k)), (si, k)
        assert np.array_equal(in_image_fov(bnd, c.P2, c.V2C, c.R0, shape), _boundary_kept(gold, k)), k


def test_boundary_cloud_covers_its_cases(gold):
    bnd, kind = gold["boundary_points"], gold["boundary_kind"]
    n_sets = len(gold["set_calib"])
    for k in range(n_sets):
        m = _boundary_kept(gold, k)
        edge = m[kind == 0].reshape(-1, 3)
        # every set's own edge triples straddle its edges: the point on one side, its neighbour on the other
        assert (edge.any(1) & ~edge.all(1)).sum() >= 4 * 40, k
        assert not m[kind == 4].any()                                    # non-finite points are dropped
        c, _ = _set(gold, k)
        _, rect, _ = project(bnd, c.P2, c.V2C, c.R0)
        near = kind == 2
        assert (m & near & (rect[:, 2] < 0)).any(), "no kept point behind the camera plane"
    # x = 0.1f itself is dropped (fp32 comparison), its upper neighbour can be kept
    x = bnd[:, 0]
    m0 = _boundary_kept(gold, 0)
    clip = kind == 1
    assert m0[clip].any() and np.all(x[clip & m0] == np.nextafter(np.float32(0.1), np.float32(1)))
    # rectified depth and uvw2 at zero, from both sides, for both calibrations
    for ci in range(2):
        c = _calib(gold, ci)
        _, rect, uvw = project(bnd[kind == 3], c.P2, c.V2C, c.R0)
        for a in (rect[:, 2], uvw[:, 2]):
            assert np.abs(a).min() < 1e-6 and (a < 0).any() and (a > 0).any()


def test_image_fov_crop_symbols_and_argument_validation():
    from sassd_b200 import lib as L
    lib = L.load()
    assert "sassd_image_fov_crop" in L.exported_symbols()
    a, b, c = ctypes.c_void_p(8), ctypes.c_void_p(16), ctypes.c_void_p(24)   # never dereferenced on these paths
    ws = 1 << 20
    f = lib.sassd_image_fov_crop
    assert f(None, a, 100, 1, a, 0.1, b, c, a, ws, None) == -1
    assert f(a, None, 100, 1, a, 0.1, b, c, a, ws, None) == -1
    assert f(a, a, 100, 1, None, 0.1, b, c, a, ws, None) == -1
    assert f(a, a, 100, 1, a, 0.1, None, c, a, ws, None) == -1
    assert f(a, a, 100, 1, a, 0.1, b, None, a, ws, None) == -1
    assert f(a, a, 100, 1, a, 0.1, b, c, None, ws, None) == -1
    assert f(a, a, 100, 0, a, 0.1, b, c, a, ws, None) == -1            # batch < 1
    assert f(a, a, 100, 257, a, 0.1, b, c, a, ws, None) == -1          # batch > 256
    assert f(a, a, -1, 1, a, 0.1, b, c, a, ws, None) == -1             # negative capacity
    assert f(a, a, 100, 1, a, 0.1, a, c, a, ws, None) == -1            # in place
    assert f(a, a, 1 << 20, 1, a, 0.1, b, c, a, 8, None) == -3         # workspace too small
    from sassd_b200 import ops
    assert ops._KERNELS["sassd_image_fov_crop"] == 1


def test_crop_kinds_exclude_each_other():
    from sassd_b200.detectors import CROP_FRUSTUM, CROP_IMAGE_FOV, CROP_NONE, _crop_kind
    assert _crop_kind(False, False, False) == CROP_NONE == False      # noqa: E712  (graph keys of earlier kinds)
    assert _crop_kind(True, False, True) == CROP_FRUSTUM == True      # noqa: E712
    assert _crop_kind(False, True, True) == CROP_IMAGE_FOV
    with pytest.raises(ValueError):
        _crop_kind(True, True, True)
    with pytest.raises(ValueError):
        _crop_kind(False, True, False)                                  # the crop reads the meta blocks


def test_drive_reader(gold, tmp_path):
    stems = [0, 1, 2, 5, 6]
    clouds = [np.full((k + 1, 4), k, np.float32) for k in range(3)]
    drive = write_drive(str(tmp_path / "2011_09_26"), stems, [(375, 1242), (370, 1224)], clouds, gold, ci=1)
    d = K.KittiDrive(drive)
    assert d.ids == stems and d.result_name == "%010d.txt" and not d.labelled
    assert np.array_equal(d.calib.P2, gold["calib1_P2"]) and np.array_equal(d.calib.V2C, gold["calib1_Tr"])
    pts, m = d.frame(5)
    assert np.array_equal(pts, clouds[0]) and m["sample_idx"] == 5 and m["img_shape"] == (370, 1224, 3)
    assert d.meta(2)["img_shape"] == (375, 1242, 3)
    got = list(K.Prefetcher(d, K.padded_batches(d.ids, 2), depth=2, workers=2))
    assert [b[0] for b in got] == [[0, 1], [2, 5], [6, None]]
    assert got[2][1][1].shape == (0, 4) and got[2][2][1]["sample_idx"] == -1
    assert got[2][2][1]["img_shape"] == (375, 1242, 3)
    # an explicit calibration directory
    _write_calib(str(tmp_path / "cal"), gold, 0)
    assert np.array_equal(K.KittiDrive(drive, str(tmp_path / "cal")).calib.P2, gold["calib0_P2"])


def test_drive_reader_refusals(gold, tmp_path):
    clouds = [np.zeros((3, 4), np.float32)]
    drive = write_drive(str(tmp_path / "day"), [0, 1, 2], [(375, 1242)], clouds, gold)
    os.remove(os.path.join(drive, "velodyne_points", "data", "0000000001.bin"))
    with pytest.raises(ValueError, match="differ"):
        K.KittiDrive(drive)                       # a sweep is missing: the sorted listings would pair frames wrongly
    clouds[0].tofile(os.path.join(drive, "velodyne_points", "data", "0000000007.bin"))
    with pytest.raises(ValueError, match="differ"):
        K.KittiDrive(drive)
    drive2 = write_drive(str(tmp_path / "day2"), [0, 1], [(375, 1242)], clouds, gold)
    _header_only(os.path.join(drive2, "image_02", "data", "12.png"), 375, 1242)
    with pytest.raises(ValueError, match="010d"):
        K.KittiDrive(drive2)
    drive3 = write_drive(str(tmp_path / "day3"), [0], [(375, 1242)], clouds, gold)
    os.remove(os.path.join(str(tmp_path / "day3"), "calib_velo_to_cam.txt"))
    with pytest.raises(FileNotFoundError, match="calib_velo_to_cam"):
        K.KittiDrive(drive3)


def test_test_split_reads_testing(golden_dir, tmp_path):
    g = np.load(os.path.join(golden_dir, "results.npz"))
    root = str(tmp_path / "kitti")
    write_testing(root, [7481, 7490], [(375, 1242), (370, 1224)], [str(g["calib_txt"])],
                  [np.ones((4, 4), np.float32), np.zeros((2, 4), np.float32)])
    s = K.KittiSplit(root, "test", "velodyne")
    assert s.dir == os.path.join(root, "testing") and not s.labelled and s.result_name == "%06d.txt"
    pts, m = s.frame(7490)
    assert pts.shape == (2, 4) and m["img_shape"] == (370, 1224, 3) and m["sample_idx"] == 7490
    with pytest.raises(ValueError, match="no labels"):
        s.gt_annos()


def test_driver_arguments_without_labels(tmp_path):
    from sassd_b200 import test as T
    cfg = os.path.join(ROOT, "configs", "car_cfg.py")
    for bad in (["--drive", "d"], ["--data-root", "r", "--split", "test"], ["--data-root", "r", "--calib-dir", "c"],
                ["--drive", "d", "--out", "o", "--lidar", "velodyne_reduced"], [],
                ["--drive", "d", "--data-root", "r", "--out", "o"]):
        with pytest.raises(SystemExit):
            T.parse_args([cfg, "w.pth"] + bad)
    a = T.parse_args([cfg, "w.pth", "--drive", "d", "--calib-dir", "c", "--out", "o"])
    assert a.drive == "d" and a.calib_dir == "c" and a.lidar == "velodyne" and a.max_points == 131072
    a = T.parse_args([cfg, "w.pth", "--data-root", "r", "--split", "test", "--out", "o"])
    assert a.split == "test" and a.lidar == "velodyne"


def test_driver_on_a_drive_runs_up_to_the_device(gold, tmp_path, monkeypatch):
    from sassd_b200 import lib
    from sassd_b200 import test as T
    drive = write_drive(str(tmp_path / "day"), [0, 1], [(375, 1242)], [np.ones((3, 4), np.float32)], gold)
    args = T.parse_args([os.path.join(ROOT, "configs", "car_cfg.py"), str(tmp_path / "none.pth"), "--drive", drive,
                         "--out", str(tmp_path / "out")])
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(lib.SassdError, match="CUDA device"):
        T.run(args)


# ------------------------------------------------------------------ GPU: the kernel
def _pool(z):
    """(cloud, set, kept mask) for every sweep x set and the boundary cloud under every set."""
    n_sets = len(z["set_calib"])
    pool = [(_sweep(z, si), k, _kept(z, si, k)) for si in range(len(z["sweep_seed"])) for k in range(n_sets)]
    pool += [(z["boundary_points"], k, _boundary_kept(z, k)) for k in range(n_sets)]
    return pool


def _run_fov(frames, sets, z, dev, cap_extra=0):
    from sassd_b200 import ops
    from sassd_b200.results import meta_block
    counts = [f.shape[0] for f in frames]
    off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
    pts = np.concatenate([f[:, :4] for f in frames] + [np.zeros((max(cap_extra, 1), 4), np.float32)], 0)
    meta = np.stack([meta_block(*_set(z, k)) for k in sets])
    out, off_out = ops.image_fov_crop(torch.from_numpy(pts).to(dev), torch.from_numpy(off).to(dev), len(frames),
                                      torch.from_numpy(meta).to(dev))
    torch.cuda.synchronize()
    return out.cpu().numpy(), off_out.cpu().numpy()


def _check_rows(frames, masks, out, off_out):
    exp_off = np.concatenate([[0], np.cumsum([int(m.sum()) for m in masks])])
    np.testing.assert_array_equal(off_out, exp_off)
    for b, (f, m) in enumerate(zip(frames, masks)):
        got = out[off_out[b]:off_out[b + 1]]
        assert np.array_equal(got.view(np.uint32), np.ascontiguousarray(f[m, :4]).view(np.uint32)), "frame %d" % b


@pytest.mark.gpu
def test_kernel_keeps_the_reference_rows_at_batch_1(gold):
    dev = torch.device("cuda:0")
    for f, k, m in _pool(gold):
        out, off_out = _run_fov([f], [k], gold, dev, cap_extra=2049)
        _check_rows([f], [m], out, off_out)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [2, 16])
def test_kernel_keeps_the_reference_rows_in_mixed_batches(gold, B):
    dev = torch.device("cuda:0")
    pool = _pool(gold)
    empty = (np.zeros((0, 4), np.float32), 1, np.zeros(0, bool))
    case = [pool[(7 * b + 2) % len(pool)] for b in range(B - 1)] + [empty]
    if B == 2:
        case = [pool[-1], empty]
    frames = [f for f, _, _ in case]
    out, off_out = _run_fov(frames, [k for _, k, _ in case], gold, dev, cap_extra=4099)
    _check_rows(frames, [m for _, _, m in case], out, off_out)


# ------------------------------------------------------------------ GPU: end to end
def _model():
    import sassd_b200 as S
    from sassd_b200 import checkpoint
    cfg = S.Config.fromfile(os.path.join(ROOT, "configs", "car_cfg.py"))
    model, _, _ = S.build_from_config(cfg, device="cuda:0")
    checkpoint.load_state_dict_into(model, checkpoint.make_synthetic_state_dict(0, 1))
    model.class_names = NAMES
    return model


def _same_annos(got, exp):
    n = 0
    for g, e in zip(got, exp):
        assert set(g) == set(e)
        for k in e:
            assert g[k].dtype == e[k].dtype and np.array_equal(g[k], e[k]), k
        n += len(e["name"])
    return n


def _e2e_batches(z):
    """Two batches of two sweeps, under crop sets of both calibrations: (sweeps, metas, host-cropped clouds)."""
    out = []
    for sis, ks in (((0, 1), (0, 3)), ((2, 0), (2, 1))):
        metas = [dict(calib=_set(z, k)[0], img_shape=_set(z, k)[1], sample_idx=10 * si + k) for si, k in zip(sis, ks)]
        out.append(([_sweep(z, si) for si in sis], metas, [_sweep(z, si)[_kept(z, si, k)] for si, k in zip(sis, ks)]))
    return out


@pytest.mark.gpu
def test_image_fov_step_detects_like_the_host_cropped_clouds_eager_captured_and_streamed(gold):
    model = _model()
    batches = _e2e_batches(gold)
    n = 0
    for full, metas, cropped in batches:
        got, aux = model.forward_points(full, metas=metas, image_fov=True, return_aux=True)
        exp, aux_e = model.forward_points(cropped, metas=metas, return_aux=True)
        n += _same_annos(got, exp)
        assert torch.equal(aux["ndet"], aux_e["ndet"])
        nd = aux["ndet"].cpu().numpy()
        for b in range(len(full)):
            assert torch.equal(aux["det"][b, :nd[b]], aux_e["det"][b, :nd[b]])
    assert n > 0, "no detection to compare"
    with pytest.raises(ValueError):
        model.forward_points(batches[0][0], image_fov=True)
    with pytest.raises(ValueError):
        model.forward_points(batches[0][0], metas=batches[0][1], image_fov=True, frustum_planes=[np.zeros((6, 4))] * 2)
    # captured: the image-FOV graph against the plain formatting graph fed the host-cropped clouds
    model.enable_cuda_graph(2, 131072)
    per_call = []
    for full, metas, cropped in batches:
        got = model.forward_points(full, metas=metas, image_fov=True)
        _same_annos(got, model.forward_points(cropped, metas=metas))
        per_call.append(got)
    assert {k for k in model._graphs if k[1]} == {(2, True, False), (0, True, False)}
    model.disable_cuda_graph()
    # detect_stream: image-FOV slots against the per-call results
    order = [0, 1, 1, 0, 1]
    got = list(model.detect_stream([(batches[i][0], batches[i][1]) for i in order], 2, 131072, depth=4, kitti=True,
                                   image_fov=True))
    assert len(got) == len(order)
    for i, g in zip(order, got):
        _same_annos(g, per_call[i])
    with pytest.raises(ValueError):
        list(model.detect_stream([], 2, 131072, image_fov=True))


def _files(d):
    return {f: open(os.path.join(d, f)).read() for f in sorted(os.listdir(d))}


@pytest.mark.gpu
def test_driver_on_a_synthetic_drive_and_testing_split(gold, golden_dir, tmp_path):
    from sassd_b200 import checkpoint
    from sassd_b200 import test as T
    from tests.test_kitti_format import _calib_txt
    ckpt = str(tmp_path / "synthetic.pth")
    checkpoint.save_checkpoint(checkpoint.make_synthetic_state_dict(0, 1), ckpt)
    cfg = os.path.join(ROOT, "configs", "car_cfg.py")
    model = _model()
    clouds = [synth_cloud(3000 + k, fov_deg=180.0) for k in range(5)]
    B = 4

    # a raw drive: 12 frames with a gap in the stems, two image sizes; whole batches, so that the per-call steps run the
    # driver's batches
    stems = [0, 1, 2, 3, 4, 5, 6, 8, 9, 10, 11, 12]
    drive = write_drive(str(tmp_path / "2011_09_26"), stems, [(375, 1242), (370, 1224)], clouds, gold, ci=1)
    src = K.KittiDrive(drive)
    frames = [src.frame(s) for s in stems]
    annos = []
    for s in range(0, len(frames), B):
        chunk = frames[s:s + B]
        annos += model.forward_points([p for p, _ in chunk], metas=[m for _, m in chunk], image_fov=True)
    want = str(tmp_path / "want_drive")
    T.write_results(want, stems, annos, "%010d.txt")
    out, js = str(tmp_path / "out_drive"), str(tmp_path / "drive.json")
    printed = []
    res = T.run(T.parse_args([cfg, ckpt, "--drive", drive, "--batch", str(B), "--out", out, "--json", js]),
                log=lambda *a, **k: printed.append(" ".join(a)))
    assert res["frames"] == len(stems) and "ap" not in res and len(printed) == 1 and "frames/s" in printed[0]
    assert sorted(os.listdir(out)) == ["%010d.txt" % s for s in stems]
    assert _files(out) == _files(want)
    assert sum(len(a["name"]) for a in annos) > 0, "no detection to compare"
    assert os.path.exists(js)

    # the testing split: full sweeps cropped to the camera frustum, as for val
    from sassd_b200.frustum import camera_frustum_planes
    root = str(tmp_path / "kitti")
    ids = [7481, 7482, 7490, 7500, 7517, 7518, 7519, 7600]
    calibs = [_calib(gold, 0), _calib(gold, 1)]
    write_testing(root, ids, [(375, 1242), (370, 1224)], [_calib_txt(c) for c in calibs], clouds)
    split = K.KittiSplit(root, "test", "velodyne")
    frames = [split.frame(i) for i in ids]
    annos = []
    for s in range(0, len(frames), B):
        chunk = frames[s:s + B]
        annos += model.forward_points([p for p, _ in chunk], metas=[m for _, m in chunk], frustum_planes=[
            camera_frustum_planes(m["calib"], m["img_shape"]) for _, m in chunk])
    want = str(tmp_path / "want_test")
    T.write_results(want, ids, annos)
    out = str(tmp_path / "out_test")
    res = T.run(T.parse_args([cfg, ckpt, "--data-root", root, "--split", "test", "--batch", str(B), "--out", out]),
                log=lambda *a, **k: None)
    assert res["frames"] == len(ids) and "ap" not in res
    assert _files(out) == _files(want)
