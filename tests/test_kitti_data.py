"""Host side of KITTI split evaluation (sassd_b200.kitti_data, sassd_b200.test, the row-width result gather): the
label reader against the reference's own (tests/golden/labels.npz, tests/golden/make_golden_labels.py), PNG header
shapes, split files, batch padding, the plane cache, the world-size-2 gather of KITTI rows over gloo and a run of the
driver up to its first device call."""
import os
import struct
import sys
import zlib

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from sassd_b200 import kitti_data as K
from sassd_b200.results import Calibration, annos_from_rows, empty_result_anno, meta_block, rows_from_annos

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["Car", "Pedestrian", "Cyclist"]


def write_png(path, h, w, colour=2):
    """A valid PNG of h x w black pixels, written with zlib and struct only."""
    def chunk(kind, data):
        return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xffffffff)
    ch = {0: 1, 2: 3, 6: 4}[colour]
    raw = b"".join(b"\x00" + bytes(w * ch) for _ in range(h))
    with open(path, "wb") as fh:
        fh.write(K.PNG_SIGNATURE + chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, 8, colour, 0, 0, 0))
                 + chunk(b"IDAT", zlib.compress(raw)) + chunk(b"IEND", b""))


# ------------------------------------------------------------------ labels
def test_label_reader_matches_the_reference(tmp_path, golden_dir):
    z = np.load(os.path.join(golden_dir, "labels.npz"))
    ids = [int(i) for i in z["ids"]]
    for i in ids:
        (tmp_path / ("%06d.txt" % i)).write_text(str(z["text_%d" % i]))
    annos = K.read_labels(str(tmp_path), ids)
    assert len(annos) == len(ids)
    for i, anno in zip(ids, annos):
        want = {k[len("anno_%d_" % i):]: z[k] for k in z.files if k.startswith("anno_%d_" % i)}
        assert set(anno) == set(want), (i, set(anno) ^ set(want))
        for k, w in want.items():
            got = anno[k]
            assert got.dtype == w.dtype and got.shape == w.shape, (i, k, got.dtype, w.dtype, got.shape, w.shape)
            assert np.array_equal(got, w), (i, k)
    # the fixture covers what it claims: DontCare, Van, an empty file, scored lines
    names = np.concatenate([a["name"] for a in annos if a["name"].size])
    assert {"DontCare", "Van"} <= set(names.tolist())
    assert any(a["name"].size == 0 for a in annos)
    assert any(a["score"].size and a["score"].any() for a in annos)


# ------------------------------------------------------------------ files
@pytest.mark.parametrize("hw", [(375, 1242), (370, 1224), (376, 1241), (1, 1), (2, 70000)])
def test_png_shape_from_ihdr(tmp_path, hw):
    p = str(tmp_path / "a.png")
    write_png(p, *hw) if hw[1] < 10000 else _header_only(p, *hw)
    assert K.png_shape(p) == (hw[0], hw[1], 3)


def _header_only(path, h, w):
    ihdr = struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0)
    with open(path, "wb") as fh:
        fh.write(K.PNG_SIGNATURE + struct.pack(">I", 13) + b"IHDR" + ihdr + struct.pack(">I", zlib.crc32(b"IHDR" + ihdr)))


def test_png_channels_and_refusals(tmp_path):
    p = str(tmp_path / "g.png")
    write_png(p, 4, 5, colour=0)
    assert K.png_shape(p) == (4, 5, 1)
    write_png(p, 4, 5, colour=6)
    assert K.png_shape(p) == (4, 5, 4)
    good = open(p, "rb").read()
    bad = {"truncated": good[:20], "signature": b"\x89PNX" + good[4:], "jpeg": b"\xff\xd8\xff\xe0" + good[4:],
           "empty": b"", "not IHDR": good[:12] + b"IDAT" + good[16:],
           "zero width": good[:16] + struct.pack(">I", 0) + good[20:]}
    for what, data in bad.items():
        q = tmp_path / "bad.png"
        q.write_bytes(data)
        with pytest.raises(ValueError):
            K.png_shape(str(q))
        assert what


def test_point_files_of_bad_size_are_refused(tmp_path):
    pts = np.arange(40, dtype=np.float32).reshape(10, 4)
    p = tmp_path / "000001.bin"
    pts.tofile(p)
    assert np.array_equal(K.read_points(str(p)), pts)
    for n in (4, 15, 17, 163):
        p.write_bytes(pts.tobytes()[:n] if n <= 160 else pts.tobytes() + b"\0\0\0")
        with pytest.raises(ValueError):
            K.read_points(str(p))
    p.write_bytes(b"")
    assert K.read_points(str(p)).shape == (0, 4)


def test_split_file_and_padding(tmp_path):
    (tmp_path / "ImageSets").mkdir()
    (tmp_path / "ImageSets" / "val.txt").write_text("000001\n000004\n000007\n\n000010\n")
    assert K.read_split(str(tmp_path), "val") == [1, 4, 7, 10]
    assert K.padded_batches([1, 4, 7, 10], 3) == [[1, 4, 7], [10, None, None]]
    assert K.padded_batches([1, 4, 7], 3) == [[1, 4, 7]]
    assert K.padded_batches(list(range(37)), 16)[-1] == [32, 33, 34, 35, 36] + [None] * 11
    from sassd_b200.test import rank_batches
    ids = list(range(37))
    for world in (1, 2, 3):
        per = [rank_batches(ids, r, world, 4) for r in range(world)]
        assert len({len(b) for b in per}) == 1                         # one block size on every rank
        got = sorted(i for b in per for ids_ in b for i in ids_ if i is not None)
        assert got == ids
        for r in range(world):
            assert [i for ids_ in per[r] for i in ids_ if i is not None] == ids[r::world]


def _calib(golden_dir, ci=0):
    z = np.load(os.path.join(golden_dir, "frustum.npz"))
    return Calibration({"P2": z["calib%d_P2" % ci], "Tr_velo_to_cam": z["calib%d_Tr" % ci],
                        "R0_rect": z["calib%d_R0" % ci]})


def test_plane_cache(golden_dir):
    from sassd_b200.frustum import camera_frustum_planes
    cache = K.PlaneCache()
    c0, c1 = _calib(golden_dir, 0), _calib(golden_dir, 1)
    p = cache(c0, (375, 1242, 3))
    assert np.array_equal(p, camera_frustum_planes(c0, (375, 1242)))
    assert cache(Calibration({"P2": c0.P2, "Tr_velo_to_cam": c0.V2C, "R0_rect": c0.R0}), (375, 1242)) is p
    assert len(cache) == 1
    assert not np.array_equal(cache(c0, (370, 1224)), p)
    assert not np.array_equal(cache(c1, (375, 1242)), p)
    assert len(cache) == 3


def test_meta_block_layout(golden_dir):
    c = _calib(golden_dir)
    m = meta_block(c, (370, 1224, 3))
    assert m.dtype == np.float64 and m.shape == (36,)
    assert np.array_equal(m[:12], c.P2.ravel()) and np.array_equal(m[12:24], c.V2C.ravel())
    assert np.array_equal(m[24:33], c.R0.ravel()) and tuple(m[33:]) == (370.0, 1224.0, 0.0)


def test_rows_and_annos_round_trip():
    rng = np.random.default_rng(3)
    rows = rng.normal(size=(3, 8, 14))
    rows[..., 13] = rng.integers(0, 3, (3, 8))
    n_out = np.array([2, 0, 8], np.int32)
    annos = annos_from_rows(rows, n_out, NAMES, [5, 6, 7])
    assert set(annos[1]) == set(empty_result_anno()) and annos[1]["bbox"].shape == (0, 4)
    a = annos[0]
    for k, dt in (("alpha", np.float32), ("dimensions", np.float32), ("location", np.float32),
                  ("rotation_y", np.float32), ("score", np.float32), ("bbox", np.float64), ("occluded", np.int64),
                  ("image_idx", np.int64), ("truncated", np.float64)):
        assert a[k].dtype == dt, k
    assert a["name"].dtype.kind == "U" and list(a["image_idx"]) == [5, 5]
    back, n_back = rows_from_annos(annos, NAMES, 8)
    assert np.array_equal(n_back, n_out)
    again = annos_from_rows(back, n_back, NAMES, [5, 6, 7])
    for x, y in zip(annos, again):
        for k in x:
            assert x[k].dtype == y[k].dtype and np.array_equal(x[k], y[k]), k


# ------------------------------------------------------------------ multi-rank gather of KITTI rows
def _worker(rank, world, port, q):
    sys.path.insert(0, ROOT)
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    from sassd_b200 import dist as D
    from sassd_b200.results import annos_from_rows, rows_from_annos
    from sassd_b200.test import rank_batches
    D.init_from_env(backend="gloo")
    ids = list(range(100, 111))             # 11 frames, 6 local frames per rank after padding at batch 3
    local = [i for b in rank_batches(ids, rank, world, 3) for i in b]
    rows = np.zeros((len(local), 4, 14))
    n = np.zeros(len(local), np.int32)
    for j, i in enumerate(local):
        if i is not None:
            n[j] = i % 4
            rows[j, :, :13] = i + np.arange(13) / 16.0
            rows[j, :, 13] = i % 3
    annos = annos_from_rows(rows, n, NAMES, [-1 if i is None else i for i in local])
    from sassd_b200.test import gather_annos
    got = gather_annos(annos, ids, NAMES, 4, torch.device("cpu"))
    q.put((rank, [(int(a["image_idx"][0]) if len(a["name"]) else None, len(a["name"]),
                   float(a["bbox"][0, 0]) if len(a["name"]) else None) for a in got]))
    dist.destroy_process_group()


def test_kitti_rows_gather_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want = [(i if i % 4 else None, i % 4, (i + 1 / 16.0) if i % 4 else None) for i in range(100, 111)]
    for _, got in res:
        assert got == want                  # split order restored on every rank, padding dropped


def test_gather_width_default_is_the_detection_row():
    from sassd_b200 import dist as D
    g = D.DetectionGather(2, 3, torch.device("cpu"))
    assert g.width == 9 and g.row == 2 * 3 * 9 + 2
    a, b = g(torch.arange(54, dtype=torch.float32).reshape(2, 3, 9), torch.tensor([1, 2], dtype=torch.int32))
    assert a.shape == (1, 2, 3, 9) and b.tolist() == [[1, 2]]


# ------------------------------------------------------------------ driver, up to the first device call
def write_split(root, ids, shapes, calib_txts, points):
    """A minimal KITTI tree: split file, velodyne(_reduced), calib, image_2 PNG headers."""
    os.makedirs(os.path.join(root, "ImageSets"), exist_ok=True)
    with open(os.path.join(root, "ImageSets", "val.txt"), "w") as fh:
        fh.write("".join("%06d\n" % i for i in ids))
    for sub in ("velodyne", "velodyne_reduced", "calib", "image_2", "label_2"):
        os.makedirs(os.path.join(root, "training", sub), exist_ok=True)
    for j, i in enumerate(ids):
        t = os.path.join(root, "training")
        points[j].astype(np.float32).tofile(os.path.join(t, "velodyne", "%06d.bin" % i))
        points[j].astype(np.float32).tofile(os.path.join(t, "velodyne_reduced", "%06d.bin" % i))
        with open(os.path.join(t, "calib", "%06d.txt" % i), "w") as fh:
            fh.write(calib_txts[j % len(calib_txts)])
        _header_only(os.path.join(t, "image_2", "%06d.png" % i), *shapes[j % len(shapes)])


@pytest.mark.parametrize("n_frames, world, batch", [(17, 2, 8), (33, 2, 16), (2, 4, 4)])
def test_prefetcher_pads_batches_without_a_real_frame(tmp_path, golden_dir, n_frames, world, batch):
    """Under torchrun a rank's last batch - or, with fewer frames than ranks, every batch - can be all padding."""
    from sassd_b200.test import rank_batches
    g = np.load(os.path.join(golden_dir, "results.npz"))
    ids = [10 + 3 * k for k in range(n_frames)]
    write_split(str(tmp_path), ids, [(370, 1224), (375, 1242)], [str(g["calib_txt"])],
                [np.full((k % 3, 4), k, np.float32) for k in range(n_frames)])
    split = K.KittiSplit(str(tmp_path), "val", "velodyne")
    per_rank = [rank_batches(ids, rank, world, batch) for rank in range(world)]
    assert any(all(i is None for i in b) for batches in per_rank for b in batches), "case without an all-padding batch"
    seen = []
    for batches in per_rank:
        got = list(K.Prefetcher(split, batches, depth=2, workers=2))
        assert [b[0] for b in got] == batches
        for b_ids, points, metas in got:
            assert len(points) == len(metas) == batch
            for i, p, m in zip(b_ids, points, metas):
                if i is None:       # padding: no points, the split's first frame's calibration and image size
                    assert p.shape == (0, 4) and m["sample_idx"] == -1 and m["img_shape"] == (370, 1224, 3)
                    assert np.array_equal(m["calib"].P2, split.meta(ids[0])["calib"].P2)
                else:
                    seen.append(i)
                    assert m["sample_idx"] == i and p.shape[0] == ids.index(i) % 3
    assert sorted(seen) == ids
    # the padding meta gives the device formatter a valid block
    assert meta_block(split.pad_frame()[1]["calib"], split.pad_frame()[1]["img_shape"])[33] == 370.0


def test_driver_runs_up_to_the_device(tmp_path, golden_dir, monkeypatch):
    from sassd_b200 import lib
    from sassd_b200 import test as T
    g = np.load(os.path.join(golden_dir, "results.npz"))
    ids = [3, 8, 21]
    write_split(str(tmp_path), ids, [(375, 1242), (370, 1224)], [str(g["calib_txt"])],
                [np.ones((5, 4)) * k for k in range(3)])
    split = K.KittiSplit(str(tmp_path), "val", "velodyne")
    reader = K.Prefetcher(split, K.padded_batches(split.ids, 2), depth=1, workers=2)
    got = list(reader)
    assert [b[0] for b in got] == [[3, 8], [21, None]]
    assert [m["sample_idx"] for m in got[1][2]] == [21, -1] and got[1][1][1].shape == (0, 4)
    assert [m["img_shape"] for m in got[0][2]] == [(375, 1242, 3), (370, 1224, 3)]
    assert np.array_equal(got[0][1][1], np.ones((5, 4), np.float32))
    args = T.parse_args([os.path.join(ROOT, "configs", "car_cfg.py"), str(tmp_path / "none.pth"),
                         "--data-root", str(tmp_path), "--batch", "2", "--lidar", "velodyne_reduced"])
    assert args.max_points == 32768 and args.split == "val"
    monkeypatch.setattr(torch.cuda, "is_available", lambda: False)
    with pytest.raises(lib.SassdError, match="CUDA device"):
        T.run(args)
