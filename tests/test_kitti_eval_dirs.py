"""Evaluating KITTI result directories: the device parser of label / result files (csrc/kitti_parse.cu,
kitti_eval.read_block), the flat annotation form (kitti_eval.AnnoBlock), kitti_eval.eval_dirs and the command line
``python -m sassd_b200.kitti_eval``.

* CPU: the command's argument errors, FileNotFoundError for a missing frame, AnnoBlock.from_annos against the
  flattening of annotation dicts, eval_many on blocks against it on dicts through the host path.
* GPU: every column of read_block equals AnnoBlock.from_annos(read_labels(...)) bit for bit on result files of
  write_results, GT files, fuzzed numbers, empty files, score-column quirks, files the device defers to the host (which
  raise what read_labels raises or give its values) and files of many lines; eval_dirs and the command against
  eval_many on read_labels.
"""
import os

import numpy as np
import pytest

from oracle import kitti_eval as O
from sassd_b200 import kitti_eval as K
from sassd_b200 import kitti_data as KD
from tests.test_kitti_eval import GOLD, _annos
from tests.test_kitti_eval_coco import _perturbed_sets, _same_tables

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ["Car", "Van", "Pedestrian", "Cyclist", "Truck", "DontCare", "Person_sitting", "Misc", "Tram"]


# ------------------------------------------------------------------------------------------------------ fixtures
def _number(rng, fast=False):
    """A number as some writer formats it: %.0f .. %.6f, %e, repr, 15-19 significant digits, values at and past
    2^53, 1e22 / 1e23, signed zeros, a sign, a bare point on either side.  ``fast``: only forms the device parses
    itself (no repr, no more than 15 significant digits, no significand past 2^53 or exponent past 22)."""
    x = float(rng.normal(0, 1) * 10.0 ** int(rng.integers(-4, 7)))
    kind = int(rng.choice([0, 1, 2, 3, 4, 5, 6, 7, 11, 12, 13])) if fast else int(rng.integers(0, 14))
    if kind <= 6:
        return "%.*f" % (kind, x)
    if kind == 7:
        return "%e" % x
    if kind == 8:
        return repr(x)
    if kind == 9:
        return "%.*g" % (int(rng.integers(15, 20)), x)
    if kind == 10:
        return str(rng.choice(["9007199254740991", "9007199254740992", "9007199254740993", "-9007199254740993",
                               "1e22", "1e23", "-1e22", "1e-22", "1e-23", "4.5e15", "0.0000000000000000000001"]))
    if kind == 11:
        return str(rng.choice(["-0.00", "-0", "+0.0", "+1", "-1", ".5", "5.", "-.5", "+5.", "0.0", "00012.50",
                               "1E5", "1e+05", "2.5e-3", "9007199254740991", "1e22", "-1e-22", "4.5e15"]))
    if kind == 12:
        return "%d" % int(rng.integers(-3, 4))
    return "%.2f" % x


def _line(rng, fields=15, name=None, fast=False):
    name = NAMES[int(rng.integers(0, len(NAMES)))] if name is None else name
    nums = [_number(rng, fast) for _ in range(fields - 1)]
    if fast and abs(float(nums[1])) >= 2.0 ** 63:       # an occluded value past int64 goes to the host
        nums[1] = "3"
    return " ".join([name] + nums)


def fuzz_files(rng, fast=False):
    """{file id: bytes}: fuzzed numbers in lines of 15, 16 and 17 fields, empty files, the score-column quirks, a file
    of 1000 lines and upper-case names."""
    files = {0: b"", 1: _line(rng, fast=fast).encode(), 2: (_line(rng, fast=fast) + "\n").encode()}
    for i in range(3, 40):
        first = int(rng.choice([15, 16, 17]))
        lines = [_line(rng, first, fast=fast)] + [
            _line(rng, int(rng.choice([first, 16, 17]) if first != 15 else rng.choice([15, 16, 17])), fast=fast)
            for _ in range(int(rng.integers(0, 8)))]
        if first == 16:     # a scored file converts every line's 16th field
            lines = [lines[0]] + [l if len(l.split(" ")) >= 16 else l + " 0.5" for l in lines[1:]]
        text = "\n".join(lines) + ("\n" if i % 3 else "")      # some files end without a newline
        files[i] = text.encode()
    files[40] = ("\n".join(_line(rng, 16, fast=True) for _ in range(1000)) + "\n").encode()   # rows of many CTAs
    files[41] = ("CAR 0 0 0 1 2 3 4 1.5 1.6 3.9 1 2 3 0.1\nPEDESTRIAN 0 0 0 1 2 3 4 1 1 1 1 2 3 0.1\n"
                 "cyclist 0 0 0 1 2 3 4 1 1 1 1 2 3 0.1\nDONTCARE -1 -1 -10 1 2 3 4 -1 -1 -1 -1000 -1000 -1000 -10\n"
                 "dontcare -1 -1 -10 1 2 3 4 -1 -1 -1 -1000 -1000 -1000 -10\n").encode()
    return files


def deferred_files(rng):
    """{file id: bytes} the device hands to the host reader: each raises what read_label raises or gives its values."""
    good = _line(rng, 16)
    plain = _line(rng, 15)
    return {
        100: (good + "\r\n" + good + "\r\n").encode(),                      # CRLF
        101: (good.replace(" ", "\t", 1) + "\n").encode(),                   # a tab
        102: (plain.replace(plain.split(" ")[3], "1_000.5") + "\n").encode(),   # an underscore
        103: ("Car 0 0 nan 1 2 3 4 1 1 1 1 2 3 0.1\n").encode(),
        104: ("Car 0 0 -inf 1 2 3 4 1 1 1 1 2 3 0.1\n").encode(),
        105: ("Car 0 inf 0 1 2 3 4 1 1 1 1 2 3 0.1\n").encode(),             # int(inf): OverflowError
        106: ("Car 0 nan 0 1 2 3 4 1 1 1 1 2 3 0.1\n").encode(),             # int(nan): ValueError
        107: ("Car 0 0  0 1 2 3 4 1 1 1 1 2 3 0.1\n").encode(),              # a double space inside the fields
        108: ("Car 0 0 0 1 2 3 4 1 1 1 1 2 3 0.1 0.7  x\n" + plain + " 0.2\n").encode(),   # one after them: 18 fields
        109: ("Car 0 0 0 1 2 3 4 1 1 1 1 2 3 0.1 0.7 \n").encode(),          # a trailing space: stripped
        110: ("  Car 0 0 0 1 2 3 4 1 1 1 1 2 3 0.1 0.7\n").encode(),         # leading spaces: stripped
        111: (good + "\n\n" + good + "\n").encode(),                         # an empty line: IndexError
        112: ("Café 0 0 0 1 2 3 4 1 1 1 1 2 3 0.1\n").encode("utf-8"),       # a non-ASCII name
        113: b"Car 0 0 0 1 2 3 4 1 1 1 1 2 3 0.1\xff\n",                      # not UTF-8: UnicodeDecodeError
        114: ("Car 0 0 0 1 2 3 4 1 1 1 1 2\n").encode(),                     # a missing field: IndexError
        115: ("Car 0 0 0 1 2 3 x4 1 1 1 1 2 3 0.1\n").encode(),              # not a number: ValueError
        116: ("Car 0 0 0 1 2 3 4 1 1 1 1 2 3 0.1 0.5\n" + plain + "\n").encode(),   # a scored file's short line
        117: ("Car 0 0 0 1.00000000000000000001 2 3 4 1 1 1 1 2 3 0.1\n").encode(),  # 21 significant digits
        118: ("Car 0 0 0 1e400 2 3 4 1 1 1 1 2 3 0.1\n").encode(),           # an exponent past the fast path
        119: ("Car 0 1e30 0 1 2 3 4 1 1 1 1 2 3 0.1\n").encode(),            # occluded beyond int64
        120: ("Car 0 0 0 1 2 3 4 1 1 1 1 2 3 0.1\r").encode(),               # a lone CR ends the line
        121: ("Car 0 0 0 1 2 3 4 1 1 1 1 2 3 0.1 \x0b\n").encode(),          # a control character strip() removes
        122: ("Car 0 0 0 -1e-400 2 3 4 1 1 1 1 2 3 0.1\n").encode(),
    }


def write_files(d, files):
    os.makedirs(d, exist_ok=True)
    for i, data in files.items():
        with open(os.path.join(d, "%06d.txt" % i), "wb") as fh:
            fh.write(data)
    return sorted(files)


def _host_block(d, ids):
    return K.AnnoBlock.from_annos(KD.read_labels(d, ids), "cpu")


def _same_block(got, want):
    np.testing.assert_array_equal(got.off, want.off)
    assert got.trunc_dtype == want.trunc_dtype
    for k in K.AnnoBlock.COLUMNS:
        a, b = getattr(got, k).cpu().numpy(), getattr(want, k).cpu().numpy()
        assert a.dtype == b.dtype and a.shape == b.shape, (k, a.dtype, b.dtype, a.shape, b.shape)
        assert a.tobytes() == b.tobytes(), (k, np.flatnonzero((a != b).reshape(len(a), -1).any(1))[:5])


def _gt_files(rng, ids):
    from tests.kitti_root import _rig, label_lines
    return {i: "".join(l + "\n" for l in label_lines(i % 8, _rig(i % 2), rng)).encode() for i in ids}


def _write_sets(tmp, gts, sets, ids):
    """GT and result directories of annotation dicts: the GT as label files, each set by test.write_results."""
    from sassd_b200 import test as T
    from sassd_b200.results import annos_to_kitti_label
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
    return gt_dir, dirs


# ------------------------------------------------------------------------------------------------------------ CPU
@pytest.mark.parametrize("argv, message", [
    (["--data-root", "{root}"], "--results"),
    (["--data-root", "{root}", "--results", "{root}", "--classes", "Car", "Bus"], "unknown class Bus"),
    (["--data-root", "{root}", "--split", "nosuch", "--results", "{root}"], "nosuch.txt does not exist"),
    (["--data-root", "{root}", "--results", "{root}/missing"], "is not a directory"),
])
def test_command_argument_errors(tmp_path, capsys, argv, message):
    root = str(tmp_path)
    os.makedirs(os.path.join(root, "ImageSets"))
    os.makedirs(os.path.join(root, "training", "label_2"))
    open(os.path.join(root, "ImageSets", "val.txt"), "w").close()
    with pytest.raises(SystemExit) as e:
        K.parse_args([a.format(root=root) for a in argv])
    assert e.value.code == 2
    assert message in capsys.readouterr().err


def test_missing_frame_raises_file_not_found(tmp_path):
    write_files(str(tmp_path), {0: b"", 2: b""})
    with pytest.raises(FileNotFoundError, match="000001.txt"):
        K.read_block(str(tmp_path), [0, 1, 2])


def test_from_annos_gives_the_flattened_arrays():
    gts, dts = _annos(np.load(GOLD))
    for annos in (gts, dts):
        b = K.AnnoBlock.from_annos(annos, "cpu")
        names, dc = K._flat_names(annos)
        np.testing.assert_array_equal(b.off, np.concatenate([[0], np.cumsum([len(a["name"]) for a in annos])]))
        np.testing.assert_array_equal(b.name_id.numpy(), names)
        np.testing.assert_array_equal(b.dontcare.numpy(), dc)
        np.testing.assert_array_equal(b.bbox.numpy(), K._flat(annos, "bbox", 4))
        np.testing.assert_array_equal(b.cam.numpy(), K._flat_cam(annos))
        for k in ("occluded", "alpha"):
            np.testing.assert_array_equal(b.__dict__[k].numpy(), K._flat(annos, k, 1).reshape(-1))
        np.testing.assert_array_equal(b.truncated.numpy(), np.concatenate([a["truncated"] for a in annos]))
        assert b.trunc_dtype == np.concatenate([a["truncated"] for a in annos]).dtype
    np.testing.assert_array_equal(K.AnnoBlock.from_annos(dts, "cpu").score.numpy(), K._flat(dts, "score", 1).ravel())
    assert not K.AnnoBlock.from_annos(gts, "cpu").score.numpy().any()
    f32 = [dict(a, truncated=np.asarray(a["truncated"], np.float32)) for a in gts]
    assert K.AnnoBlock.from_annos(f32, "cpu").trunc_dtype == np.float32
    assert K._aos_flag(K.AnnoBlock.from_annos(dts, "cpu")) == K._aos_flag(dts)
    empty = K.AnnoBlock.from_annos([dict(gts[0], **{k: np.asarray(v)[:0] for k, v in gts[0].items()})], "cpu")
    assert empty.off.tolist() == [0, 0] and empty.bbox.shape == (0, 4) and not K._aos_flag(empty)


def test_eval_many_on_blocks_equals_it_on_dicts_on_the_host_path():
    gts, dts = _annos(np.load(GOLD))
    sets = _perturbed_sets(dts, 2)
    want = K.eval_many(gts, sets, [0, 1, 2], (11, 40, "coco"), overlap_fn=O.rotate_iou_eval)
    blocks = [K.AnnoBlock.from_annos(s, "cpu") for s in sets]
    got = K.eval_many(K.AnnoBlock.from_annos(gts, "cpu"), blocks, [0, 1, 2], (11, 40, "coco"),
                      overlap_fn=O.rotate_iou_eval)
    for a, b in zip(got, want):
        _same_tables(a, b)
    mixed = K.eval_many(gts, [sets[0], blocks[1]], [0, 1, 2], (11,), overlap_fn=O.rotate_iou_eval)
    assert [m[11][0] for m in mixed] == [w[11][0] for w in want]


# ------------------------------------------------------------------------------------------------------------ GPU
@pytest.mark.gpu
def test_read_block_equals_read_labels_bit_for_bit(tmp_path):
    import torch
    from sassd_b200 import lib, ops
    rng = np.random.default_rng(7)
    gts, dts = _annos(np.load(GOLD))
    ids = list(range(len(dts)))
    _, (res_dir,) = _write_sets(str(tmp_path / "w"), gts, [dts], ids)
    cases = {"results": (res_dir, ids)}
    gt_ids = list(range(0, 60, 3))
    cases["gt"] = (str(tmp_path / "gt"), write_files(str(tmp_path / "gt"), _gt_files(rng, gt_ids)))
    cases["fast"] = (str(tmp_path / "fast"), write_files(str(tmp_path / "fast"), fuzz_files(rng, fast=True)))
    fuzz = (str(tmp_path / "fuzz"), write_files(str(tmp_path / "fuzz"), fuzz_files(rng)))
    _same_block(K.read_block(*fuzz), _host_block(*fuzz))
    for name, (d, fids) in cases.items():
        _same_block(K.read_block(d, fids), _host_block(d, fids))
        # none of these files leaves the device: KITTI's %.2f, the writer's %.4f and the fast grammar's numbers
        buf = np.concatenate([np.fromfile(os.path.join(d, "%06d.txt" % i), np.uint8) for i in fids])
        off = np.concatenate([[0], np.cumsum([os.path.getsize(os.path.join(d, "%06d.txt" % i)) for i in fids])])
        n_lines, flags = ops.kitti_scan_labels(torch.from_numpy(buf).cuda(), torch.from_numpy(off).cuda())
        assert not (flags.cpu().numpy() & lib.KITTI_PARSE_DEFER).any(), name
        assert n_lines.cpu().numpy().tolist() == [len(a["name"]) for a in KD.read_labels(d, fids)], name
    assert _host_block(*cases["fast"]).off[-1] > 1100

    # deferred files, each alone and all of them among the fuzzed ones
    ddir = str(tmp_path / "deferred")
    files = deferred_files(rng)
    write_files(ddir, {**files, **fuzz_files(np.random.default_rng(8))})
    for i in files:
        try:
            want = _host_block(ddir, [i])
        except Exception as e:          # noqa: BLE001 - the reader's own exception is the expected outcome
            with pytest.raises(type(e)) as got:
                K.read_block(ddir, [i])
            assert str(got.value) == str(e), i
            continue
        _same_block(K.read_block(ddir, [i]), want)
    good = []
    for i in sorted(int(n[:6]) for n in os.listdir(ddir)):
        try:
            KD.read_labels(ddir, [i])
            good.append(i)
        except Exception:               # noqa: BLE001
            pass
    mixed = sorted(good, key=lambda i: (i * 7919) % 131)
    _same_block(K.read_block(ddir, mixed), _host_block(ddir, mixed))


@pytest.mark.gpu
@pytest.mark.parametrize("nsets", [1, 3])
def test_eval_dirs_equals_eval_many_on_read_labels(tmp_path, nsets):
    gts, dts = _annos(np.load(GOLD))
    ids = [3 * i + 1 for i in range(len(gts))]
    gt_dir, dirs = _write_sets(str(tmp_path), gts, _perturbed_sets(dts, nsets), ids)
    tables = (11, 40, "coco")
    for classes in ([0, 1, 2], ["Car"]):
        want = K.eval_many(KD.read_labels(gt_dir, ids), [KD.read_labels(d, ids) for d in dirs], classes, tables)
        times = {}
        got = K.eval_dirs(gt_dir, dirs, ids, classes, tables, times)
        assert len(got) == nsets and set(times) == {"read", "parse", "eval"}
        for a, b in zip(got, want):
            _same_tables(a, b)


@pytest.mark.gpu
def test_command_on_a_driver_out_directory(tmp_path):
    import json
    from sassd_b200 import checkpoint
    from sassd_b200 import test as T
    from tests.kitti_root import write_tree
    root, out, js = str(tmp_path / "kitti"), str(tmp_path / "results"), str(tmp_path / "eval.json")
    write_tree(root)
    ckpt = str(tmp_path / "synthetic.pth")
    checkpoint.save_checkpoint(checkpoint.make_synthetic_state_dict(0, 1), ckpt)
    T.run(T.parse_args([os.path.join(ROOT, "configs", "car_cfg.py"), ckpt, "--data-root", root, "--split", "trainval",
                        "--out", out, "--workers", "2"]), log=lambda *a, **k: None)
    with open(os.path.join(out, "%06d.txt" % 99), "w") as fh:    # a frame the split does not list is ignored
        fh.write("Car 0 0 0 1 2 3 4 1 1 1 1 2 3 0.1 0.9\n")
    printed = []
    res = K.main(["--data-root", root, "--split", "trainval", "--results", out, out, "--classes", "Car", "Pedestrian",
                  "--r40", "--coco", "--json", js], log=lambda *a, **k: printed.append(" ".join(a)))
    ids = KD.read_split(root, "trainval")
    want = K.eval_many(KD.read_labels(os.path.join(root, "training", "label_2"), ids), [KD.read_labels(out, ids)],
                       ["Car", "Pedestrian"], (11, 40, "coco"))[0]
    assert printed[:4] == ["== %s ==" % out, want[11][0], want[40][0], want["coco"][0]]
    assert printed[4:8] == printed[:4]
    assert printed[8] == "summary: 2 directories (moderate 3D AP)"
    assert printed[9].startswith("%-24s  Car 3d mod R11 %6.2f R40 " % (out, want[11][1]["d3"][0, 1, 0]))
    assert printed[11].startswith("frames: %d, directories: 2, read " % len(ids))
    with open(js) as fh:
        saved = json.load(fh)
    assert saved["results"][0]["dir"] == out and saved["results"][0]["text_coco"] == want["coco"][0]
    assert saved["results"][1]["ap_r40"] == K.ap_lists(want[40][1]) == res["results"][1]["ap_r40"]
