"""Generate tests/golden/labels.npz from the REFERENCE's label reader (tools/kitti_common.py get_label_anno /
get_label_annos) run on synthetic label_2 files.  The reference checkout is absent where the tests run, so the fixture
is committed; it holds the files' text and every array the reader returned.

    python tests/golden/make_golden_labels.py

The files cover Car / Van / Pedestrian lines with DontCare lines after them, an empty file and files of scored
16-field lines.  imageio (imported by kitti_common for images only) is stubbed.
"""
import importlib.util
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("SASSD_REFERENCE_ROOT", "/root/reference")


def label_files(rng):
    """{frame id: file text}."""
    def line(name, score=None):
        if name == "DontCare":
            vals = [-1, -1, -10] + list(np.round(rng.uniform(0, 1200, 4), 2)) + [-1, -1, -1, -1000, -1000, -1000, -10]
        else:
            vals = [round(float(rng.uniform(0, 1)), 2), int(rng.integers(0, 4)), round(float(rng.uniform(-3.1, 3.1)), 2)]
            vals += list(np.round(rng.uniform(0, 1200, 4), 2)) + list(np.round(rng.uniform(0.5, 4.5, 3), 2))
            vals += list(np.round(rng.uniform(-20, 60, 3), 2)) + [round(float(rng.uniform(-3.1, 3.1)), 2)]
        if score is not None:
            vals.append(round(score, 4))
        return " ".join([name] + [str(v) for v in vals])

    files = {}
    files[0] = [line("Car"), line("Van"), line("Pedestrian"), line("DontCare"), line("DontCare")]
    files[1] = []
    files[2] = [line("Car")]
    files[3] = [line("Car", float(rng.uniform(0, 1))), line("Cyclist", float(rng.uniform(0, 1))),
                line("Car", float(rng.uniform(0, 1)))]
    files[7] = [line("Van"), line("Car"), line("Truck"), line("DontCare")]
    files[12] = [line("DontCare")]
    files[15] = [line("Pedestrian", 0.5)]
    return {k: "".join(l + "\n" for l in v) for k, v in files.items()}


def main():
    sys.modules["imageio"] = types.SimpleNamespace(imread=None)
    spec = importlib.util.spec_from_file_location("ref_kitti_common", os.path.join(REF, "tools", "kitti_common.py"))
    kc = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(kc)
    files = label_files(np.random.default_rng(11))
    ids = sorted(files)
    out = {"ids": np.array(ids, np.int64)}
    with tempfile.TemporaryDirectory() as d:
        for i in ids:
            out["text_%d" % i] = np.array(files[i])
            with open(os.path.join(d, "%06d.txt" % i), "w") as fh:
                fh.write(files[i])
        for i, anno in zip(ids, kc.get_label_annos(d, ids)):
            single = kc.get_label_anno(os.path.join(d, "%06d.txt" % i))
            assert set(single) | {"image_idx"} == set(anno)
            for k, v in anno.items():
                out["anno_%d_%s" % (i, k)] = v
    np.savez_compressed(os.path.join(HERE, "labels.npz"), **out)
    print("wrote", len(ids), "label files")


if __name__ == "__main__":
    main()
