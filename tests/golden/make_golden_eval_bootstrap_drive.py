"""Generate tests/golden/eval_bootstrap_drive.npz: the REFERENCE's KITTI evaluation
(mmdet/core/evaluation/kitti_eval.py) on drive-level bootstrap lists: concatenated frame lists of synthetic drives over
the frames of tests/golden/eval_ranges.npz.  The rotated-IoU kernel is numba.cuda code; without a GPU it runs in numba's CUDA
simulator:

    NUMBA_ENABLE_CUDASIM=1 python tests/golden/make_golden_eval_bootstrap_drive.py

The frames are eval_ranges.npz's F0 frames plus one more: frame ``empty_of``'s GT with no detections.  They are grouped
into uneven synthetic drives (``groups``: one label per frame; a drive's frames are not contiguous).  Each list is
evaluated by the unmodified reference on its GT and detection lists: eval_class_v3 + get_mAP_v2 at the official
overlaps (do_eval_v2) and do_coco_style_eval, compute_aos decided as get_official_eval_result decides it (from the
list's first frame with detections).  eval_class_v3 splits a list into num_parts = 50 parts and fails on a list of
fewer frames (an empty part), so a shorter list is evaluated with one part per frame (its default set to the list's
length).  The parts only chunk the overlap computation; the sums still run over the frames in list order.

Keys: ``groups`` [F]; ``flat`` / ``off`` the lists as ReplicateLists holds them (list r = flat[off[r]:off[r + 1]]):
``ordinary`` grouped draws (the drive-level bootstrap's rows at seed 7: sorted labels, the r-th
RandomState(7).randint(0, G, G), each drawn drive's frames ascending), then the largest drive drawn G times (length !=
F), a one-frame list, and a list whose first frame has no detections; ``aos`` [R] compute_aos; per list r
``r<r>_<bbox|bev|d3|aos>`` (do_eval_v2's [class, difficulty, 2 overlap rows]; aos absent without it) and
``r<r>_coco_<...>`` (do_coco_style_eval's [class, difficulty]).
"""
import importlib.util
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import numpy.ma  # noqa: F401  (before make_golden's np.bool shim)
import numba  # noqa: F401

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import import_reference_mmdet  # noqa: E402
from make_golden_eval_bootstrap import CLASSES, COCO, KEYS, OVERLAP  # noqa: E402

ORDINARY = 6
EMPTY_OF = 0


def frames():
    """eval_ranges.npz's frames and one more: frame EMPTY_OF's GT without detections."""
    g = np.load(os.path.join(HERE, "eval_ranges.npz"))
    n = int(g["nframes"])
    gts = [{k: g["gt%d_%s" % (i, k)] for k in KEYS} for i in range(n)]
    dts = [{k: g["dt%d_%s" % (i, k)] for k in KEYS + ("score",)} for i in range(n)]
    gts.append(gts[EMPTY_OF])
    dts.append({k: v[:0] for k, v in dts[EMPTY_OF].items()})
    return gts, dts


def drive_groups(nframes):
    """Uneven drives of 1, 2, 3, ... frames over a fixed shuffle of the frames (the last drive takes the rest)."""
    order = np.random.RandomState(11).permutation(nframes)
    groups = np.zeros(nframes, np.int64)
    start, size, label = 0, 1, 0
    while start < nframes:
        groups[order[start:start + size]] = label
        start, size, label = start + size, size + 1, label + 1
    return groups


def lists(groups, empty):
    labels = np.unique(groups)
    G = len(labels)
    members = [np.flatnonzero(groups == l) for l in labels]
    rs = np.random.RandomState(7)
    rows = [np.concatenate([members[g] for g in rs.randint(0, G, G)]) for _ in range(ORDINARY)]
    big = max(range(G), key=lambda g: len(members[g]))
    rows.append(np.tile(members[big], G))
    rows.append(np.array([members[big][0]]))
    rows.append(np.concatenate([[empty]] + [members[g] for g in range(0, G, 2)]))
    assert len(rows[ORDINARY]) != len(groups)
    return rows


def main():
    assert os.environ.get("NUMBA_ENABLE_CUDASIM") == "1", "run with NUMBA_ENABLE_CUDASIM=1 (no GPU here)"
    import_reference_mmdet()
    for k in list(sys.modules):
        if k.startswith("mmdet.core.post_processing"):
            del sys.modules[k]
    spec = importlib.util.spec_from_file_location(
        "mmdet.core.post_processing.rotate_nms_gpu", "/root/reference/mmdet/core/post_processing/rotate_nms_gpu.py")
    m = importlib.util.module_from_spec(spec); sys.modules[spec.name] = m; spec.loader.exec_module(m)
    spec = importlib.util.spec_from_file_location("ref_kitti_eval", "/root/reference/mmdet/core/evaluation/kitti_eval.py")
    ke = importlib.util.module_from_spec(spec); spec.loader.exec_module(ke)

    linspace = np.linspace

    def linspace_int_num(start, stop, num=50, *a, **k):
        return linspace(start, stop, int(num), *a, **k)
    np.linspace = linspace_int_num          # the reference passes a float num (see make_golden_eval_coco.py)

    gts, dts = frames()
    groups = drive_groups(len(gts))
    rows = lists(groups, len(gts) - 1)
    ranges = np.zeros([3, 3, len(CLASSES)])
    for i, c in enumerate(CLASSES):
        ranges[:, :, i] = np.array(COCO[c])[:, None]
    out = {"groups": groups, "flat": np.concatenate(rows).astype(np.int64),
           "off": np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64),
           "ordinary": np.array(ORDINARY), "empty_of": np.array(EMPTY_OF), "aos": np.zeros(len(rows), bool)}

    def evaluate(row):
        gr, dr = [gts[f] for f in row], [dts[f] for f in row]
        compute_aos = False
        for anno in dr:                      # get_official_eval_result's decision (kitti_eval.py:818-823)
            if anno['alpha'].shape[0] != 0:
                compute_aos = bool(anno['alpha'][0] != -10)
                break
        ke.eval_class_v3.__defaults__ = (False, min(50, len(row)))        # (compute_aos, num_parts)
        res = {}
        for tag, ap in (("", ke.do_eval_v2(gr, dr, CLASSES, OVERLAP, compute_aos, [0, 1, 2])),
                        ("coco_", ke.do_coco_style_eval(gr, dr, CLASSES, ranges, compute_aos))):
            for key, v in zip(("bbox", "bev", "d3", "aos"), ap):
                if v is not None:
                    res[tag + key] = np.asarray(v)
        return compute_aos, res

    if len(sys.argv) == 3:                  # one list, in a process of its own: python THIS r DIR
        r, tmp = int(sys.argv[1]), sys.argv[2]
        aos, res = evaluate(rows[r])
        np.savez(os.path.join(tmp, "%d.npz" % r), compute_aos=aos, **res)
        return
    # the lists are independent: one process each (the simulator is slow)
    tmp = tempfile.mkdtemp()
    procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), str(r), tmp]) for r in range(len(rows))]
    for r, p in enumerate(procs):
        assert p.wait() == 0, "list %d failed" % r
    for r, row in enumerate(rows):
        res = np.load(os.path.join(tmp, "%d.npz" % r))
        out["aos"][r] = bool(res["compute_aos"])
        for name in res.files:
            if name != "compute_aos":
                out["r%d_%s" % (r, name)] = res[name]
        print(r, len(row), out["r%d_d3" % r][:, 1, 0])
    shutil.rmtree(tmp)
    np.linspace = linspace
    np.savez_compressed(os.path.join(HERE, "eval_bootstrap_drive.npz"), **out)


if __name__ == "__main__":
    main()
