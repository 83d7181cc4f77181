"""Several checkpoints of one config in one pass: detectors.CheckpointSweep runs K models over one shared front end
(crop, voxelizer, rulebooks, anchor mask; with GT the nearest voxel centres and the point and RPN targets), and
``python -m sassd_b200.test --checkpoints`` evaluates each checkpoint against one GT (kitti_eval.official_eval_many).

The contract is exact: member k's entry of every sweep result is what member k returns on its own for the same call -
detections, KITTI rows and losses, bit for bit - eager, captured and through detect_stream.

The checkpoints: seed 0's synthetic weights (the only ones whose BatchNorm statistics are calibrated) with the
auxiliary head's weights of tests/test_point_aux.py, every conv and linear weight scaled element by element by
1 + 0.1 N(0, 1) under a generator seed of its own (tests/checkpoint_weights.py)."""
import os

import numpy as np
import pytest

from tests.test_detector_set import same_annos, same_detections

from tests.checkpoint_weights import CAR_CFG, build, checkpoint_state_dict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEEDS = (1, 2, 3)


# ------------------------------------------------------------------ host: validation, driver arguments, evaluation
@pytest.fixture(scope="module")
def cpu_pair():
    return [build("cpu") for _ in range(2)]


def _swap(obj, attr, value):
    old = getattr(obj, attr)
    setattr(obj, attr, value)
    return lambda: setattr(obj, attr, old)


def _shifted_anchor_set(aset):
    import copy
    other = copy.copy(aset)
    other.anchors = aset.anchors + np.float32(0.1)
    return other


@pytest.mark.parametrize("what", ["training", "voxel_size", "max_voxels", "output_shape", "row_cap_factor", "anchors",
                                  "class_names", "train_cfg", "test_cfg", "det_cap"])
def test_sweep_refuses_members_of_different_configs(cpu_pair, what):
    import copy
    from sassd_b200.detectors import CheckpointSweep
    from sassd_b200.voxel_generator import VoxelGenerator
    a, b = cpu_pair
    CheckpointSweep([a, b])
    vg = b.voxel_generator
    kw = dict(voxel_size=list(vg.voxel_size), point_cloud_range=list(vg.point_cloud_range),
              max_num_points=vg.max_num_points_per_voxel, max_voxels=vg.max_voxels, device="cpu")
    if what == "training":
        b.train()
        restore = b.eval
    elif what in ("voxel_size", "max_voxels"):
        kw[what] = dict(voxel_size=[0.05, 0.05, 0.2], max_voxels=16000)[what]
        restore = _swap(b, "voxel_generator", VoxelGenerator(**kw))
    elif what == "output_shape":
        restore = _swap(b.neck, "sparse_shape", [41, 1600, 1408])
    elif what == "row_cap_factor":
        restore = _swap(b.neck, "row_cap_factor", b.neck.row_cap_factor * 2)
    elif what == "anchors":
        restore = _swap(b, "anchor_set", _shifted_anchor_set(b.anchor_set))
    elif what == "class_names":
        restore = _swap(b, "class_names", ["Pedestrian"])
    elif what == "train_cfg":
        cfg = copy.deepcopy(b.train_cfg)
        cfg.rpn.assigner["Car"]["pos_iou_thr"] = 0.65
        restore = _swap(b, "train_cfg", cfg)
    elif what == "test_cfg":
        cfg = copy.deepcopy(b.test_cfg)
        cfg.extra.score_thr = 0.5
        restore = _swap(b, "test_cfg", cfg)
    else:
        restore = _swap(b.extra_head, "det_cap", 256)
    try:
        with pytest.raises(ValueError):
            CheckpointSweep([a, b])
    finally:
        restore()
    CheckpointSweep([a, b])


def test_sweep_refuses_members_on_different_devices_and_empty_lists(cpu_pair):
    import sassd_b200 as S
    from sassd_b200.detectors import CheckpointSweep
    a, _ = cpu_pair
    c = build("cpu").to("meta")
    with pytest.raises(ValueError, match="device"):
        CheckpointSweep([a, c])
    with pytest.raises(ValueError):
        CheckpointSweep([])
    with pytest.raises(TypeError):
        CheckpointSweep([a, object()])
    assert S.CheckpointSweep is CheckpointSweep
    s = CheckpointSweep([a])
    assert s.class_names == ["Car"] and s.models == [a]


def test_member_reload_drops_the_sweeps_captured_steps(cpu_pair):
    from sassd_b200.detectors import CheckpointSweep
    a, b = cpu_pair
    s = CheckpointSweep([a, b])
    s._graphs, s._stream_slots, s._stream_key = {(0, False, False): object()}, [object()], (1,)
    b.refresh_packed_weights()
    assert s._graphs == {} and s._stream_slots is None and s._stream_key is None


def test_driver_arguments_for_a_sweep(tmp_path):
    from sassd_b200 import test as T
    base = ["c.py", "a.pth", "--data-root", "r"]
    a = T.parse_args(base + ["--checkpoints", "b.pth", "c.pth", "--losses", "--r40", "--out", "o", "--json", "j"])
    assert a.checkpoints == ["b.pth", "c.pth"] and a.losses and a.r40
    assert T.parse_args(base).checkpoints == []
    assert T.parse_args(base + ["--checkpoints", "x/b.pth", "y/b.pth"]).checkpoints == ["x/b.pth", "y/b.pth"]
    for bad in (["--checkpoints", "b.pth", "--model", "p.py", "p.pth"],
                ["--checkpoints", "b.pth", "--split", "test", "--out", "o"],
                ["--checkpoints", "a.pth"],
                ["--checkpoints", "b.pth", "./b.pth"],
                ["--checkpoints", "x/b.pth", "y/b.pth", "--out", "o"],
                ["--checkpoints"]):
        with pytest.raises(SystemExit):
            T.parse_args(base + bad)
    with pytest.raises(SystemExit):
        T.parse_args(["c.py", "a.pth", "--drive", "d", "--out", "o", "--checkpoints", "b.pth"])
    assert T.checkpoint_stem("/w/epoch_80.pth") == "epoch_80"


def _eval_annos():
    from tests.test_kitti_eval import GOLD, _annos
    return _annos(np.load(GOLD))


def _same_eval(got, want):
    text, ap = got
    text_w, ap_w = want
    assert text == text_w
    for k in ("bbox", "bev", "d3", "aos"):
        assert (ap[k] is None) == (ap_w[k] is None), k
        if ap_w[k] is not None:
            np.testing.assert_array_equal(ap[k], ap_w[k])


def test_official_eval_many_equals_official_eval_per_set():
    from oracle import kitti_eval as O
    from sassd_b200 import kitti_eval as K
    gts, dts = _eval_annos()
    empty = [{k: v[:0] for k, v in d.items()} for d in dts]
    rs = np.random.RandomState(5)
    fewer = [{k: v[:len(v) // 2] for k, v in d.items()} for d in dts]
    rescored = [dict(d, score=rs.permutation(d["score"])) for d in dts]
    sets = [dts, empty, dts, fewer, rescored]
    got = K.official_eval_many(gts, sets, [0, 1, 2], overlap_fn=O.rotate_iou_eval)
    assert len(got) == len(sets)
    for res, d in zip(got, sets):
        assert set(res) == {11, 40}
        for rp in (11, 40):
            _same_eval(res[rp], K.official_eval(gts, d, [0, 1, 2], overlap_fn=O.rotate_iou_eval, recall_positions=rp))
    # the reference's table (tests/golden/eval.npz) and the oracle, which share no code with official_eval
    g = np.load(os.path.join(ROOT, "tests", "golden", "eval.npz"))
    assert got[0][11][0] == str(g["official_text"]) and got[2][11][0] == str(g["official_text"])
    for s in (1, 3):
        _same_eval(got[s][11], O.official_eval(gts, sets[s], [0, 1, 2]))
    _same_eval(got[0][11], got[2][11])
    _same_eval(got[0][40], got[2][40])
    assert got[1][11][1]["aos"] is None and got[0][11][1]["aos"] is not None
    one = K.official_eval_many(gts, [dts], ["Car"], recall_positions=(40,), overlap_fn=O.rotate_iou_eval)
    assert len(one) == 1 and set(one[0]) == {40}
    _same_eval(one[0][40], K.official_eval(gts, dts, ["Car"], overlap_fn=O.rotate_iou_eval, recall_positions=40))
    with pytest.raises(ValueError, match="11 or 40"):
        K.official_eval_many(gts, [dts], [0], recall_positions=(11, 41), overlap_fn=O.rotate_iou_eval)


def test_official_eval_many_runs_the_gt_side_once_per_class_and_difficulty(monkeypatch):
    from oracle import kitti_eval as O
    from sassd_b200 import kitti_eval as K
    gts, dts = _eval_annos()
    gts, dts = gts[:20], dts[:20]
    calls = {"gt": 0, "overlaps": 0}
    clean_gt, overlaps = K.clean_gt, K._rotated_overlaps

    def count_gt(*a, **k):
        calls["gt"] += 1
        return clean_gt(*a, **k)

    def count_overlaps(*a, **k):
        calls["overlaps"] += 1
        return overlaps(*a, **k)
    monkeypatch.setattr(K, "clean_gt", count_gt)
    monkeypatch.setattr(K, "_rotated_overlaps", count_overlaps)
    K.official_eval_many(gts, [dts] * 4, [0, 1], overlap_fn=O.rotate_iou_eval)
    # two classes x three difficulties, one call per frame, for all metrics and sets; the BEV and 3D overlaps one
    # pass each
    assert calls == {"gt": 2 * 3 * len(gts), "overlaps": 2}


def test_gathered_row_blocks_keep_each_checkpoints_annotations():
    import torch
    from sassd_b200 import test as T
    from sassd_b200.results import annos_from_rows
    rs = np.random.RandomState(2)
    ids, cap = [4, 9, 11, 12, 20], 8
    sets = []
    for k in range(3):          # formatter-layout rows (label 0 = Car), a frame without rows among them
        rows = rs.uniform(-5, 5, (len(ids), cap, 14))
        rows[..., 13] = 0
        n = rs.randint(0, cap + 1, len(ids)).astype(np.int32)
        n[k] = 0
        sets.append(annos_from_rows(rows, n, ["Car"], ids))
    local = [s + [s[0]] for s in sets]         # a padding frame ends the rank's batches
    got = T.gather_annos_many(local, ids, ["Car"], cap, torch.device("cpu"))
    assert len(got) == 3
    for g, w in zip(got, sets):
        same_annos(g, w, "gathered")
    same_annos(T.gather_annos(local[1], ids, ["Car"], cap, torch.device("cpu")), sets[1], "one set")


# ------------------------------------------------------------------ GPU: the bit-for-bit contracts
@pytest.fixture(scope="module")
def models():
    from sassd_b200 import checkpoint
    out = []
    for seed in SEEDS:
        m = build("cuda:0")
        checkpoint.load_state_dict_into(m, checkpoint_state_dict(seed))
        out.append(m)
    return out


@pytest.fixture(scope="module")
def kitti_root(tmp_path_factory):
    """tests/kitti_root.py's synthetic labelled root, with velodyne_reduced: each full sweep cropped to its camera
    frustum (ops.frustum_crop, bit for bit the reference's reduced clouds)."""
    import torch
    from sassd_b200 import ops
    from sassd_b200.kitti_data import KittiSplit
    from tests.kitti_root import write_tree
    root = str(tmp_path_factory.mktemp("sweep") / "kitti")
    write_tree(root)
    split = KittiSplit(root, "trainval", "velodyne")
    os.makedirs(os.path.join(root, "training", "velodyne_reduced"))
    for i in split.ids:
        pts, meta = split.frame(i)
        planes = torch.from_numpy(np.asarray(split.planes(meta["calib"], meta["img_shape"]), np.float64)[None])
        off = torch.tensor([0, len(pts)], dtype=torch.int32, device="cuda")
        kept, k_off = ops.frustum_crop(torch.from_numpy(pts).cuda(), off, 1, planes.cuda())
        kept[:int(k_off[1])].cpu().numpy().tofile(split.path("velodyne_reduced", i, "bin"))
    return root


def _batches(root, B):
    """Batches of the split's frames with their GT: dict(full, reduced, metas, planes, gts, labels) each."""
    from sassd_b200.kitti_data import KittiSplit
    full = KittiSplit(root, "trainval", "velodyne", gt_classes=["Car"])
    reduced = KittiSplit(root, "trainval", "velodyne_reduced")
    ids = full.ids if B > 1 else full.ids[:3]
    out = []
    for j in range(0, len(ids), B):
        frames = [full.frame(i) for i in ids[j:j + B]]
        out.append(dict(full=[p for p, _, _ in frames], reduced=[reduced.frame(i)[0] for i in ids[j:j + B]],
                        metas=[m for _, m, _ in frames],
                        planes=[full.planes(m["calib"], m["img_shape"]) for _, m, _ in frames],
                        gts=[g[0] for _, _, g in frames], labels=[g[1] for _, _, g in frames]))
    return out


KINDS = ("crop_kitti_losses", "reduced_losses", "reduced")


def _call(kind, f):
    if kind == "crop_kitti_losses":
        return f["full"], dict(frustum_planes=f["planes"], metas=f["metas"], gt_bboxes=f["gts"], gt_labels=f["labels"])
    if kind == "reduced_losses":
        return f["reduced"], dict(gt_bboxes=f["gts"], gt_labels=f["labels"])
    return f["reduced"], {}


def _stream_item(kind, f):
    if kind == "crop_kitti_losses":
        return f["full"], f["planes"], f["metas"], (f["gts"], f["labels"])
    if kind == "reduced_losses":
        return f["reduced"], (f["gts"], f["labels"])
    return f["reduced"]


def _stream_kw(kind):
    return dict(crop=kind.startswith("crop"), kitti="kitti" in kind, losses=kind.endswith("losses"))


def _same(kind, got, want, what):
    """One member's result of a kind: detections or KITTI annotations, with the losses when the kind has them."""
    if kind.endswith("losses"):
        (res, losses), (res_w, losses_w) = got, want
        assert losses == losses_w, what
    else:
        res, res_w = got, want
    (same_annos if "kitti" in kind else same_detections)(res, res_w, what)


def _release(*objs):
    import gc
    import torch
    for o in objs:
        o.disable_cuda_graph()
        o.refresh_packed_weights()
    gc.collect()
    torch.cuda.empty_cache()


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 4])
def test_each_member_of_a_sweep_is_that_model(models, kitti_root, B):
    from sassd_b200.detectors import CheckpointSweep
    sweep = CheckpointSweep(models)
    batches = _batches(kitti_root, B)
    want = {}
    n_boxes, nonzero = 0, 0
    for kind in KINDS:                                                   # eager
        for s, f in enumerate(batches):
            pts, kw = _call(kind, f)
            want[kind, s] = [m.forward_points(pts, **kw) for m in models]
            got = sweep.forward_points(pts, **kw)
            assert len(got) == len(models)
            for k in range(len(models)):
                _same(kind, got[k], want[kind, s][k], "eager %s B=%d batch %d member %d" % (kind, B, s, k))
            if kind == "reduced":
                n_boxes += sum(len(d["boxes_lidar"]) for r in got for d in r if d["boxes_lidar"] is not None)
            if kind == "reduced_losses":
                nonzero += sum(v != 0 for _, losses in got for v in losses.values())
    assert n_boxes > 0 and nonzero > 0
    for k in range(1, len(models)):              # different weights, different outputs
        assert want["reduced_losses", 0][k][1] != want["reduced_losses", 0][0][1]
    for obj in models + [sweep]:                                         # captured
        obj.enable_cuda_graph(B, 131072)
    for kind in KINDS:
        for s, f in enumerate(batches):
            pts, kw = _call(kind, f)
            got = sweep.forward_points(pts, **kw)
            for k, m in enumerate(models):
                _same(kind, got[k], want[kind, s][k], "captured %s B=%d batch %d member %d" % (kind, B, s, k))
                _same(kind, m.forward_points(pts, **kw), want[kind, s][k], "member captured %s" % kind)
    assert set(sweep._graphs) == {(0, False, False), (1, True, True), (0, False, True)}
    _release(sweep, *models)
    for kind in KINDS[:2]:                                               # streamed, depth 2
        items = [_stream_item(kind, f) for f in batches]
        got = list(sweep.detect_stream(items, B, 131072, depth=2, **_stream_kw(kind)))
        assert len(got) == len(batches)
        for k, m in enumerate(models):
            own = list(m.detect_stream(items, B, 131072, depth=2, **_stream_kw(kind)))
            for s in range(len(batches)):
                _same(kind, got[s][k], want[kind, s][k], "stream %s B=%d batch %d member %d" % (kind, B, s, k))
                _same(kind, own[s], want[kind, s][k], "member stream %s" % kind)
            _release(m)
        _release(sweep)


@pytest.mark.gpu
def test_a_sweep_of_one_model_is_that_model(models, kitti_root):
    from sassd_b200.detectors import CheckpointSweep
    m = models[0]
    one = CheckpointSweep([m])
    f = _batches(kitti_root, 4)[0]
    for captured in (False, True):
        if captured:
            m.enable_cuda_graph(4, 131072)
            one.enable_cuda_graph(4, 131072)
        for kind in KINDS:
            pts, kw = _call(kind, f)
            got = one.forward_points(pts, **kw)
            assert len(got) == 1
            _same(kind, got[0], m.forward_points(pts, **kw), "one %s captured=%s" % (kind, captured))
    _release(one, m)
    kind = KINDS[0]
    items = [_stream_item(kind, f)] * 2
    got = list(one.detect_stream(items, 4, 131072, depth=2, **_stream_kw(kind)))
    own = list(m.detect_stream(items, 4, 131072, depth=2, **_stream_kw(kind)))
    for g, o in zip(got, own):
        _same(kind, g[0], o, "one stream")
    _release(one, m)


# kernels of the shared front end (voxelizer, rulebooks, anchor mask, nearest voxel centres) and of a member's tail
FRONT = ("vox_emit_kernel", "hash_build_kernel", "conv_mark_kernel", "nbr_fill_kernel", "amask_lookup_kernel",
         "three_nn_kernel")
TAIL = "point_aux_head_kernel"


def _kernel_counts(obj, pts, kw):
    import torch
    from torch.profiler import ProfilerActivity, profile
    obj.forward_points(pts, **kw)          # captures the kind
    g = obj._graph_for(1, True, True)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.graph.replay()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return {k: sum(k in n for n in names) for k in FRONT + (TAIL,)}


@pytest.mark.gpu
def test_a_captured_sweep_step_runs_the_front_end_once(models, kitti_root):
    from sassd_b200.detectors import CheckpointSweep
    f = _batches(kitti_root, 4)[0]
    pts, kw = _call("crop_kitti_losses", f)
    counts = {}
    for K in (1, 3):
        sweep = CheckpointSweep(models[:K])
        sweep.enable_cuda_graph(4, 131072)
        counts[K] = _kernel_counts(sweep, pts, kw)
        _release(sweep)
    for k in FRONT:
        assert counts[1][k] > 0 and counts[3][k] == counts[1][k], (k, counts)
    assert counts[1][TAIL] > 0 and counts[3][TAIL] == 3 * counts[1][TAIL], counts


@pytest.mark.gpu
def test_driver_sweep_matches_single_checkpoint_runs(kitti_root, tmp_path):
    import gc
    import torch
    from sassd_b200 import checkpoint
    from sassd_b200 import test as T
    ckpts = []
    for seed in SEEDS:
        ckpts.append(str(tmp_path / ("epoch_%d.pth" % (2 * seed))))
        checkpoint.save_checkpoint(checkpoint_state_dict(seed), ckpts[-1])
    base = ["--data-root", kitti_root, "--split", "trainval", "--batch", "4", "--workers", "2", "--losses", "--r40"]
    quiet = dict(log=lambda *a, **k: None)
    singles = []
    for i, c in enumerate(ckpts):
        singles.append(T.run(T.parse_args([CAR_CFG, c, "--out", str(tmp_path / ("single_%d" % i))] + base), **quiet))
        gc.collect()
        torch.cuda.empty_cache()
    printed = []
    out = str(tmp_path / "sweep")
    res = T.run(T.parse_args([CAR_CFG, ckpts[0], "--checkpoints"] + ckpts[1:] + ["--out", out,
                             "--json", str(tmp_path / "sweep.json")] + base),
                log=lambda *a, **k: printed.append(" ".join(str(x) for x in a)))
    assert [e["path"] for e in res["checkpoints"]] == ckpts
    for i, (e, single) in enumerate(zip(res["checkpoints"], singles)):
        for key in ("text", "ap", "text_r40", "ap_r40", "losses", "losses_per_batch"):
            assert e[key] == single[key], (i, key)
        got_dir, want_dir = os.path.join(out, "epoch_%d" % (2 * SEEDS[i])), str(tmp_path / ("single_%d" % i))
        names = sorted(os.listdir(want_dir))
        assert sorted(os.listdir(got_dir)) == names and len(names) == 8
        for n in names:
            with open(os.path.join(got_dir, n), "rb") as a, open(os.path.join(want_dir, n), "rb") as b:
                assert a.read() == b.read(), (i, n)
        assert printed.count("== epoch_%d.pth ==" % (2 * SEEDS[i])) == 1
        assert single["text"] in printed and single["text_r40"] in printed
    assert any(e["losses"] != res["checkpoints"][0]["losses"] for e in res["checkpoints"][1:])
    summary = printed[printed.index("summary: 3 checkpoints (moderate 3D AP)") + 1:][:3]
    assert [s.split()[0] for s in summary] == [os.path.basename(c) for c in ckpts]
    assert all("Car 3d mod R11" in s and "R40" in s and "rpn_cls_loss" in s for s in summary)
    with open(str(tmp_path / "sweep.json")) as fh:
        import json
        assert json.load(fh)["checkpoints"][2]["losses"] == singles[2]["losses"]


@pytest.mark.gpu
def test_a_sweep_step_holds_one_networks_activations_at_a_time(models, kitti_root):
    """Each member's activations are freed before the next member runs: the peak of a sweep step, eager and while its
    graph is captured, stays near one model's instead of growing by a network per member."""
    import torch
    from sassd_b200 import detectors as D
    f = _batches(kitti_root, 4)[0]
    pts, kw = _call("crop_kitti_losses", f)
    peaks = {}
    for name, obj in (("single", models[0]), ("sweep", D.CheckpointSweep(models))):
        obj.forward_points(pts, **kw)       # per-model caches (packed weights, empty-scene maps) stay out of the peaks
        for captured in (False, True):
            _release(obj)
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            if captured:
                slot = D._GraphedStep(obj, 4, 131072, crop=D.CROP_FRUSTUM, kitti=True, losses=True,
                                      run_step=D._run_step if name == "single" else D._sweep_step)
                del slot
            else:
                obj.forward_points(pts, **kw)
            torch.cuda.synchronize()
            peaks[name, captured] = torch.cuda.max_memory_allocated() - base
    for captured in (False, True):
        assert peaks["sweep", captured] < 1.25 * peaks["single", captured], peaks
