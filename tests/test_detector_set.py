"""One model per class: detectors.DetectorSet runs several single-class models in one step over shared crops, voxels
and rulebooks (csrc/merge.cu gathers their detections), and ``python -m sassd_b200.test --model`` writes and evaluates
their merged KITTI results.

The contract is exact: each frame's detections from the set are the concatenation, in member order, of what each
member's own forward_points returns for that frame (labels shifted into the set's class list), eager, captured and
through detect_stream; with ``metas`` each frame's KITTI rows are the concatenation of the members' rows.

The members: the Car model of configs/car_cfg.py, and Pedestrian and Cyclist models built from the same config with
one class each and configs/multi_cfg.py's anchor sizes for that class.  Each has weights of its own (member_state_dict):
seed 0's synthetic weights, the only ones whose BatchNorm statistics are calibrated, with every conv and linear weight
of the Pedestrian and Cyclist models - sparse backbone, BEV neck, RPN head, PSWarp head - scaled element by element by
1 + 0.1 N(0, 1) under a seed of their own.  Activations stay in range, every member keeps boxes, and a step that ran
one member's backbone, neck or heads for another would break the equalities.  The frames include an empty one and one
on which some member keeps nothing while another keeps boxes."""
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAR_CFG = os.path.join(ROOT, "configs", "car_cfg.py")
# (class, seed of its weight perturbation (member_state_dict; 0: none), anchor sizes of configs/multi_cfg.py)
MEMBERS = (("Car", 0, [1.6, 3.9, 1.56]), ("Pedestrian", 1, [0.6, 0.8, 1.73]), ("Cyclist", 2, [0.6, 1.76, 1.73]))
WEIGHT_NOISE = 0.1


def member_state_dict(seed):
    """Seed 0's synthetic weights (checkpoint.make_synthetic_state_dict, calibrated BatchNorm), every conv and linear
    weight multiplied element by element by 1 + WEIGHT_NOISE * N(0, 1) drawn under ``seed``; seed 0 leaves them as
    they are."""
    import torch
    from sassd_b200 import checkpoint
    sd = checkpoint.make_synthetic_state_dict(0, 1)
    if seed:
        g = torch.Generator().manual_seed(int(seed))
        for k in sorted(sd):
            if k.endswith(".weight") and sd[k].dim() >= 2:
                sd[k] = sd[k] * (1.0 + WEIGHT_NOISE * torch.randn(sd[k].shape, generator=g))
    return sd
SHAPES = [(375, 1242, 3), (370, 1224, 3), (376, 1241, 3)]


def member_config_text(name, sizes):
    """configs/car_cfg.py turned into a single-class model for ``name`` with the given anchor sizes."""
    with open(CAR_CFG) as fh:
        text = fh.read()
    return text + ("\ndata['val']['class_names'] = [%r]\n"
                   "data['val']['anchor_generator'] = {%r: dict(_anchor, sizes=%r)}\n" % (name, name, sizes))


def member_config(tmp_dir, name, sizes):
    path = os.path.join(str(tmp_dir), "%s_cfg.py" % name.lower())
    with open(path, "w") as fh:
        fh.write(member_config_text(name, sizes))
    return path


def build_member(tmp_dir, name, sizes, device):
    import sassd_b200 as S
    cfg = S.Config.fromfile(CAR_CFG if name == "Car" else member_config(tmp_dir, name, sizes))
    model, _, _ = S.build_from_config(cfg, device=device)
    assert model.class_names == [name]
    return model


# ------------------------------------------------------------------ host: validation, class lists, driver arguments
@pytest.fixture(scope="module")
def cpu_pair(tmp_path_factory):
    d = tmp_path_factory.mktemp("cfg")
    return [build_member(d, n, s, "cpu") for n, _, s in MEMBERS[:2]]


def _swap(obj, attr, value):
    old = getattr(obj, attr)
    setattr(obj, attr, value)
    return old


@pytest.mark.parametrize("what", ["voxel_size", "point_cloud_range", "max_num_points", "max_voxels", "output_shape",
                                  "row_cap_factor", "class", "training"])
def test_set_refuses_members_that_cannot_share_a_step(cpu_pair, what):
    from sassd_b200.detectors import DetectorSet
    from sassd_b200.voxel_generator import VoxelGenerator
    a, b = cpu_pair
    DetectorSet([a, b])
    vg = b.voxel_generator
    kw = dict(voxel_size=list(vg.voxel_size), point_cloud_range=list(vg.point_cloud_range),
              max_num_points=vg.max_num_points_per_voxel, max_voxels=vg.max_voxels, device="cpu")
    change = dict(voxel_size=[0.05, 0.05, 0.2], point_cloud_range=[0., -40., -3., 70.4, 40., 2.], max_num_points=4,
                  max_voxels=16000)
    if what in change:
        kw[what] = change[what]
        old = _swap(b, "voxel_generator", VoxelGenerator(**kw))
        restore = lambda: setattr(b, "voxel_generator", old)  # noqa: E731
    elif what == "output_shape":
        old = _swap(b.neck, "sparse_shape", [41, 1600, 1408])
        restore = lambda: setattr(b.neck, "sparse_shape", old)  # noqa: E731
    elif what == "row_cap_factor":
        old = _swap(b.neck, "row_cap_factor", b.neck.row_cap_factor * 2)
        restore = lambda: setattr(b.neck, "row_cap_factor", old)  # noqa: E731
    elif what == "class":
        old = _swap(b, "class_names", list(a.class_names))
        restore = lambda: setattr(b, "class_names", old)  # noqa: E731
    else:
        b.train()
        restore = b.eval
    try:
        with pytest.raises(ValueError):
            DetectorSet([a, b])
    finally:
        restore()
    DetectorSet([a, b])


def test_set_class_list_and_label_offsets(cpu_pair):
    from sassd_b200.detectors import DetectorSet, merged_classes
    assert merged_classes([["Car"], ["Pedestrian"], ["Cyclist"]]) == (["Car", "Pedestrian", "Cyclist"], [0, 1, 2])
    assert merged_classes([["Car", "Van"], ["Pedestrian"], ["Cyclist", "Tram"]]) == (
        ["Car", "Van", "Pedestrian", "Cyclist", "Tram"], [0, 2, 3])
    assert merged_classes([["Car"]]) == (["Car"], [0])
    with pytest.raises(ValueError):
        merged_classes([["Car", "Van"], ["Van"]])
    a, b = cpu_pair
    s = DetectorSet([b, a])
    assert s.class_names == ["Pedestrian", "Car"] and s.label_offsets == [0, 1]
    assert s.det_cap == a.extra_head.det_cap + b.extra_head.det_cap
    assert DetectorSet([a]).class_names == ["Car"] and DetectorSet([a]).label_offsets == [0]
    with pytest.raises(ValueError):
        DetectorSet([])


def test_member_reload_or_precision_change_drops_the_sets_captured_steps(cpu_pair):
    from sassd_b200 import ops
    from sassd_b200.detectors import DetectorSet
    a, b = cpu_pair
    s = DetectorSet([a, b])
    for change in (lambda: b.refresh_packed_weights(), lambda: a.set_precision(a.neck.fcn.precision)):
        s._graphs, s._stream_slots, s._stream_key = {(0, False): object()}, [object()], (1,)
        own = _swap(a, "_graphs", {(0, False, False): "kept"})
        change()
        assert s._graphs == {} and s._stream_slots is None and s._stream_key is None
        a._graphs = own
    assert a.neck.fcn.precision == ops.DEFAULT_PRECISION


def test_driver_takes_repeated_models_and_refuses_losses_with_them():
    from sassd_b200 import test as T
    a = T.parse_args(["c.py", "w.pth", "--data-root", "r", "--model", "p.py", "p.pth", "--model", "y.py", "y.pth"])
    assert a.model == [["p.py", "p.pth"], ["y.py", "y.pth"]]
    assert T.parse_args(["c.py", "w.pth", "--data-root", "r"]).model == []
    a = T.parse_args(["c.py", "w.pth", "--drive", "d", "--out", "o", "--model", "p.py", "p.pth"])
    assert a.model == [["p.py", "p.pth"]]
    for bad in (["--losses", "--model", "p.py", "p.pth"], ["--model", "p.py"]):
        with pytest.raises(SystemExit):
            T.parse_args(["c.py", "w.pth", "--data-root", "r"] + bad)


def test_merge_detections_is_exported():
    from sassd_b200 import lib
    assert "sassd_merge_detections" in lib.exported_symbols()
    with open(os.path.join(ROOT, "include", "sassd_b200.h")) as fh:
        assert "int sassd_merge_detections(" in fh.read()


def test_member_config_builds_a_single_class_model():
    import sassd_b200 as S
    for name, _, sizes in MEMBERS[1:]:
        ns = {"__file__": CAR_CFG}
        exec(compile(member_config_text(name, sizes), CAR_CFG, "exec"), ns)
        cfg = S.Config({k: v for k, v in ns.items() if not k.startswith("__")}, CAR_CFG)
        assert cfg.data["val"]["class_names"] == [name]
        assert cfg.data["val"]["anchor_generator"][name]["sizes"] == sizes
        assert cfg.model["bbox_head"]["num_class"] == 1


# ------------------------------------------------------------------ GPU: the bit-for-bit contracts
@pytest.fixture(scope="module")
def members(tmp_path_factory):
    from sassd_b200 import checkpoint
    d = tmp_path_factory.mktemp("members")
    out = []
    for name, seed, sizes in MEMBERS:
        m = build_member(d, name, sizes, "cuda:0")
        checkpoint.load_state_dict_into(m, member_state_dict(seed))
        out.append(m)
    return out


MIXED_CANDIDATES = (50, 100, 150, 200, 300, 400, 600, 800, 1200, 1600)


def _mixed_frame(members):
    """The first leading slice of synth_cloud(11) on which some member keeps no box and another keeps boxes."""
    from sassd_b200.synth import synth_cloud
    full = synth_cloud(11)
    pool = [full[:n].copy() for n in MIXED_CANDIDATES]
    kept = np.array([_kept(m.forward_points(pool)) for m in members])       # [member, candidate]
    for j in range(len(pool)):
        if kept[:, j].min() == 0 and kept[:, j].max() > 0:
            return pool[j], kept[:, j]
    raise AssertionError("no candidate frame with a member that keeps nothing beside one that keeps boxes: %s" %
                         kept.tolist())


def _frames(members):
    """A synthetic 20 k-point frame, an empty one, a mixed one (_mixed_frame) and a narrower 20 k-point frame."""
    from sassd_b200.synth import synth_cloud
    return [synth_cloud(12), np.zeros((0, 4), np.float32), _mixed_frame(members)[0], synth_cloud(13, fov_deg=20.0)]


def _calibs(golden_dir):
    from sassd_b200.results import Calibration
    z = np.load(os.path.join(golden_dir, "frustum.npz"))
    return [Calibration({"P2": z["calib%d_P2" % c], "Tr_velo_to_cam": z["calib%d_Tr" % c],
                         "R0_rect": z["calib%d_R0" % c]}) for c in range(2)]


def _sweeps(golden_dir):
    """Full sweeps, the second one empty, with their metas and frustum planes."""
    from sassd_b200.frustum import camera_frustum_planes
    from sassd_b200.synth import synth_cloud
    calibs = _calibs(golden_dir)
    pts = [synth_cloud(30 + j, fov_deg=180.0) if j != 1 else np.zeros((0, 4), np.float32) for j in range(4)]
    metas = [dict(calib=calibs[j % 2], img_shape=SHAPES[j % 3], sample_idx=40 + j) for j in range(len(pts))]
    return pts, metas, [camera_frustum_planes(m["calib"], m["img_shape"]) for m in metas]


def concat_detections(per_member, offsets):
    """Per member a list of per-frame detection dicts -> the per-frame concatenation in member order."""
    out = []
    for frame in zip(*per_member):
        parts = [(d, o) for d, o in zip(frame, offsets) if d["boxes_lidar"] is not None]
        if not parts:
            out.append(dict(boxes_lidar=None, scores=None, label_preds=None))
            continue
        out.append(dict(boxes_lidar=np.concatenate([d["boxes_lidar"] for d, _ in parts]),
                        scores=np.concatenate([d["scores"] for d, _ in parts]),
                        label_preds=np.concatenate([d["label_preds"] + o for d, o in parts])))
    return out


def concat_annos(per_member):
    """Per member a list of per-frame KITTI annotation dicts -> the per-frame concatenation in member order."""
    from sassd_b200.results import empty_result_anno
    out = []
    for frame in zip(*per_member):
        parts = [a for a in frame if len(a["name"])]
        if not parts:
            out.append(empty_result_anno())
            continue
        out.append({k: np.concatenate([a[k] for a in parts]) for k in parts[0]})
    return out


def same_detections(got, exp, what):
    assert len(got) == len(exp), what
    for j, (g, e) in enumerate(zip(got, exp)):
        assert set(g) == set(e), (what, j)
        for k in e:
            if e[k] is None:
                assert g[k] is None, (what, j, k)
            else:
                assert g[k].dtype == e[k].dtype and np.array_equal(g[k], e[k]), (what, j, k)


def same_annos(got, exp, what):
    assert len(got) == len(exp), what
    for j, (g, e) in enumerate(zip(got, exp)):
        assert set(g) == set(e), (what, j)
        for k in e:
            assert np.array_equal(g[k], e[k]), (what, j, k)
            if e[k].dtype.kind != "U":
                assert g[k].dtype == e[k].dtype, (what, j, k)


def _kept(results):
    """Boxes kept per frame."""
    return [0 if r["boxes_lidar"] is None else len(r["boxes_lidar"]) for r in results]


@pytest.mark.gpu
def test_members_have_their_own_weights_and_outputs(members):
    for i in range(len(members)):
        for j in range(i + 1, len(members)):
            for mod in ("neck.backbone.conv1.0.weight", "neck.fcn.conv3.weight", "rpn_head.conv_cls.weight",
                        "extra_head.convs.0.weight"):
                wi, wj = members[i].state_dict()[mod], members[j].state_dict()[mod]
                assert not np.array_equal(wi.cpu().numpy(), wj.cpu().numpy()), (i, j, mod)
    frames = _frames(members)
    res = [m.forward_points(frames) for m in members]
    kept = [_kept(r) for r in res]
    for (name, _, _), k, m in zip(MEMBERS, kept, members):
        assert k[0] > 0 and k[3] > 0 and k[1] == 0 and max(k) <= m.extra_head.det_cap, (name, k)
    mixed = [k[2] for k in kept]
    assert min(mixed) == 0 and max(mixed) > 0, kept
    for i in range(len(members)):             # the same frame, different weights and anchors: different boxes
        for j in range(i + 1, len(members)):
            a, b = res[i][0]["boxes_lidar"], res[j][0]["boxes_lidar"]
            assert a.shape != b.shape or not np.array_equal(a, b), (i, j)


@pytest.mark.gpu
def test_plain_steps_equal_the_members_concatenated(members):
    from sassd_b200.detectors import DetectorSet
    dset = DetectorSet(members)
    assert dset.class_names == ["Car", "Pedestrian", "Cyclist"] and dset.label_offsets == [0, 1, 2]
    frames = _frames(members)
    batches = {1: [frames[:1], frames[1:2], frames[2:3]], 4: [frames, frames[::-1]]}
    for B, bl in batches.items():
        for fb in bl:                                                    # eager
            exp = concat_detections([m.forward_points(fb) for m in members], dset.label_offsets)
            same_detections(dset.forward_points(fb), exp, "eager B=%d" % B)
        for obj in members + [dset]:                                     # captured
            obj.enable_cuda_graph(B, 32768)
        for fb in bl:
            exp = concat_detections([m.forward_points(fb) for m in members], dset.label_offsets)
            same_detections(dset.forward_points(fb), exp, "captured B=%d" % B)
        assert list(dset._graphs) == [(0, False)]
        own = [dict(m._graphs) for m in members]
        for obj in members + [dset]:
            obj.disable_cuda_graph()
        assert all(list(o) == [(0, False, False)] for o in own)
        got = list(dset.detect_stream(bl, B, 32768, depth=2))           # streamed
        per_member = [list(m.detect_stream(bl, B, 32768, depth=2)) for m in members]
        for i in range(len(bl)):
            same_detections(got[i], concat_detections([p[i] for p in per_member], dset.label_offsets),
                            "stream B=%d batch %d" % (B, i))
    assert max(_kept(dset.forward_points(frames[:1]))) > 0


@pytest.mark.gpu
def test_kitti_steps_equal_the_members_rows_concatenated(members, golden_dir):
    from sassd_b200.detectors import DetectorSet
    for m, (name, _, _) in zip(members, MEMBERS):
        m.class_names = [name]
    dset = DetectorSet(members)
    pts, metas, planes = _sweeps(golden_dir)
    kinds = [("frustum", dict(frustum_planes=planes)), ("image_fov", dict(image_fov=True)), ("none", {})]
    n_rows = 0

    def args(kind, idx):
        kw = dict(metas=[metas[i] for i in idx])
        if kind == "frustum":
            kw["frustum_planes"] = [planes[i] for i in idx]
        elif kind == "image_fov":
            kw["image_fov"] = True
        return [pts[i] if kind != "none" else pts[i][pts[i][:, 0] > 0][:30000] for i in idx], kw

    orders = {1: [[0], [1], [3]], 4: [[0, 1, 2, 3], [3, 2, 1, 0]]}
    for kind, _ in kinds:
        for B, order in orders.items():
            for idx in order:                                            # eager
                fb, kw = args(kind, idx)
                got = dset.forward_points(fb, **kw)
                same_annos(got, concat_annos([m.forward_points(fb, **kw) for m in members]), "eager %s" % kind)
                n_rows += sum(len(a["name"]) for a in got)
            for obj in members + [dset]:                                 # captured
                obj.enable_cuda_graph(B, 131072)
            for idx in order:
                fb, kw = args(kind, idx)
                same_annos(dset.forward_points(fb, **kw), concat_annos([m.forward_points(fb, **kw) for m in members]),
                           "captured %s B=%d" % (kind, B))
            for obj in members + [dset]:
                obj.disable_cuda_graph()
    assert n_rows > 0
    # streamed, with the frustum crop and with the image-FOV crop
    for kind, B in (("frustum", 4), ("image_fov", 1)):
        order = orders[B]
        items = []
        for idx in order:
            fb, kw = args(kind, idx)
            items.append((fb, kw["frustum_planes"], kw["metas"]) if kind == "frustum" else (fb, kw["metas"]))
        kw = dict(crop=kind == "frustum", kitti=True, image_fov=kind == "image_fov")
        got = list(dset.detect_stream(items, B, 131072, depth=2, **kw))
        per_member = [list(m.detect_stream(items, B, 131072, depth=2, **kw)) for m in members]
        for i in range(len(order)):
            same_annos(got[i], concat_annos([p[i] for p in per_member]), "stream %s B=%d" % (kind, B))


@pytest.mark.gpu
def test_a_set_of_one_model_is_that_model(members, golden_dir):
    from sassd_b200.detectors import DetectorSet
    car = members[0]
    car.class_names = ["Car"]
    one = DetectorSet([car])
    frames = _frames(members)
    pts, metas, planes = _sweeps(golden_dir)
    for captured in (False, True):
        if captured:
            car.enable_cuda_graph(4, 131072)
            one.enable_cuda_graph(4, 131072)
        same_detections(one.forward_points(frames), car.forward_points(frames), "plain captured=%s" % captured)
        kw = dict(frustum_planes=planes, metas=metas)
        same_annos(one.forward_points(pts, **kw), car.forward_points(pts, **kw), "kitti captured=%s" % captured)
    car.disable_cuda_graph()
    one.disable_cuda_graph()
    got = list(one.detect_stream([frames, frames[::-1]], 4, 32768, depth=2))
    exp = list(car.detect_stream([frames, frames[::-1]], 4, 32768, depth=2))
    for g, e in zip(got, exp):
        same_detections(g, e, "stream")


@pytest.mark.gpu
def test_driver_with_models_writes_and_evaluates_the_merged_results(tmp_path, monkeypatch):
    from sassd_b200 import checkpoint
    from sassd_b200 import test as T
    from sassd_b200.kitti_data import KittiSplit
    from sassd_b200.kitti_eval import official_eval
    from tests.kitti_root import write_tree
    root = str(tmp_path / "kitti")
    write_tree(root)
    cfgs, ckpts = [], []
    for name, seed, sizes in MEMBERS:
        cfgs.append(CAR_CFG if name == "Car" else member_config(tmp_path, name, sizes))
        ckpts.append(str(tmp_path / ("%s.pth" % name)))
        checkpoint.save_checkpoint(member_state_dict(seed), ckpts[-1])
    written = []
    write0 = T.write_results

    def record(out_dir, ids, annos, name="%06d.txt"):
        written.append(annos)
        return write0(out_dir, ids, annos, name)

    monkeypatch.setattr(T, "write_results", record)
    base = ["--data-root", root, "--split", "trainval", "--batch", "4", "--workers", "2"]
    quiet = dict(log=lambda *a, **k: None)
    outs = [str(tmp_path / ("out_%d" % i)) for i in range(len(MEMBERS))]
    for c, k, o in zip(cfgs, ckpts, outs):
        T.run(T.parse_args([c, k, "--out", o] + base), **quiet)
    out = str(tmp_path / "out_set")
    res = T.run(T.parse_args([cfgs[0], ckpts[0], "--out", out, "--model", cfgs[1], ckpts[1], "--model", cfgs[2],
                              ckpts[2]] + base), **quiet)
    names = sorted(os.listdir(out))
    assert names == sorted(os.listdir(outs[0])) and len(names) == 8
    n_lines = [0] * len(MEMBERS)
    for f in names:
        parts = []
        for i, o in enumerate(outs):
            with open(os.path.join(o, f)) as fh:
                lines = fh.read().splitlines()
            n_lines[i] += len(lines)
            parts += lines
        with open(os.path.join(out, f)) as fh:
            assert fh.read().splitlines() == parts, f
    assert min(n_lines) > 0, n_lines
    classes = [n for n, _, _ in MEMBERS]
    merged = concat_annos(written[:len(MEMBERS)])
    same_annos(written[-1], merged, "driver annotations")
    text, ap = official_eval(KittiSplit(root, "trainval", "velodyne").gt_annos(), merged, classes)
    assert res["text"] == text
    for k in ("bbox", "bev", "d3", "aos"):
        assert (ap[k] is None) == (res["ap"][k] is None), k
        if ap[k] is not None:
            assert np.array_equal(np.asarray(res["ap"][k]), np.asarray(ap[k])), k
