"""Host-side plumbing of the detector step: the table of captured single-step graphs, the detect_stream slots, the
status word and the split of the fixed-size detection rows into per-frame arrays."""
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cpu_model_with_captures():
    """A CPU-built detector whose graph table and stream slots hold placeholders (capturing needs a GPU)."""
    import sassd_b200 as S
    model, _, _ = S.build_from_config(S.Config.fromfile(os.path.join(ROOT, "configs", "car_cfg.py")), device="cpu")
    model._graph_args = (1, 32768)
    model._graphs = {(False, False, False): object(), (True, True, False): object()}
    model._stream_slots = [object(), object()]
    model._stream_key = (1, 32768, 2, False, False)
    return model


def test_weight_reload_and_precision_change_drop_every_captured_step():
    from sassd_b200 import checkpoint, ops
    for change in (lambda m: checkpoint.load_state_dict_into(m, m.state_dict()),
                   lambda m: m.set_precision(ops.PREC_FP32)):
        model = _cpu_model_with_captures()
        change(model)
        assert model._graphs == {}
        assert model._stream_slots is None and model._stream_key is None
        assert model._graph_args == (1, 32768)        # the next forward_points call re-captures at the same shape


def test_disable_cuda_graph_empties_the_table_and_keeps_the_stream_slots():
    model = _cpu_model_with_captures()
    slots, key = model._stream_slots, model._stream_key
    model.disable_cuda_graph()
    assert model._graphs == {} and model._graph_args is None
    assert model._stream_slots is slots and model._stream_key == key


def test_raise_on_status_names_the_flags():
    from sassd_b200 import lib as L
    for ok in (0, np.int32(0), torch.zeros(1, dtype=torch.int32)):
        L.raise_on_status(ok)
    with pytest.raises(L.SassdError, match=r"capacity overflow on device: \['GUIDED_CAP', 'NMS_CAP'\]"):
        L.raise_on_status(4 | 8)
    with pytest.raises(L.SassdError, match="GT_CAP"):
        L.raise_on_status(torch.tensor([64], dtype=torch.int32))
    with pytest.raises(L.SassdError, match="ROWS_CAP"):
        L.raise_on_status(np.array([2], np.int32)[0])


def test_split_detections_per_frame():
    from sassd_b200 import lib as L
    from sassd_b200.single_stage_heads import split_detections, unpack_detections
    rng = np.random.default_rng(0)
    det = rng.standard_normal((3, 6, 9)).astype(np.float32)
    det[..., 8] = rng.integers(0, 3, (3, 6))
    n = np.array([2, 0, 6], np.int32)
    bbs, scs, lbs = split_detections(det, n)
    assert bbs[1] is None and scs[1] is None and lbs[1] is None
    for b in (0, 2):
        k = n[b]
        assert bbs[b].dtype == np.float32 and np.array_equal(bbs[b], det[b, :k, :7])
        assert scs[b].dtype == np.float32 and np.array_equal(scs[b], det[b, :k, 7])
        assert lbs[b].dtype == np.int64 and np.array_equal(lbs[b], det[b, :k, 8])
        assert not any(np.shares_memory(a, det) for a in (bbs[b], scs[b], lbs[b]))
    # the device-tensor entry point splits the same way and checks the status word
    got = unpack_detections(torch.from_numpy(det), torch.from_numpy(n), torch.zeros(1, dtype=torch.int32))
    for x, y in zip(got, (bbs, scs, lbs)):
        assert all((a is None and b is None) or np.array_equal(a, b) for a, b in zip(x, y))
    with pytest.raises(L.SassdError, match="DET_CAP"):
        unpack_detections(torch.from_numpy(det), torch.from_numpy(n), torch.tensor([32], dtype=torch.int32))


@pytest.mark.gpu
def test_capture_collects_dead_detectors_first_and_keeps_the_collector_off(golden_dir, monkeypatch):
    """A dropped detector lives on in its model <-> captured-step cycles until the cyclic collector runs.  Run during
    another capture, the collector would destroy those CUDA graphs mid-capture and invalidate it, at whatever allocation
    it happens to fire.  So a capture collects first and records with the collector off."""
    import gc
    import weakref
    from sassd_b200 import detectors
    from tests.test_kitti_format import _model, _sweeps_and_metas
    assert gc.isenabled()
    pts, _, _ = _sweeps_and_metas(golden_dir, [0])
    old = _model()
    old.enable_cuda_graph(1, 32768)
    old.forward_points(pts)
    assert old._graphs
    dead = weakref.ref(old)
    del old
    seen = []
    run = detectors._run_step

    def spy(*args, **kwargs):
        if torch.cuda.is_current_stream_capturing():
            seen.append((gc.isenabled(), dead() is None))
        return run(*args, **kwargs)

    monkeypatch.setattr(detectors, "_run_step", spy)
    model = _model()
    model.enable_cuda_graph(1, 32768)
    got = model.forward_points(pts)
    assert seen == [(False, True)], "capture ran with the collector on, or with a dead detector's graphs alive"
    assert gc.isenabled() and len(got) == 1
    model.disable_cuda_graph()


@pytest.mark.gpu
def test_enable_cuda_graph_recaptures_every_kind_at_the_new_shape(golden_dir):
    """A second enable_cuda_graph at another shape replaces the kinds captured at the first one: a crop graph left at
    batch 1 would never fit a batch of 2 again, and every cropped call would quietly run eagerly."""
    from tests.test_frustum_crop import _same
    from tests.test_kitti_format import _model, _sweeps_and_metas
    model = _model()
    pts, _, planes = _sweeps_and_metas(golden_dir, [0, 1])
    model.enable_cuda_graph(1, 32768)
    model.forward_points(pts[:1], frustum_planes=planes[:1])
    assert model._graphs[(True, False, False)].batch == 1
    model.enable_cuda_graph(2, 131072)
    got = model.forward_points(pts, frustum_planes=planes)
    assert set(model._graphs) == {(False, False, False), (True, False, False)}
    for g in model._graphs.values():
        assert (g.batch, g.maxpts) == (2, 131072)
    assert model._graphs[(True, False, False)].fits(2, [p.shape[0] for p in pts])
    model.disable_cuda_graph()
    _same(got, model.forward_points(pts, frustum_planes=planes))
