"""The device tracker inside the bottom-up step (sb_bottomup_attach_tracker: k_track after the grouping kernel) against
the host tracker with stable greedy ties, on the C4 network of bench.py (heads calibrated as bench.py does) and the
tracking clip's frames."""
import ctypes

import numpy as np
import pytest

from sleap_b200.nn import tracking as T
from track_cases import _close, host_twin

pytestmark = pytest.mark.gpu

N_FRAMES = 48
KW = dict(tracker="simple", similarity="instance", match="greedy", track_window=5)


@pytest.fixture(scope="module")
def c4():
    import bench
    from flow_clip import clip_frames
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    gray = np.ascontiguousarray(clip_frames(N_FRAMES)[:, :, :, :1])
    spec = bench.c4_spec()
    w = A.make_synthetic_weights(A.compile_model(spec, 1), bench.SEED)
    m0 = DeviceModel(spec, w, input_channels=1, precision=0)
    cms0, pafs0 = m0.forward(gray[:2])
    w = bench.calibrate_heads(w, cms0, pafs0, 2)
    del m0
    return DeviceModel(spec, w, input_channels=1, precision=0), gray, bench


def _predictor(c4, batch_size, generic=False):
    from sleap_b200.nn.inference import BottomUpPredictor
    model, _, bench = c4
    pred = BottomUpPredictor(model, bench.NODES, bench.EDGES, peak_threshold=0.2, batch_size=batch_size,
                             integral_refinement=True, max_peaks_per_sample=1024, max_node_peaks=32, max_instances_per_frame=32)
    pred.inference_model.bottomup_layer.return_paf_graph = generic     # the synchronous sb_infer_bottomup path
    return pred


def _summary(frames):
    """Instances (their points), order and tracks of every frame, exactly."""
    return [[(np.asarray(x.numpy()).tobytes(), x.track.name, x.track.spawned_on) for x in lf.instances] for lf in frames]


def _assert_same(a, b):
    """Same instances, order and tracks; tracking scores within 1e-12 relative (CUDA's exp is within an ulp of numpy's)."""
    assert _summary(a) == _summary(b)
    for fa, fb in zip(a, b):
        for xa, xb in zip(fa.instances, fb.instances):
            assert _close(float(xa.tracking_score), float(xb.tracking_score)), (fa.frame_idx, xa.tracking_score, xb.tracking_score)


@pytest.mark.parametrize("generic", [False, True])
def test_predict_with_device_tracker_equals_host(c4, generic, tmp_path):
    _, gray, _ = c4
    results = []
    for bs in (1, 3, 8):
        pred = _predictor(c4, bs, generic)
        pred.tracker = host_twin(**KW)
        host = pred.predict(gray)
        pred.tracker = T.Tracker.make_tracker_by_name(track_device=0, **KW)
        dev = pred.predict(gray)
        assert sum(len(lf.instances) for lf in dev) > N_FRAMES
        _assert_same(host, dev)
        results.append(dev)
    _assert_same(results[0], results[1])
    _assert_same(results[0], results[2])
    from sleap_b200.io.labels import Labels
    path = str(tmp_path / "tracked.slp")
    pred.to_labels(dev).save(path)
    back = Labels.load_file(path)
    assert [[back.tracks[i.track][1] for i in lf.instances] for lf in back.labeled_frames] == \
        [[x.track.name for x in lf.instances] for lf in dev]


def test_device_loop_tracks_equal_run_tracker(c4):
    """K steps of sb_infer_bottomup_dev with the tracker attached, fetched with sb_bottomup_device_tracks, equal
    run_tracker (stable greedy) on the same result records."""
    import torch
    from sleap_b200.nn.inference import LabeledFrame, PredictedInstance
    model, gray, _ = c4
    B = 8
    pred = _predictor(c4, B)
    layer = pred.inference_model.bottomup_layer
    layer._configure(B, *gray.shape[1:])
    dev_tr = T.Tracker.make_tracker_by_name(track_device=0, **KW)
    layer.tracker = dev_tr
    layer.attach_tracker(gray.shape[1:3])
    I, C = layer.max_instances, layer.paf_scorer.n_nodes
    rec_ptr = ctypes.c_void_p()
    model.handle.call("sb_bottomup_device_records", model.model_id, ctypes.byref(rec_ptr))
    from sleap_b200 import parallel

    class _V:
        pass
    v = _V()
    width = parallel.record_width(I, C)
    v.__cuda_array_interface__ = {"shape": (B, width), "typestr": "<f4", "data": (rec_ptr.value, False), "version": 2}
    host_frames, dev_frames = [], []
    for k in range(N_FRAMES // B):
        frames_dev = torch.from_numpy(gray[k * B:(k + 1) * B]).cuda()
        torch.cuda.synchronize()
        model.handle.call("sb_infer_bottomup_dev", model.model_id, ctypes.c_void_p(frames_dev.data_ptr()), B)
        trk = np.zeros((B, 2 + 3 * dev_tr._device.max_instances))
        model.handle.call("sb_bottomup_device_tracks", model.model_id, B, trk.ctypes.data_as(ctypes.c_void_p))
        rec = torch.as_tensor(v, device="cuda").cpu().numpy()
        Id = dev_tr._device.max_instances
        for b in range(B):
            r = rec[b]
            pts = r[:I * C * 2].reshape(I, C, 2)
            vals = r[I * C * 2:I * C * 3].reshape(I, C)
            scores = r[I * C * 3:I * C * 3 + I]
            insts = [PredictedInstance.from_numpy(pts[j], vals[j], float(scores[j])) for j in range(int(r[I * C * 3 + I]))
                     if not np.all(np.isnan(pts[j]))]
            t = k * B + b
            host_frames.append(LabeledFrame(0, t, insts))
            assert trk[b, 1] == 0
            n = int(trk[b, 0])
            dev_frames.append(LabeledFrame(0, t, dev_tr.apply_device_tracks(insts, t, trk[b, 2:2 + n], trk[b, 2 + Id:2 + Id + n],
                                                                            trk[b, 2 + 2 * Id:2 + 2 * Id + n])))
    layer.detach_tracker()
    host = T.run_tracker(host_frames, host_twin(**KW))
    assert sum(len(lf.instances) for lf in host) > N_FRAMES
    _assert_same(host, dev_frames)


def test_predictor_checks_device_and_ranks(c4):
    _, gray, _ = c4
    pred = _predictor(c4, 4)
    pred.tracker = T.Tracker.make_tracker_by_name(track_device=1, **KW)     # not the model's GPU
    with pytest.raises(ValueError):
        pred.predict(gray[:4])
    pred.tracker = T.Tracker.make_tracker_by_name(track_device=0, **KW)
    model = pred.inference_model.bottomup_layer.keras_model
    model.peer_gather = object()                                           # as a multi-rank run sets it
    try:
        with pytest.raises(ValueError):
            pred.predict(gray[:4])
    finally:
        model.peer_gather = None
