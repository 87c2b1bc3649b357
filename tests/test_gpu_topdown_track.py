"""The device tracker inside the fused top-down step (sb_topdown_attach_tracker: k_track after the record kernel) against
the host tracker with stable greedy ties, on a small centroid / centered-instance UNet pair and the tracking clip's
frames.  The thresholds are calibrated so that frames hold a few centroids and that some nodes and some whole crops
come out NaN."""
import numpy as np
import pytest

from sleap_b200 import _lib
from sleap_b200.nn import tracking as T
from track_cases import _close, host_twin

pytestmark = pytest.mark.gpu

N_FRAMES = 48
NODES = list("abcd")
KW = dict(tracker="simple", similarity="instance", match="greedy", track_window=5)
CONFIGS = {
    "simple/instance/greedy": KW,
    "simplemaxtracks/centroid/hungarian": dict(tracker="simplemaxtracks", similarity="centroid", match="hungarian", track_window=5,
                                               max_tracks=3, max_tracking=True),
    "simple/normalized_instance/greedy": dict(tracker="simple", similarity="normalized_instance", match="greedy", track_window=5),
}


@pytest.fixture(scope="module")
def pair():
    """(centroid model, instance model, gray frames, centroid threshold, instance threshold)."""
    from scipy.ndimage import maximum_filter
    from flow_clip import clip_frames
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.inference import TopDownPredictor
    from sleap_b200.nn.model import DeviceModel
    gray = np.ascontiguousarray(clip_frames(N_FRAMES)[:, :, :, :1])
    ccfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=2, middle_block=True, up_interpolate=True)
    cspec = dict(backbone="unet", backbone_cfg=ccfg, head_type="centroid", part_names=None, edges=None,
                 heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
    icfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=4, middle_block=True, up_interpolate=False)
    ispec = dict(backbone="unet", backbone_cfg=icfg, head_type="centered_instance", part_names=NODES, edges=None,
                 heads=[dict(name="CenteredInstanceConfmapsHead", channels=len(NODES), output_stride=4)])
    cw = A.make_synthetic_weights(A.compile_model(cspec, 1, 0.5), 41)
    iw = A.make_synthetic_weights(A.compile_model(ispec, 1), 43)
    cmodel = DeviceModel(cspec, cw, input_channels=1, input_scale=0.5, precision=1)
    imodel = DeviceModel(ispec, iw, input_channels=1, precision=1)
    # centroid threshold: the median over frames of the 5th-highest local maximum of the centroid map
    cms = np.concatenate([cmodel.forward(gray[i:i + 16])[0] for i in range(0, N_FRAMES, 16)])[..., 0]
    fifth = []
    for c in cms:
        v = np.sort(c[c == maximum_filter(c, size=3, mode="constant", cval=-np.inf)])[::-1]
        fifth.append(v[min(4, len(v) - 1)])
    thr_c = float(np.median(fifth))
    # instance threshold: a quarter of the crops have no node above it
    pred = TopDownPredictor(cmodel, imodel, crop_size=64, peak_threshold=thr_c, integral_refinement=True, batch_size=8)
    pred.inference_model.instance_peaks.peak_threshold = -1e9
    out = pred.inference_model.predict(gray, batch_size=8)
    crop_max = np.concatenate([np.nanmax(out["instance_peak_vals"][b, :n], axis=-1) for b, n in enumerate(out["n_valid"])])
    thr_i = float(np.quantile(crop_max, 0.25))
    return cmodel, imodel, gray, thr_c, thr_i


def _predictor(pair, batch_size, max_instances=None):
    from sleap_b200.nn.inference import TopDownPredictor
    cmodel, imodel, _, thr_c, thr_i = pair
    pred = TopDownPredictor(cmodel, imodel, crop_size=64, peak_threshold=thr_c, integral_refinement=True, batch_size=batch_size,
                            max_instances=max_instances)
    pred.inference_model.instance_peaks.peak_threshold = thr_i
    assert pred.inference_model._can_fuse()
    return pred


def _summary(frames):
    """Instances (their points), order and tracks of every frame, exactly."""
    return [(lf.frame_idx, [(np.asarray(x.numpy()).tobytes(), x.track.name, x.track.spawned_on) for x in lf.instances])
            for lf in frames]


def _assert_same(a, b, tr_a=None, tr_b=None):
    """Same instances, order and tracks; tracking scores within 1e-12 relative (CUDA's exp is within an ulp of numpy's)."""
    assert _summary(a) == _summary(b)
    for fa, fb in zip(a, b):
        for xa, xb in zip(fa.instances, fb.instances):
            assert _close(float(xa.tracking_score), float(xb.tracking_score)), (fa.frame_idx, xa.tracking_score, xb.tracking_score)
    if tr_a is not None:
        assert [(t.name, t.spawned_on) for t in tr_a.spawned_tracks] == [(t.name, t.spawned_on) for t in tr_b.spawned_tracks]


def _no_host_track(*a, **k):
    raise AssertionError("Tracker.track called on the fused route")


def test_workload_has_nan_nodes_and_crops(pair):
    """The calibration gives what the other tests rely on: a few centroids per frame, NaN nodes and all-NaN crops."""
    _, _, gray, _, _ = pair
    im = _predictor(pair, 8).inference_model
    out = im.predict(gray, batch_size=8)
    nv = out["n_valid"]
    print(f"centroids per frame: mean {nv.mean():.2f}, min {nv.min()}, max {nv.max()}")
    assert 2 <= nv.mean() <= 8 and nv.max() >= 3
    rows = np.concatenate([out["instance_peaks"][b, :n] for b, n in enumerate(nv)])
    nan_nodes = np.isnan(rows).any(-1)
    assert nan_nodes.all(-1).any(), "no crop with every node NaN"
    assert (nan_nodes.any(-1) & ~nan_nodes.all(-1)).any(), "no crop with some nodes NaN"


@pytest.mark.parametrize("max_instances", [3, None])
@pytest.mark.parametrize("config", list(CONFIGS))
def test_fused_route_equals_host(pair, config, max_instances, monkeypatch):
    _, _, gray, _, _ = pair
    kw = CONFIGS[config]
    for bs in (1, 3, 8):
        pred = _predictor(pair, bs, max_instances)
        host_tr = pred.tracker = host_twin(**kw)
        host = pred.predict(gray)
        dev_tr = pred.tracker = T.Tracker.make_tracker_by_name(track_device=0, **kw)
        with monkeypatch.context() as mp:
            mp.setattr(T.Tracker, "track", _no_host_track)
            dev = pred.predict(gray)
        assert sum(len(lf.instances) for lf in dev) > N_FRAMES
        assert len(dev_tr.spawned_tracks) > 1
        _assert_same(host, dev, host_tr, dev_tr)


def test_routes_agree(pair):
    """fused = False (the per-frame device tracker on the consumer thread) gives the fused route's frames and tracks."""
    _, _, gray, _, _ = pair
    kw = CONFIGS["simplemaxtracks/centroid/hungarian"]
    pred = _predictor(pair, 3)
    fused_tr = pred.tracker = T.Tracker.make_tracker_by_name(track_device=0, **kw)
    fused = pred.predict(gray)
    pred.inference_model.fused = False
    frame_tr = pred.tracker = T.Tracker.make_tracker_by_name(track_device=0, **kw)
    per_frame = pred.predict(gray)
    assert sum(len(lf.instances) for lf in fused) > N_FRAMES
    _assert_same(fused, per_frame, fused_tr, frame_tr)


def test_state_carries_over_calls(pair):
    """One device tracker over two predict calls; the second one's larger batch reconfigures the pipeline, which drops the
    attachment, and the tracker is attached again with its queues intact."""
    _, _, gray, _, _ = pair
    pred = _predictor(pair, 4, max_instances=4)     # a cap no other test uses: the first call configures for 4 frames
    dev_tr = pred.tracker = T.Tracker.make_tracker_by_name(track_device=0, **KW)
    dev = pred.predict(gray[:20])
    assert pred.centroid_model.configured_for[0] == 4
    pred.batch_size = 8
    dev += pred.predict(gray[20:])
    assert pred.centroid_model.configured_for[0] == 8
    pred = _predictor(pair, 4, max_instances=4)
    host_tr = pred.tracker = host_twin(**KW)
    host = pred.predict(gray[:20])
    pred.batch_size = 8
    host += pred.predict(gray[20:])
    assert len(dev_tr.spawned_tracks) > 1
    _assert_same(host, dev, host_tr, dev_tr)


def test_over_capacity_raises_at_first_frame(pair):
    _, _, gray, _, _ = pair
    pred = _predictor(pair, 8)
    first = next(lf.frame_idx for lf in pred.predict(gray) if len(lf.instances) > 2)
    tr = pred.tracker = T.Tracker.make_tracker_by_name(track_device=0, **KW)
    tr.device_max_instances = 2
    with pytest.raises(_lib.SleapB200Error, match=rf"frame {first} has \d+ instances, more than the device tracker's capacity of 2"):
        pred.predict(gray)


def test_track_abi(pair):
    _, imodel, gray, _, _ = pair
    pred = _predictor(pair, 8)
    im = pred.inference_model
    mc = im.centroid_crop.keras_model
    plain = im.predict_on_batch(gray[:8])
    tr = im.tracker = T.Tracker.make_tracker_by_name(track_device=0, **KW)
    tracked = im.predict_on_batch(gray[:8])
    assert set(tracked) - set(plain) == {"track_n", "track_flags", "track_order", "track_ids", "tracking_scores"}
    for k, v in plain.items():                       # the step's outputs do not change with a tracker attached
        assert v.dtype == tracked[k].dtype and v.shape == tracked[k].shape and v.tobytes() == tracked[k].tobytes(), k
    assert (tracked["track_flags"] == 0).all() and tracked["track_n"].sum() > 0
    rec = np.zeros((8, 2 + 3 * tr._device.max_instances))
    im.detach_tracker()
    im.tracker = None
    with pytest.raises(_lib.SleapB200Error):         # nothing attached
        mc.handle.call("sb_topdown_tracks", mc.model_id, 0, 8, _lib.ptr(rec))
    other = T.DeviceTracker(0, dict(tr.device_params, n_nodes=len(NODES) - 1, max_instances=8, track_table=16), handle=mc.handle)
    with pytest.raises(_lib.SleapB200Error):         # other node count than the instance model's
        mc.handle.call("sb_topdown_attach_tracker", mc.model_id, other.id, 1024.0, 1024.0)
    with pytest.raises(_lib.SleapB200Error):         # no tracker of that id on this handle
        mc.handle.call("sb_topdown_attach_tracker", mc.model_id, 10 ** 6, 1024.0, 1024.0)
    with pytest.raises(_lib.SleapB200Error):         # image size <= 0
        mc.handle.call("sb_topdown_attach_tracker", mc.model_id, tr._device.id, 0.0, 1024.0)
    pred.tracker = T.Tracker.make_tracker_by_name(track_device=1, **KW)     # not the model's GPU
    with pytest.raises(ValueError):
        pred.predict(gray[:4])


def test_multiclass_pipeline_refuses_a_tracker():
    from test_gpu_topdown_multiclass_step import NODES as MC_NODES, _predictor as mc_predictor
    imgs = np.random.default_rng(9).integers(0, 256, size=(4, 192, 224, 1), dtype=np.uint8)
    im = mc_predictor(1, imgs).inference_model
    im.predict_on_batch(imgs)                        # configures the multi-class pipeline
    mc = im.centroid_crop.keras_model
    dev = T.Tracker.make_tracker_by_name(track_device=0, **KW)._device_tracker(len(MC_NODES), handle=mc.handle)
    with pytest.raises(_lib.SleapB200Error):
        mc.handle.call("sb_topdown_attach_tracker", mc.model_id, dev.id, 192.0, 224.0)
