"""The double-buffered (submit / collect) loops of the single-instance, top-down and top-down identity models against the
per-batch route, bit for bit.

predict_batches of SingleInstanceInferenceModel, TopDownInferenceModel and TopDownMultiClassInferenceModel submits batch
i + 1 (upload on a copy stream, and for top-down the instance stage of batch i and the centroid stage of batch i + 1) before
it collects batch i.  A frame's outputs do not depend on its batch, and the streamed step runs the launches of the
synchronous one, so every batch dict must equal predict_on_batch's on the same frames, array for array, NaNs included.
Cases: frame counts that are not a multiple of B, a single batch, B = 1, an all-black batch (no centroid, crop count 0),
more crops than max_crops_per_call, max_instances set and unset, precisions 0 / 1 / 2 on the trained fixture models, the
predictor with labels on frame arrays and on a video, the device tracker inside the stream, and the refusals of the
submit / collect calls."""
from ctypes import byref

import numpy as np
import pytest

import reference_models as rm
from sleap_b200 import _lib
from sleap_b200.nn import tracking as T
from track_cases import _close

pytestmark = pytest.mark.gpu

NODES = list("abcd")


# ------------------------------------------------------------------------------------------------ helpers
def per_batch(im, imgs, bs):
    return [im.predict_on_batch(np.asarray(imgs[i:i + bs])) for i in range(0, len(imgs), bs)]


def assert_same_batches(got, want):
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert sorted(a) == sorted(b), (i, sorted(a), sorted(b))
        for k in a:
            x, y = np.asarray(a[k]), np.asarray(b[k])
            assert x.dtype == y.dtype and x.shape == y.shape, (i, k, x.dtype, y.dtype, x.shape, y.shape)
            assert x.tobytes() == y.tobytes(), (i, k)


def check_stream(im, imgs, bs):
    """predict_batches == the per-batch loop on the same frames (streamed first: the per-batch calls reuse its pipeline)."""
    got = list(im.predict_batches(imgs, bs))
    assert_same_batches(got, per_batch(im, imgs, bs))
    return got


def variants(img, n):
    """n distinct frames from one: flips and rolls."""
    out = []
    for k in range(n):
        f = img[::-1] if k % 2 else img
        out.append(np.roll(f, 7 * (k // 2), axis=1))
    return np.ascontiguousarray(np.stack(out))


def per_batch_route(self, data, batch_size=4):
    """Stands in for predict_batches: one predict_on_batch per batch."""
    imgs = data
    for i in range(0, len(imgs), batch_size):
        yield self.predict_on_batch(np.asarray(imgs[i:i + batch_size]))


def frames_summary(frames):
    """Frame indices, instances (points, point confidences, score) and tracks, exactly."""
    return [(lf.frame_idx, [(x.numpy().tobytes(), x.point_confidences.tobytes(), x.score, getattr(x.track, "name", None))
                            for x in lf.instances]) for lf in frames]


# ------------------------------------------------------------------------------------------------ synthetic top-down pair
@pytest.fixture(scope="module")
def pair():
    """The centroid / centered-instance UNet pair of the top-down tracker tests on gray clip frames, with an all-black
    stretch (frames 12-15: no centroid), and its thresholds."""
    from scipy.ndimage import maximum_filter
    from flow_clip import clip_frames
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    gray = np.ascontiguousarray(clip_frames(21)[:, :, :, :1])
    gray = np.ascontiguousarray(np.concatenate([gray[:12], np.zeros((4,) + gray.shape[1:], np.uint8), gray[12:]]))
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
    cms = np.concatenate([cmodel.forward(gray[i:i + 5])[0] for i in range(0, 10, 5)])[..., 0]
    fifth = []
    for c in cms:
        v = np.sort(c[c == maximum_filter(c, size=3, mode="constant", cval=-np.inf)])[::-1]
        fifth.append(v[min(4, len(v) - 1)])
    return cmodel, imodel, gray, float(np.median(fifth))


def td_predictor(pair, bs, max_instances=None, chunk=64):
    from sleap_b200.nn.inference import TopDownPredictor
    cmodel, imodel, _, thr = pair
    pred = TopDownPredictor(cmodel, imodel, crop_size=64, peak_threshold=thr, integral_refinement=True, batch_size=bs,
                            max_instances=max_instances)
    pred.inference_model.instance_peaks.peak_threshold = 0.05
    pred.inference_model.instance_peaks.max_crops_per_call = chunk
    assert pred.inference_model._can_fuse()
    return pred


@pytest.mark.parametrize("max_instances,chunk", [(None, 64), (3, 64), (None, 5)])
def test_topdown_stream_synthetic(pair, max_instances, chunk):
    _, _, gray, _ = pair
    im = td_predictor(pair, 4, max_instances, chunk).inference_model
    got = check_stream(im, gray, 4)                        # 25 frames: 7 batches, the last of 1; batch 3 all black
    assert got[3]["n_valid"].sum() == 0 and got[3]["instance_peaks"].shape[1] == 0
    n = sum(int(g["n_valid"].sum()) for g in got)
    assert n > 30
    if chunk < 64:
        assert max(int(g["n_valid"].sum()) for g in got) > chunk          # some batch runs several instance chunks
    check_stream(im, gray[:3], 4)                          # one batch
    check_stream(im, gray[:6], 1)                          # B = 1


def test_topdown_tracker_in_stream(pair, monkeypatch):
    """TopDownPredictor.predict with a device tracker: the streamed route gives the per-batch fused route's instances,
    tracks and tracking scores, and the host tracker never runs."""
    from sleap_b200.nn.inference import TopDownInferenceModel
    from test_gpu_topdown_track import CONFIGS
    _, _, gray, _ = pair

    def no_host_track(*a, **k):
        raise AssertionError("Tracker.track called on the fused route")

    for name, kw in CONFIGS.items():
        pred = td_predictor(pair, 4)
        with monkeypatch.context() as mp:
            mp.setattr(T.Tracker, "track", no_host_track)
            tr_s = pred.tracker = T.Tracker.make_tracker_by_name(track_device=0, **kw)
            streamed = pred.predict(gray)
            mp.setattr(TopDownInferenceModel, "predict_batches", per_batch_route)
            tr_b = pred.tracker = T.Tracker.make_tracker_by_name(track_device=0, **kw)
            batched = pred.predict(gray)
        assert sum(len(lf.instances) for lf in streamed) > 20, name
        assert len(tr_s.spawned_tracks) > 1, name
        assert frames_summary(streamed) == frames_summary(batched), name
        for fa, fb in zip(streamed, batched):
            for xa, xb in zip(fa.instances, fb.instances):
                assert _close(float(xa.tracking_score), float(xb.tracking_score)), name
        assert [(t.name, t.spawned_on) for t in tr_s.spawned_tracks] == [(t.name, t.spawned_on) for t in tr_b.spawned_tracks]


def test_early_stop_collects(pair):
    """A consumer that stops after one batch leaves nothing submitted: the tracker detaches and a synchronous call runs."""
    _, _, gray, _ = pair
    pred = td_predictor(pair, 4)
    im = pred.inference_model
    im.tracker = T.Tracker.make_tracker_by_name(track_device=0, **dict(tracker="simple", similarity="instance", match="greedy",
                                                                      track_window=5))
    gen = im.predict_batches(gray, 4)
    next(gen)
    gen.close()
    im.detach_tracker()
    im.tracker = None
    assert_same_batches([im.predict_on_batch(gray[:4])], per_batch(im, gray[:4], 4))


def test_topdown_refusals(pair):
    """Each refusal is SB_ERR_INVALID with its message and leaves the pipeline usable."""
    from sleap_b200.nn.inference import _topdown_params
    _, _, gray, _ = pair
    pred = td_predictor(pair, 4)
    im = pred.inference_model
    cc, fp = im.centroid_crop, im.instance_peaks
    mc, mi = cc.keras_model, fp.keras_model
    h, mid = mc.handle, mc.model_id
    K = im._configure_fused(4, *gray.shape[1:])
    want = im.predict_on_batch(gray[:4])
    b0, b1 = np.ascontiguousarray(gray[:4]), np.ascontiguousarray(gray[4:8])

    def collect(slot, B=4, fn="sb_topdown_collect"):
        return im._run_fused(B, K, fn, slot)

    def fails(msg, fn, *args):
        with pytest.raises(_lib.SleapB200Error, match=msg):
            h.call(fn, mid, *args)

    def clean():
        h.call("sb_topdown_submit", mid, _lib.ptr(b0), 4, 0)
        assert_same_batches([collect(0)], [want])

    fails("holds no submitted batch", "sb_topdown_collect", 1, 4, *([None] * 6))
    h.call("sb_topdown_submit", mid, _lib.ptr(b0), 4, 0)
    fails("slot 0 holds a batch that was not collected", "sb_topdown_submit", _lib.ptr(b1), 4, 0)
    fails("a batch was submitted and not collected", "sb_infer_topdown", _lib.ptr(b1), 1, 4, *([None] * 6))
    fails("a batch was submitted and not collected", "sb_topdown_attach_tracker", -1, 1.0, 1.0)
    fails("holds a batch of 4 frames, not 3", "sb_topdown_collect", 0, 3, *([None] * 6))
    fails("is not multi-class: call sb_topdown_submit", "sb_topdown_multiclass_submit", _lib.ptr(b1), 4, 1)
    fails("a top-down batch was submitted and not collected", "sb_infer_centroids", _lib.ptr(b1), 1, 4, *([None] * 5))
    fails("bad slot / batch", "sb_topdown_submit", _lib.ptr(b1), 4, 2)
    fails("bad slot / batch", "sb_topdown_submit", _lib.ptr(b1), 5, 1)
    h.call("sb_topdown_submit", mid, _lib.ptr(b1), 4, 1)
    fails("slot 0 was submitted first", "sb_topdown_collect", 1, 4, *([None] * 6))
    assert_same_batches([collect(0), collect(1)], [want, im.predict_on_batch(gray[4:8])])
    clean()
    # the instance model reconfigured between submit and collect: the collect fails cleanly, the configure again recovers
    h.call("sb_topdown_submit", mid, _lib.ptr(b0), 4, 0)
    mi.configure_chain("sb_global_configure", fp.params())
    mi.chain = None
    fails("a model was reconfigured", "sb_topdown_collect", 0, 4, *([None] * 6))
    im._configure_fused(4, *gray.shape[1:])
    fails("holds no submitted batch", "sb_topdown_collect", 0, 4, *([None] * 6))
    clean()
    # the pipeline configured again between submit and collect
    h.call("sb_topdown_submit", mid, _lib.ptr(b0), 4, 0)
    p, _ = _topdown_params(cc, fp)
    h.call("sb_topdown_configure", byref(p), 4, *gray.shape[1:])
    fails("holds no submitted batch", "sb_topdown_collect", 0, 4, *([None] * 6))
    clean()


def test_topdown_tracks_slot_refusals(pair):
    """sb_topdown_tracks from a slot reads only the track records of the batch last collected from it, with its B."""
    from sleap_b200.nn.inference import _topdown_params
    _, _, gray, _ = pair
    im = td_predictor(pair, 4).inference_model
    mc = im.centroid_crop.keras_model
    h, mid = mc.handle, mc.model_id
    p, _ = _topdown_params(im.centroid_crop, im.instance_peaks)
    h.call("sb_topdown_configure", byref(p), 4, *gray.shape[1:])       # a fresh pipeline: no slot collected yet
    im.tracker = T.Tracker.make_tracker_by_name(track_device=0, tracker="simple", similarity="instance", match="greedy",
                                                track_window=5)
    K = im._configure_fused(4, *gray.shape[1:])
    rec = np.zeros((4, 2 + 3 * im.tracker._device.max_instances))
    b0 = np.ascontiguousarray(gray[:4])

    def slot_tracks(slot, B, msg):
        with pytest.raises(_lib.SleapB200Error, match=msg):
            h.call("sb_topdown_tracks", mid, slot, B, _lib.ptr(rec))

    slot_tracks(1, 4, "slot 1 holds no collected batch of 4 frames")
    h.call("sb_topdown_submit", mid, _lib.ptr(b0), 4, 0)
    slot_tracks(0, 4, "slot 0 holds no collected batch of 4 frames")
    out = im._run_fused(4, K, "sb_topdown_collect", 0, slot=0)
    assert out["track_n"].sum() > 0
    slot_tracks(0, 3, "slot 0 holds no collected batch of 3 frames")
    im.detach_tracker()
    im.tracker = None


# ------------------------------------------------------------------------------------------------ trained fixtures
@pytest.mark.parametrize("precision", [0, 1, 2])
def test_single_instance_trained(precision, monkeypatch):
    from sleap_b200.io.video import Video
    from sleap_b200.nn.inference import Predictor, SingleInstanceInferenceModel
    imgs, _ = rm.frames("robot")
    frames = variants(imgs[0], 4)
    frames = np.ascontiguousarray(np.concatenate([imgs, frames, imgs[::-1]]))      # 8 frames
    pred = Predictor.from_model_paths([rm.model_dir("minimal_robot.single_instance")], precision=precision, batch_size=3)
    im = pred.inference_model
    for bs in (3, 1, 8, 16):
        check_stream(im, frames, bs)
    streamed = pred.predict(frames)
    via_video = pred.predict(Video.from_numpy(frames))
    monkeypatch.setattr(SingleInstanceInferenceModel, "predict_batches", per_batch_route)
    batched = pred.predict(frames)
    assert sum(len(lf.instances) for lf in streamed) == len(frames)
    assert frames_summary(streamed) == frames_summary(batched) == frames_summary(via_video)


def test_single_instance_stream_refusals():
    """A batch above the configured B, a collect of a slot that holds no submitted batch and a call of another chain are
    refused; the stream runs afterwards."""
    from sleap_b200.nn.inference import Predictor
    imgs, _ = rm.frames("robot")
    im = Predictor.from_model_paths([rm.model_dir("minimal_robot.single_instance")], precision=1).inference_model
    layer = im.single_instance_layer
    m = layer.keras_model
    want = im.predict_on_batch(imgs)
    layer._configure(2, *imgs.shape[1:])
    pts, vals = np.zeros((2, 4, 2), np.float32), np.zeros((2, 4), np.float32)
    with pytest.raises(_lib.SleapB200Error, match="bad slot / batch"):
        m.handle.call("sb_global_submit", m.model_id, _lib.ptr(imgs), 3, 0)
    with pytest.raises(_lib.SleapB200Error, match="slot 1 holds no submitted batch"):
        m.handle.call("sb_global_collect", m.model_id, 1, 2, _lib.ptr(pts), _lib.ptr(vals))
    with pytest.raises(_lib.SleapB200Error, match="bottom-up predictor not configured"):
        m.handle.call("sb_bottomup_submit", m.model_id, _lib.ptr(imgs), 2, 0)
    assert_same_batches(list(im.predict_batches(imgs, 2)), [want])


def _topdown_trained(precision, max_instances):
    from sleap_b200.nn.inference import Predictor
    paths = [rm.model_dir("minimal_instance.centroid"), rm.model_dir("minimal_instance.centered_instance")]
    return Predictor.from_model_paths(paths, precision=precision, max_instances=max_instances, batch_size=2)


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("max_instances", [None, 1])
def test_topdown_trained(precision, max_instances, monkeypatch):
    from sleap_b200.io.video import Video
    from sleap_b200.nn.inference import TopDownInferenceModel
    imgs, _ = rm.frames("minimal_instance")
    frames = np.ascontiguousarray(np.concatenate([variants(imgs[0], 4), np.zeros_like(imgs), imgs]))    # 6 frames
    pred = _topdown_trained(precision, max_instances)
    im = pred.inference_model
    assert im._can_fuse()
    for bs in (2, 4, 1, 8):
        got = check_stream(im, frames, bs)
        assert sum(int(g["n_valid"].sum()) for g in got) >= (8 if max_instances is None else 4)
    im.instance_peaks.max_crops_per_call = 3                  # several instance chunks per batch
    check_stream(im, frames, 4)
    im.instance_peaks.max_crops_per_call = 64
    streamed = pred.predict(frames)
    via_video = pred.predict(Video.from_numpy(frames))
    monkeypatch.setattr(TopDownInferenceModel, "predict_batches", per_batch_route)
    batched = pred.predict(frames)
    assert frames_summary(streamed) == frames_summary(batched) == frames_summary(via_video)


@pytest.mark.parametrize("precision", [0, 1, 2])
def test_topdown_multiclass_trained(precision, monkeypatch):
    """min_tracks_2node.topdown_multiclass behind the synthetic centroid model of the identity step tests."""
    from sleap_b200.io.video import Video
    from sleap_b200.nn.inference import Predictor, TopDownMultiClassInferenceModel, TopDownMultiClassPredictor
    from test_gpu_topdown_multiclass_step import _models
    imgs, _ = rm.frames("tracks_2node")
    frames = np.ascontiguousarray(np.concatenate([variants(imgs[0], 3), np.zeros_like(imgs), imgs]))    # 5 frames
    cmodel, _ = _models(precision)
    cfg = Predictor._read_config(rm.model_dir("min_tracks_2node.topdown_multiclass"))
    _, _, imodel = Predictor._load(cfg, precision, cmodel.handle, resize_in_graph=False)
    thr = max(float(np.quantile(cmodel.forward(frames[:1])[0], 0.999)), 1e-3)
    pred = TopDownMultiClassPredictor(cmodel, imodel, crop_size=cfg[0]["data"]["instance_cropping"]["crop_size"], peak_threshold=thr,
                                      batch_size=2)
    im = pred.inference_model
    assert im._can_fuse()
    im.instance_peaks.return_class_vectors = True
    for bs in (2, 1, 8):
        got = check_stream(im, frames, bs)
    assert sum(len(g["class_vectors"]) for g in got) > 0
    im.instance_peaks.max_crops_per_call = 2
    check_stream(im, frames, 2)
    im.instance_peaks.max_crops_per_call = 64
    im.instance_peaks.return_class_vectors = False
    streamed = pred.predict(frames)
    via_video = pred.predict(Video.from_numpy(frames))
    monkeypatch.setattr(TopDownMultiClassInferenceModel, "predict_batches", per_batch_route)
    batched = pred.predict(frames)
    assert frames_summary(streamed) == frames_summary(batched) == frames_summary(via_video)


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("max_instances,chunk", [(None, 64), (2, 3)])
def test_topdown_multiclass_synthetic(precision, max_instances, chunk):
    from test_gpu_topdown_multiclass_step import _predictor
    frames = np.random.default_rng(9).integers(0, 256, size=(7, 192, 224, 1), dtype=np.uint8)
    frames[2:4] = 0                                        # B = 2: batch 1 has no centroid
    im = _predictor(precision, frames[:2], max_instances, chunk).inference_model
    im.instance_peaks.return_class_vectors = True
    for bs in (2, 3, 1, 8):
        check_stream(im, frames, bs)


def test_multiclass_refusals():
    from test_gpu_topdown_multiclass_step import _predictor
    frames = np.random.default_rng(9).integers(0, 256, size=(2, 192, 224, 1), dtype=np.uint8)
    im = _predictor(1, frames).inference_model
    want = im.predict_on_batch(frames)
    mc = im.centroid_crop.keras_model
    with pytest.raises(_lib.SleapB200Error, match="is multi-class: call sb_topdown_multiclass_submit"):
        mc.handle.call("sb_topdown_submit", mc.model_id, _lib.ptr(frames), 2, 0)
    mc.handle.call("sb_topdown_multiclass_submit", mc.model_id, _lib.ptr(frames), 2, 0)
    with pytest.raises(_lib.SleapB200Error, match="a batch was submitted and not collected"):
        mc.handle.call("sb_infer_topdown_multiclass", mc.model_id, _lib.ptr(frames), 1, 2, *([None] * 8))
    with pytest.raises(_lib.SleapB200Error, match="is multi-class"):
        mc.handle.call("sb_topdown_collect", mc.model_id, 0, 2, *([None] * 6))
    K = im._configure_fused(2, *frames.shape[1:])
    assert_same_batches([im._run_fused(2, K, "sb_topdown_multiclass_collect", 0)], [want])
