"""Top-down models fed ground-truth centroids (CentroidCropGroundTruth: a centered-instance model on labelled frames) on
the fused, streamed top-down step: sb_topdown_gt_submit on a pipeline configured with centroid_model = -1.

The fused route (predict_on_batch) and the streamed route (predict on labels) must equal the staged route
(fused = False: FrameResizer + sb_crop_centered, crops through host memory, one sb_infer_global per chunk) bit for bit,
NaN positions included; multi-class class probabilities within the 1e-5 of the centroid-model form's test.

Every model of this module lives on the module's own handle, closed when the module ends: the device memory its models,
pipelines and staged-route resizers take is released for the tests that follow."""
from ctypes import byref

import numpy as np
import pytest
from numpy.testing import assert_allclose, assert_array_equal

import reference_models as rm
from sleap_b200 import _lib
from test_gpu_multiclass_step import assert_bit_equal
from test_gpu_predict_pipeline import assert_same_batches, frames_summary
from test_gpu_topdown_multiclass_step import NODES, dense_weights
from test_gpu_topdown_precrop import _edge_centroids

pytestmark = pytest.mark.gpu

F = np.float32
CROP = 64
SB_ERR_INVALID, SB_ERR_UNSUPPORTED = -1, -3
KEYS = ("centroids", "centroid_vals", "instance_peaks", "instance_peak_vals", "n_valid")


def _frames(n, H, W, seed):
    """Smooth uint8 frames (box-filtered noise): the instance network sees structure, not white noise."""
    from scipy.ndimage import uniform_filter
    rng = np.random.default_rng(seed)
    x = uniform_filter(rng.random((n, H, W)).astype(F), size=(1, 9, 9))
    x = (x - x.min()) / (x.max() - x.min())
    return np.ascontiguousarray((x * 255).astype(np.uint8)[..., None])


def _centroids(H, W, counts, seed, nan_rows=()):
    """counts[b] centroids of frame b: the edge set of the top-down precrop tests (inside, on every edge, hanging off every
    side, wholly outside), then random ones; (b, i) in nan_rows: an all-NaN centroid (an instance without visible nodes)."""
    rng = np.random.default_rng(seed)
    edge = _edge_centroids(H, W, CROP)
    out = []
    for b, n in enumerate(counts):
        c = np.concatenate([edge, rng.uniform(0, [W, H], (max(n - len(edge), 0), 2)).astype(F)])[:n] if b % 2 == 0 else \
            rng.uniform(-8, [W + 8, H + 8], (n, 2)).astype(F)
        c = np.array(c, F).reshape(-1, 2)
        for bb, i in nan_rows:
            if bb == b:
                c[i] = np.nan
        out.append(c)
    return out


@pytest.fixture(scope="module")
def dev():
    """The module's handle and the synthetic models built on it, by key; the handle is closed after the module."""
    h = _lib.Handle(0)
    models = {}
    yield h, models
    models.clear()
    h.close()


def _model(dev, key, make):
    h, models = dev
    if key not in models:
        models[key] = make(h)
    return models[key]


def _instance_model(dev, precision):
    """The centered-instance UNet of the top-down precrop tests (4 nodes, output stride 4, no resize op)."""
    def make(h):
        from sleap_b200.nn import architectures as A
        from sleap_b200.nn.model import DeviceModel
        icfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=4, middle_block=True, up_interpolate=False)
        ispec = dict(backbone="unet", backbone_cfg=icfg, head_type="centered_instance", part_names=NODES, edges=None,
                     heads=[dict(name="CenteredInstanceConfmapsHead", channels=len(NODES), output_stride=4)])
        return DeviceModel(ispec, A.make_synthetic_weights(A.compile_model(ispec, 1), 43), input_channels=1, precision=precision,
                           handle=h)
    return _model(dev, ("instance", precision), make)


def _class_model(dev, precision, n_fc=3, units=64, n_classes=4):
    """The centered-instance UNet with a ClassVectorsHead of the top-down multi-class step tests."""
    def make(h):
        import layer_audit as la
        from sleap_b200.nn import architectures as A
        from sleap_b200.nn.model import DeviceModel
        icfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=4, middle_block=True, up_interpolate=False)
        ispec = dict(backbone="unet", backbone_cfg=icfg, head_type="multi_class_topdown", part_names=NODES, edges=None,
                     classes=[f"c{i}" for i in range(n_classes)],
                     heads=[dict(name="CenteredInstanceConfmapsHead", channels=len(NODES), output_stride=4),
                            dict(name="ClassVectorsHead", channels=n_classes, output_stride=16, vector=True, num_fc_layers=n_fc,
                                 num_fc_units=units, global_pool=True)])
        icm = A.compile_model(ispec, 1)
        iw = la.synthetic_weights(icm, 63)
        iw.update(dense_weights(icm.vector_taps["ClassVectorsHead"]["C"], n_fc, units, n_classes, 65, logit_scale=8.0))
        return DeviceModel(ispec, iw, input_channels=1, precision=precision, handle=h)
    return _model(dev, ("class", precision), make)


def _predictor(dev, precision, scale, bs=4, chunk=64):
    from sleap_b200.nn.inference import TopDownPredictor
    imodel = _instance_model(dev, precision)
    imodel.config_input_scale = scale
    pred = TopDownPredictor(None, imodel, crop_size=CROP, peak_threshold=0.05, batch_size=bs)
    im = pred.inference_model
    im.instance_peaks.max_crops_per_call = chunk
    assert im.ground_truth and im._can_fuse() and im.centroid_crop.input_scale == scale
    return pred


def _fused_and_staged(im, ex, keys=KEYS):
    im.fused = True
    a = im.predict_on_batch(ex)
    im.fused = False
    b = im.predict_on_batch(ex)
    im.fused = True
    assert not a["flags"].any()
    for k in keys:
        assert np.asarray(a[k]).shape == np.asarray(b[k]).shape, k
        assert_array_equal(a[k], b[k], err_msg=k)
    return a


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("scale", [1.0, 0.5, 0.75])
def test_fused_equals_staged(dev, precision, scale):
    for (H, W), chunk in (((97, 131), 64), ((160, 200), 4)):
        frames = _frames(5, H, W, H + W)
        cents = _centroids(H, W, [14, 0, 3, 5, 1], H * W, nan_rows=[(2, 1)])
        im = _predictor(dev, precision, scale, chunk=chunk).inference_model
        out = _fused_and_staged(im, dict(image=frames, centroids=cents))
        assert out["n_valid"].tolist() == [14, 0, 3, 5, 1]
        assert np.isnan(out["instance_peaks"][2, 1]).all()                 # the all-NaN centroid's crop has no peaks
        assert np.isfinite(out["instance_peaks"]).any()
        for B in (1, 3):                                                   # batch sizes that do not divide the 5 frames
            for i in range(0, 5, B):
                _fused_and_staged(im, dict(image=frames[i:i + B], centroids=cents[i:i + B]))
        _fused_and_staged(im, dict(image=frames[1:2], centroids=cents[1:2]))       # a batch without centroids


def _labels(frames, counts, seed, n_nodes=4, nan_inst=None):
    """Labels over in-memory frames: counts[b] random instances in frame b (some nodes invisible, some off-frame);
    nan_inst = (b, i): instance i of frame b has no visible node."""
    from sleap_b200.io.labels import Instance, LabeledFrame, Labels, Skeleton
    from sleap_b200.io.video import Video
    rng = np.random.default_rng(seed)
    H, W = frames.shape[1:3]
    sk = Skeleton([str(i) for i in range(n_nodes)], [])
    lfs = []
    for b, n in enumerate(counts):
        insts = []
        for i in range(n):
            c = rng.uniform(-10, [W + 10, H + 10])
            p = (c + rng.normal(0, 12, (n_nodes, 2))).astype(F)
            p[rng.random(n_nodes) < 0.2] = np.nan
            if (b, i) == nan_inst:
                p[:] = np.nan
            insts.append(Instance(p, sk))
        lfs.append(LabeledFrame(0, b, insts))
    lab = Labels(lfs, [{}], [sk])
    lab.set_video(0, Video.from_numpy(frames))
    return lab


def _no_staged_crops(monkeypatch):
    from sleap_b200.nn.inference import CentroidCropGroundTruth

    def refuse(*a, **k):
        raise AssertionError("the staged ground-truth crop ran on the fused route")
    monkeypatch.setattr(CentroidCropGroundTruth, "call", refuse)


@pytest.mark.parametrize("scale", [1.0, 0.5])
def test_stream_equals_staged(dev, scale, monkeypatch):
    """predict(labels) streams (no staged crop runs), and its batches and labelled frames equal the staged route's, at batch
    sizes 1 and 3 over 7 frames, one without instances and one with an all-NaN instance."""
    from sleap_b200.io.labels import LabelsReader
    frames = _frames(7, 120, 150, 5)
    lab = _labels(frames, [3, 0, 5, 2, 1, 4, 2], 11, nan_inst=(2, 3))
    for bs in (1, 3):
        pred = _predictor(dev, 1, scale, bs=bs, chunk=5)
        im = pred.inference_model
        reader = LabelsReader(lab, with_centroids=True)
        with monkeypatch.context() as mp:
            _no_staged_crops(mp)
            streamed = list(im.predict_examples(pred._label_examples(reader), bs, reader.max_instance_count()))
            fused_frames = pred.predict(lab)
        im.fused = False
        staged = [(b, im.predict_on_batch(b)) for b in pred._label_examples(reader)]
        staged_frames = pred.predict(lab)
        im.fused = True
        assert len(streamed) == len(staged) == -(-7 // bs)
        for (ba, a), (bb, b) in zip(streamed, staged):
            assert_array_equal(ba["frame_ind"], bb["frame_ind"])
            assert not a["flags"].any()
            for k in KEYS:                                               # NaN positions, not NaN payloads
                assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
                assert_array_equal(a[k], b[k], err_msg=k)
        assert frames_summary(fused_frames) == frames_summary(staged_frames)
        assert sum(len(lf.instances) for lf in fused_frames) >= 12


def test_results_do_not_depend_on_K(dev):
    frames = _frames(4, 97, 131, 3)
    ex = dict(image=frames, centroids=_centroids(97, 131, [2, 0, 3, 1], 7))
    im = _predictor(dev, 1, 0.5).inference_model
    a = im.predict_on_batch(ex)
    assert im._pipeline.caps[1] == 3
    assert im._configure_ground_truth(4, 11, frames.shape[1:]) == 11
    b = im.predict_on_batch(ex)
    assert im._pipeline.caps[1] == 11
    assert_same_batches([a], [b])


# ------------------------------------------------------------------------------------------------ multi-class
def _mc_predictor(dev, precision, bs=4, chunk=64):
    from sleap_b200.nn.inference import TopDownMultiClassPredictor
    imodel = _class_model(dev, precision)
    pred = TopDownMultiClassPredictor(None, imodel, crop_size=64, integral_refinement=True, batch_size=bs)
    im = pred.inference_model
    im.instance_peaks.peak_threshold = 0.0
    im.instance_peaks.max_crops_per_call = chunk
    assert im.ground_truth and im._can_fuse()
    return pred


def _mc_same(a, b):
    for k in ("centroids", "centroid_vals"):
        assert_bit_equal(a[k], b[k], k)
    assert np.array_equal(np.isnan(a["instance_scores"]), np.isnan(b["instance_scores"])), "class assignments differ"
    assert_bit_equal(a["instance_peaks"], b["instance_peaks"], "points")
    assert_bit_equal(a["instance_peak_vals"], b["instance_peak_vals"], "point values")
    assert_allclose(a["instance_scores"], b["instance_scores"], atol=1e-5, rtol=0)


@pytest.mark.parametrize("precision", [0, 1, 2])
def test_multiclass_fused_equals_staged(dev, precision):
    frames = _frames(4, 192, 224, 17)
    ex = dict(image=frames, centroids=_centroids(224, 192, [5, 0, 3, 2], 19, nan_rows=[(3, 0)])[:4])
    ex["centroids"] = [c % F(190) for c in ex["centroids"]]               # keep them on the frame, NaN stays NaN
    for chunk in (64, 3):
        im = _mc_predictor(dev, precision, chunk=chunk).inference_model
        im.instance_peaks.return_class_vectors = True
        fused = im.predict_on_batch(ex)
        im.fused = False
        staged = im.predict_on_batch(ex)
        im.fused = True
        _mc_same(fused, staged)
        assert not fused["flags"].any() and np.isfinite(fused["instance_scores"]).sum() >= 3
        assert len(fused["class_vectors"]) == 10                            # every crop's probabilities, in crop order


def test_multiclass_stream_and_fixture(dev, monkeypatch):
    """Streamed multi-class predict on synthetic labels equals the staged route, and on the trained
    min_tracks_2node.topdown_multiclass fixture (its labels) in all three precisions."""
    from sleap_b200.io.labels import LabelsReader
    from sleap_b200.nn.inference import TopDownMultiClassPredictor
    frames = _frames(5, 192, 224, 23)
    lab = _labels(frames, [3, 1, 0, 4, 2], 29)
    pred = _mc_predictor(dev, 1, bs=2, chunk=4)
    im = pred.inference_model
    reader = LabelsReader(lab, with_centroids=True)
    with monkeypatch.context() as mp:
        _no_staged_crops(mp)
        streamed = list(im.predict_examples(pred._label_examples(reader), 2, reader.max_instance_count()))
    im.fused = False
    for (_, a), b in zip(streamed, pred._label_examples(reader)):
        _mc_same(a, im.predict_on_batch(b))
    im.fused = True
    labels = rm.labels_tracks_2node()
    d = rm.model_dir("min_tracks_2node.topdown_multiclass")
    for precision in (0, 1, 2):
        p = TopDownMultiClassPredictor.from_trained_models(confmap_model_path=d, peak_threshold=0.7, integral_refinement=False,
                                                           precision=precision, handle=dev[0])
        assert p.inference_model._can_fuse()
        ex = next(p._label_examples(LabelsReader(labels, with_centroids=True)))
        fused = p.inference_model.predict_on_batch(ex)
        p.inference_model.fused = False
        _mc_same(fused, p.inference_model.predict_on_batch(ex))
        staged_frames = p.predict(labels)
        p.inference_model.fused = True
        with monkeypatch.context() as mp:
            _no_staged_crops(mp)
            got = p.predict(labels)
        assert len(got) == 1 and len(got[0].instances) == 2
        assert [(lf.frame_idx, [(x.numpy().tobytes(), x.point_confidences.tobytes(), x.track.name) for x in lf.instances])
                for lf in got] == [(lf.frame_idx, [(x.numpy().tobytes(), x.point_confidences.tobytes(), x.track.name)
                                                   for x in lf.instances]) for lf in staged_frames]


# ------------------------------------------------------------------------------------------------ trained fixtures
@pytest.mark.parametrize("name", ["minimal_instance.centered_instance", "minimal_instance.centered_instance_with_scaling"])
@pytest.mark.parametrize("precision", [0, 1, 2])
def test_trained_fixture_predict_labels(dev, name, precision, monkeypatch):
    from sleap_b200.nn.inference import TopDownPredictor
    labels = rm.labels_minimal_instance()
    pred = TopDownPredictor.from_trained_models(confmap_model_path=rm.model_dir(name), precision=precision, handle=dev[0])
    assert pred.inference_model._can_fuse()
    with monkeypatch.context() as mp:
        _no_staged_crops(mp)
        fused = pred.predict(labels)
    pred.inference_model.fused = False
    staged = pred.predict(labels)
    assert len(fused) == 1 and len(fused[0].instances) == 2
    assert frames_summary(fused) == frames_summary(staged)


# ------------------------------------------------------------------------------------------------ refusals
def _submit(m, frames, table, counts, slot):
    return _lib.lib().sb_topdown_gt_submit(m.handle.h, m.model_id, _lib.ptr(frames), _lib.ptr(table), _lib.ptr(counts),
                                           frames.shape[0], slot)


def test_refusals_keep_the_pipeline(dev):
    from sleap_b200.nn.inference import _centroid_table, _ground_truth_params, topdown_multiclass_params
    frames = _frames(3, 97, 131, 31)
    cents = _centroids(97, 131, [2, 1, 3], 37)
    ex = dict(image=frames, centroids=cents)
    im = _predictor(dev, 1, 0.5).inference_model
    want = im.predict_on_batch(ex)
    m = im.instance_peaks.keras_model
    K = im._pipeline.caps[1]
    table, counts = _centroid_table(cents, K)
    L, h = _lib.lib(), m.handle.h

    def same():
        assert_same_batches([im.predict_on_batch(ex)], [want])

    def refused(rc, code=SB_ERR_INVALID, text=None):
        assert rc == code, rc
        if text:
            assert text.encode() in L.sb_last_error(h), L.sb_last_error(h)
        same()

    for bad in ([K + 1, 0, 0], [-1, 1, 1]):                              # a count above K or below 0
        refused(_submit(m, frames, table, np.asarray(bad, np.int32), 0), text="centroids")
    refused(_submit(m, frames, table, counts, 2))                        # a bad slot
    assert _submit(m, frames, table, counts, 0) == 0                     # an occupied slot
    refused_while_busy = _submit(m, frames, table, counts, 0)
    assert refused_while_busy == SB_ERR_INVALID
    assert _submit(m, frames, table, counts, 1) == 0
    out = lambda slot: im._run_ground_truth(3, K, slot)                  # noqa: E731
    with pytest.raises(_lib.SleapB200Error):                             # an out-of-order collect
        out(1)
    assert_same_batches([out(0), out(1)], [want, want])
    same()
    # the centroid-model calls on a ground-truth pipeline
    z = np.zeros(64, F)
    zi = np.zeros(4, np.int32)
    for rc in (L.sb_infer_topdown(h, m.model_id, _lib.ptr(frames), 1, 3, *[_lib.ptr(z)] * 4, _lib.ptr(zi), _lib.ptr(zi)),
               L.sb_infer_topdown_multiclass(h, m.model_id, _lib.ptr(frames), 1, 3, *[_lib.ptr(z)] * 5, _lib.ptr(zi), _lib.ptr(zi), None),
               L.sb_topdown_submit(h, m.model_id, _lib.ptr(frames), 3, 0),
               L.sb_topdown_multiclass_submit(h, m.model_id, _lib.ptr(frames), 3, 0),
               L.sb_topdown_attach_tracker(h, m.model_id, 0, 97.0, 131.0)):
        refused(rc, text="sb_topdown_gt_submit")
    # the multi-class form at an input scale != 1
    mc = _mc_predictor(dev, 1).inference_model
    fp = mc.instance_peaks
    frames_mc = _frames(2, 192, 224, 41)
    ex_mc = dict(image=frames_mc, centroids=[np.array([[50, 60]], F), np.array([[100, 90], [30, 170]], F)])
    want_mc = mc.predict_on_batch(ex_mc)
    p = topdown_multiclass_params(_ground_truth_params(mc.centroid_crop, fp, 2), fp.keras_model.cm.vector_taps[fp.CLASS_VECTORS],
                                  fp.class_head, fp.dense)
    p.topdown.precrop_resize = 0.5
    assert L.sb_topdown_multiclass_configure(fp.keras_model.handle.h, byref(p), 2, 192, 224, 1) == SB_ERR_UNSUPPORTED
    assert_same_batches([mc.predict_on_batch(ex_mc)], [want_mc])
