"""Top-down predictors built from a centroid model alone, ground-truth instances standing in for the instance model
(FindInstancePeaksGroundTruth: the labelled instance nearest each predicted centroid), on the fused, streamed top-down
step: sb_topdown_gt_instances_submit / _collect on a pipeline configured with instance_model = -1.

The fused route (predict_on_batch) and the streamed route (predict on labels) must equal the host route (fused = False:
the centroid list to the host, the match in numpy) in every key of the batch dict, dtypes, shapes and NaN positions
included.  The labels are built around the centroids the model finds, so that every rule of the match fires: frames
without labelled instances or without centroids, invisible nodes, all-NaN instances first and later, exact distance ties,
and centroids whose every instance is all NaN.

Every model of this module lives on the module's own handle, closed when the module ends."""
from ctypes import byref

import numpy as np
import pytest
from numpy.testing import assert_array_equal

import reference_models as rm
from sleap_b200 import _lib
from test_gpu_predict_pipeline import frames_summary
from test_gpu_reference_models import _matched

pytestmark = pytest.mark.gpu

F = np.float32
SB_ERR_INVALID = -1
KEYS = ("centroids", "centroid_vals", "instance_peaks", "instance_peak_vals", "n_valid", "flags")


def _frames(n, H, W, seed):
    """Smooth uint8 frames (box-filtered noise), frame 1 all black."""
    from scipy.ndimage import uniform_filter
    rng = np.random.default_rng(seed)
    x = uniform_filter(rng.random((n, H, W)).astype(F), size=(1, 9, 9))
    x = (x - x.min()) / (x.max() - x.min())
    out = (x * 255).astype(np.uint8)[..., None]
    if n > 1:
        out[1] = 0
    return np.ascontiguousarray(out)


@pytest.fixture(scope="module")
def dev():
    """The module's handle and the synthetic models built on it, by key; the handle is closed after the module."""
    h = _lib.Handle(0)
    models = {}
    yield h, models
    models.clear()
    h.close()


def _centroid_model(dev, precision, scale):
    """A centroid UNet (output stride 2) at input scale `scale`, and a threshold that passes a few dozen peaks per frame."""
    h, models = dev
    key = ("centroid", precision, scale)
    if key not in models:
        from sleap_b200.nn import architectures as A
        from sleap_b200.nn.model import DeviceModel
        spec = dict(backbone="unet", backbone_cfg=dict(filters=8, filters_rate=2, max_stride=16, output_stride=2, middle_block=True,
                                                       up_interpolate=True),
                    head_type="centroid", part_names=None, edges=None, heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
        m = DeviceModel(spec, A.make_synthetic_weights(A.compile_model(spec, 1, scale), 61), input_channels=1, input_scale=scale,
                        precision=precision, handle=h)
        cms = m.forward(_frames(2, 128, 160, 1))[0]
        models[key] = (m, float(np.quantile(cms, 0.97)), float(np.quantile(cms, 0.6)))
    return models[key]


def _predictor(dev, precision, scale, max_instances=None, bs=4, max_peaks=256, low=False):
    """low: the threshold that passes many peaks per frame."""
    from sleap_b200.nn.inference import TopDownPredictor
    m, thr, thr_low = _centroid_model(dev, precision, scale)
    pred = TopDownPredictor(m, None, peak_threshold=thr_low if low else thr, batch_size=bs, max_instances=max_instances,
                            max_peaks_per_sample=max_peaks)
    assert pred.inference_model._fuses_instances() and not pred.inference_model._can_fuse()
    return pred


def _host_centroids(im, frames):
    """The centroids the host route finds on `frames`, per frame."""
    return [np.asarray(c, F) for c in im.centroid_crop.call(dict(image=frames))["centroids"]]


def _rule_instances(cents, nodes, seed):
    """Labelled instances per frame, built around the frame's centroids so that every rule of the match fires:
    frame 0: none; frame 2: an all-NaN instance 0, then for its first centroid a node 3 px right of it, the same instance
    again and one with the node 3 px below it (exact ties), then instances with invisible nodes; frame 3: an all-NaN instance
    at a later index; frame 4: only all-NaN instances (every centroid is dropped); others: random, some nodes invisible."""
    rng = np.random.default_rng(seed)
    out = []
    for b, c in enumerate(cents):
        near = c[0] if len(c) else F([40, 50])

        def rand(n):                                     # every node at least 8 px from `near` in x and in y
            off = rng.choice([-1, 1], (n, nodes, 2)) * rng.uniform(8, 30, (n, nodes, 2))
            p = (near + off).astype(F)
            p[rng.random((n, nodes)) < 0.25] = np.nan
            return p
        if b == 0:
            inst = np.zeros((0, nodes, 2), F)
        elif b == 2:
            tie = np.full((nodes, 2), np.nan, F)
            tie[0] = near + F([3, 0])
            swap = np.full((nodes, 2), np.nan, F)
            swap[1] = near + F([0, 3])
            inst = np.concatenate([np.full((1, nodes, 2), np.nan, F), tie[None], tie[None], swap[None], rand(4)])
        elif b == 3:
            inst = rand(5)
            inst[3] = np.nan
        elif b == 4:
            inst = np.full((3, nodes, 2), np.nan, F)
        else:
            inst = rand(3 + b % 3)
        out.append(inst)
    return out


def _fused_and_host(im, ex):
    im.fused = True
    a = im.predict_on_batch(ex)
    im.fused = False
    b = im.predict_on_batch(ex)
    im.fused = True
    assert list(a) == list(b)
    for k in KEYS:                                                       # NaN positions, not NaN payloads
        x, y = np.asarray(a[k]), np.asarray(b[k])
        assert x.dtype == y.dtype and x.shape == y.shape, (k, x.dtype, y.dtype, x.shape, y.shape)
        assert_array_equal(x, y, err_msg=k)
    return a


def _host_never_called(mp):
    from sleap_b200.nn.inference import FindInstancePeaksGroundTruth

    def refuse(*a, **k):
        raise AssertionError("the host match ran on the fused route")
    mp.setattr(FindInstancePeaksGroundTruth, "call", refuse)


@pytest.mark.parametrize("max_instances", [None, 1, 2, 3])
@pytest.mark.parametrize("scale", [1.0, 0.5])
@pytest.mark.parametrize("precision", [0, 1, 2])
def test_fused_equals_host(dev, precision, scale, max_instances):
    frames = _frames(6, 128, 160, 7)
    im = _predictor(dev, precision, scale, max_instances).inference_model
    cents = _host_centroids(im, frames)
    insts = _rule_instances(cents, 4, 11)
    ex = dict(image=frames, instances=insts)
    out = _fused_and_host(im, ex)
    n_cent = np.isfinite(out["centroid_vals"]).sum(1)
    assert out["n_valid"][0] == 0 and out["n_valid"][4] == 0             # no instances; only all-NaN instances
    assert out["n_valid"][2] == n_cent[2]                                # the all-NaN instance 0 is never left by a "<"
    assert np.isnan(out["instance_peaks"][2, :n_cent[2]]).all()
    if max_instances is None:
        assert out["n_valid"].sum() >= 3
    for B in (1, 4):                                                     # batches that do not divide the 6 frames
        for i in range(0, 6, B):
            _fused_and_host(im, dict(image=frames[i:i + B], instances=insts[i:i + B]))
    # no centroid above the threshold in any frame
    cc = im.centroid_crop
    thr, cc.peak_threshold = cc.peak_threshold, 1e9
    try:
        none = _fused_and_host(im, ex)
        assert none["centroids"].shape == (6, 0, 2) and none["instance_peaks"].shape == (6, 0, 4, 2)
    finally:
        cc.peak_threshold = thr


def test_ties_and_nan_picks(dev):
    """The host's picks on the rule frames, checked against what they must be: the all-NaN instance 0 of frame 2 is the
    pick of every centroid of that frame, whatever the distances of the others."""
    frames = _frames(6, 128, 160, 7)
    im = _predictor(dev, 1, 1.0).inference_model
    cents = _host_centroids(im, frames)
    insts = _rule_instances(cents, 4, 11)
    out = _fused_and_host(im, dict(image=frames, instances=insts))
    assert out["n_valid"][2] == len(cents[2]) > 0 and np.isnan(out["instance_peaks"][2, :len(cents[2])]).all()
    # without the all-NaN instance 0, instances 0 and 1 (the same points) tie exactly: the pick is instance 0, or instance 2
    # (a node 3 px below rather than right of the centroid) where its rounded distance is strictly smaller
    insts[2] = insts[2][1:]
    out = _fused_and_host(im, dict(image=frames, instances=insts))
    c = cents[2][0]
    d = [np.sqrt((insts[2][j][k, 0] - c[0]) ** 2 + (insts[2][j][k, 1] - c[1]) ** 2) for j, k in ((0, 0), (2, 1))]
    assert_array_equal(out["instance_peaks"][2, 0], insts[2][2 if d[1] < d[0] else 0])


def test_caps_past_one_pass(dev):
    """N = 40 instances of 20 nodes (the lane loop over instances and every record loop run more than one pass), frames
    with more centroids than the 4 warps, K filled to its size by the top-k and by max_peaks_per_sample; then the refusal
    of a count of N + 1 or -1, and the next valid submit into the same slot."""
    frames = _frames(3, 128, 160, 13)
    for max_instances, max_peaks in ((6, 256), (None, 8)):
        im = _predictor(dev, 1, 1.0, max_instances=max_instances, max_peaks=max_peaks, low=True).inference_model
        cents = _host_centroids(im, frames)
        K = max_instances or max_peaks
        assert len(cents[0]) == K and len(cents[2]) == K, [len(c) for c in cents]
        rng = np.random.default_rng(17)
        insts = []
        for c in cents:
            near = c[0] if len(c) else F([64, 80])
            p = (near + rng.uniform(-60, 60, (40, 20, 2))).astype(F)
            p[rng.random((40, 20)) < 0.5] = np.nan
            insts.append(p)
        ex = dict(image=frames, instances=insts)
        out = _fused_and_host(im, ex)
        assert out["n_valid"].tolist() == [len(c) for c in cents]
        assert im._pipeline.caps[1] == 40 and im._pipeline.key[2][0] == 20      # N, and the node count
    from sleap_b200.nn.inference import _instance_table
    im.predict_on_batch(ex)                                              # the host route's centroid call dropped the pipeline
    m = im.centroid_crop.keras_model
    L, h = _lib.lib(), m.handle.h
    table, _ = _instance_table(insts, 40, 20)
    for bad in ([41, 0, 0], [0, -1, 3]):
        rc = L.sb_topdown_gt_instances_submit(h, m.model_id, _lib.ptr(frames), _lib.ptr(table), _lib.ptr(np.asarray(bad, np.int32)), 3, 0)
        assert rc == SB_ERR_INVALID and b"instances" in L.sb_last_error(h)
        counts = np.asarray([40, 40, 40], np.int32)
        assert L.sb_topdown_gt_instances_submit(h, m.model_id, _lib.ptr(frames), _lib.ptr(table), _lib.ptr(counts), 3, 0) == 0
        got = im._run_gt_instances(3, 8, 20, 0)
        for k in KEYS:
            assert_array_equal(got[k], out[k], err_msg=k)


# ------------------------------------------------------------------------------------------------ trained fixture
@pytest.mark.parametrize("precision", [0, 1, 2])
def test_trained_fixture(dev, precision, monkeypatch):
    """minimal_instance.centroid on minimal_instance.slp, the host match never called: two instances within 1.5 px of the
    labels, max_instances cuts, none at threshold 1.5; and the same labelled frames as the host route."""
    from sleap_b200.nn.inference import TopDownPredictor
    labels = rm.labels_minimal_instance()
    gt = np.concatenate([i.numpy() for i in labels[0].instances])
    d = rm.model_dir("minimal_instance.centroid")
    pred = TopDownPredictor.from_trained_models(centroid_model_path=d, precision=precision, handle=dev[0])
    assert pred.inference_model._fuses_instances()
    pred.inference_model.fused = False
    host = pred.predict(labels)
    pred.inference_model.fused = True
    with monkeypatch.context() as mp:
        _host_never_called(mp)
        frames = pred.predict(labels)
        assert len(frames) == 1 and len(frames[0].instances) == 2
        _matched(gt, np.concatenate([i.numpy() for i in frames[0].instances]), 1.5)
        assert frames_summary(frames) == frames_summary(host)
        for k in (1, 2, 3):
            p = TopDownPredictor.from_trained_models(centroid_model_path=d, precision=precision, max_instances=k, handle=dev[0])
            assert len(p.predict(labels)[0].instances) == min(k, 2)
        hi = TopDownPredictor.from_trained_models(centroid_model_path=d, precision=precision, peak_threshold=1.5, handle=dev[0])
        assert len(hi.predict(labels)[0].instances) == 0


# ------------------------------------------------------------------------------------------------ streaming
def _labels(videos, order, seed, nodes=4):
    """Labels over in-memory videos: frames in `order` ((video, frame) pairs), 0-5 random instances each, some nodes
    invisible, one all-NaN instance."""
    from sleap_b200.io.labels import Instance, LabeledFrame, Labels, Skeleton
    from sleap_b200.io.video import Video
    rng = np.random.default_rng(seed)
    sk = Skeleton([str(i) for i in range(nodes)], [])
    lfs = []
    for n, (v, f) in enumerate(order):
        H, W = videos[v].shape[1:3]
        insts = []
        for i in range(int(rng.integers(0, 6))):
            p = (rng.uniform(0, [W, H]) + rng.normal(0, 12, (nodes, 2))).astype(F)
            p[rng.random(nodes) < 0.2] = np.nan
            if (n, i) == (2, 1):
                p[:] = np.nan
            insts.append(Instance(p, sk))
        lfs.append(LabeledFrame(v, f, insts))
    lab = Labels(lfs, [{} for _ in videos], [sk])
    for v, fr in enumerate(videos):
        lab.set_video(v, Video.from_numpy(fr))
    return lab


def _same_rows(a, i, b, j):
    """Frame i of batch dict a equals frame j of batch dict b, up to the batches' padding widths."""
    nr, nc = a["n_valid"][i], np.isfinite(a["centroid_vals"][i]).sum()
    assert nr == b["n_valid"][j] and nc == np.isfinite(b["centroid_vals"][j]).sum() and a["flags"][i] == b["flags"][j]
    for k, n in (("centroids", nc), ("centroid_vals", nc), ("instance_peaks", nr), ("instance_peak_vals", nr)):
        assert_array_equal(a[k][i, :n], b[k][j, :n], err_msg=k)


def test_stream_equals_host(dev, monkeypatch):
    """predict over a LabelsReader streams (the host match never runs) through batches of 3 of 3 frames of one video, 3
    of a second video of another size, then a short batch of 2 of the first; its batches equal the per-batch host loop,
    each frame equals its run alone, and its labelled frames equal the host route's."""
    from sleap_b200.io.labels import LabelsReader
    videos = [_frames(5, 128, 160, 21), _frames(3, 96, 192, 23)]
    lab = _labels(videos, [(0, 0), (0, 1), (0, 2), (1, 0), (1, 1), (1, 2), (0, 3), (0, 4)], 25)
    pred = _predictor(dev, 1, 0.5, bs=3)
    im = pred.inference_model
    reader = LabelsReader(lab, with_centroids=True)
    with monkeypatch.context() as mp:
        _host_never_called(mp)
        streamed = list(im.predict_examples(pred._label_examples(reader), 3, reader.max_instance_count()))
        fused_frames = pred.predict(lab)
        alone = [im.predict_on_batch(dict(image=b["image"][i:i + 1], instances=b["instances"][i:i + 1]))
                 for b, _ in streamed for i in range(len(b["image"]))]
    im.fused = False
    host = [(b, im.predict_on_batch(b)) for b in pred._label_examples(reader)]
    host_frames = pred.predict(lab)
    im.fused = True
    assert [len(b["image"]) for b, _ in streamed] == [3, 3, 2]
    assert len(streamed) == len(host)
    f = 0
    for (ba, a), (bb, b) in zip(streamed, host):
        assert_array_equal(ba["frame_ind"], bb["frame_ind"])
        for k in KEYS:
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape, k
            assert_array_equal(a[k], b[k], err_msg=k)
        for i in range(len(ba["image"])):
            _same_rows(a, i, alone[f], 0)
            f += 1
    assert frames_summary(fused_frames) == frames_summary(host_frames)
    assert sum(len(lf.instances) for lf in fused_frames) >= 4


# ------------------------------------------------------------------------------------------------ refusals and chain rules
def _instance_model(h):
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    icfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=4, middle_block=True, up_interpolate=False)
    ispec = dict(backbone="unet", backbone_cfg=icfg, head_type="centered_instance", part_names=list("abcd"), edges=None,
                 heads=[dict(name="CenteredInstanceConfmapsHead", channels=4, output_stride=4)])
    return DeviceModel(ispec, A.make_synthetic_weights(A.compile_model(ispec, 1), 43), input_channels=1, precision=1, handle=h)


def test_refusals_and_chain_rules(dev):
    from sleap_b200.nn.inference import TopDownPredictor, _gt_instances_params, _instance_table
    frames = _frames(3, 128, 160, 31)
    im = _predictor(dev, 1, 1.0, max_instances=3).inference_model
    insts = _rule_instances(_host_centroids(im, frames), 4, 33)
    ex = dict(image=frames, instances=insts)
    want = _fused_and_host(im, ex)
    im.predict_on_batch(ex)                                              # the host route's centroid call dropped the pipeline
    m = im.centroid_crop.keras_model
    L, h = _lib.lib(), m.handle.h
    N = im._pipeline.caps[1]
    table, counts = _instance_table(insts, N, 4)

    def submit(slot, c=counts):
        return L.sb_topdown_gt_instances_submit(h, m.model_id, _lib.ptr(frames), _lib.ptr(table), _lib.ptr(c), 3, slot)

    def same(got):
        for k in KEYS:
            assert_array_equal(got[k], want[k], err_msg=k)

    def refused(rc, text):
        assert rc == SB_ERR_INVALID, rc
        assert text.encode() in L.sb_last_error(h), L.sb_last_error(h)

    out = lambda slot: im._run_gt_instances(3, 3, 4, slot)              # noqa: E731
    refused(submit(0, np.asarray([N + 1, 0, 0], np.int32)), "instances")
    refused(submit(2), "bad slot")
    assert submit(0) == 0
    refused(submit(0), "not collected")                                  # an occupied slot
    assert submit(1) == 0
    with pytest.raises(_lib.SleapB200Error):                             # an out-of-order collect
        out(1)
    same(out(0))
    same(out(1))
    # the other calls on this pipeline
    z = np.zeros(4096, F)
    zi = np.zeros(64, np.int32)
    zc = np.zeros((3, 8, 2), F)
    for rc in (L.sb_infer_topdown(h, m.model_id, _lib.ptr(frames), 1, 3, *[_lib.ptr(z)] * 4, _lib.ptr(zi), _lib.ptr(zi)),
               L.sb_infer_topdown_multiclass(h, m.model_id, _lib.ptr(frames), 1, 3, *[_lib.ptr(z)] * 5, _lib.ptr(zi), _lib.ptr(zi), None),
               L.sb_topdown_submit(h, m.model_id, _lib.ptr(frames), 3, 0),
               L.sb_topdown_collect(h, m.model_id, 0, 3, *[_lib.ptr(z)] * 4, _lib.ptr(zi), _lib.ptr(zi)),
               L.sb_topdown_gt_submit(h, m.model_id, _lib.ptr(frames), _lib.ptr(zc), _lib.ptr(zi), 3, 0),
               L.sb_topdown_multiclass_submit(h, m.model_id, _lib.ptr(frames), 3, 0),
               L.sb_topdown_multiclass_collect(h, m.model_id, 0, 3, *[_lib.ptr(z)] * 5, _lib.ptr(zi), _lib.ptr(zi), None),
               L.sb_topdown_attach_tracker(h, m.model_id, 0, 128.0, 160.0),
               L.sb_topdown_tracks(h, m.model_id, 0, 3, _lib.ptr(np.zeros(64))) ):
        refused(rc, "sb_topdown_gt_instances_submit")
    same(im.predict_on_batch(ex))
    # configure refusals
    p, K = _gt_instances_params(im.centroid_crop)
    p.instance_model = m.model_id
    refused(L.sb_topdown_gt_instances_configure(h, byref(p), 4, N, 3, 128, 160, 1), "instance_model")
    p.instance_model = -1
    for args in ((0, N), (4, 0)):
        refused(L.sb_topdown_gt_instances_configure(h, byref(p), *args, 3, 128, 160, 1), "sizes")
    # the other forms refuse this form's calls; configuring the centroid model drops this pipeline
    imodel = _instance_model(dev[0])
    both = TopDownPredictor(m, imodel, crop_size=32, peak_threshold=im.centroid_crop.peak_threshold, batch_size=3).inference_model
    assert both._can_fuse()
    both.predict_on_batch(frames)                                        # sb_topdown_configure on the centroid model
    refused(submit(0), "sb_topdown_submit")
    gtc = TopDownPredictor(None, imodel, crop_size=32, batch_size=3).inference_model
    gtc.predict_on_batch(dict(image=frames, centroids=[np.array([[40, 50]], F)] * 3))
    refused(L.sb_topdown_gt_instances_submit(h, imodel.model_id, _lib.ptr(frames), _lib.ptr(table), _lib.ptr(counts), 3, 0),
            "sb_topdown_gt_submit")
    refused(L.sb_topdown_gt_instances_collect(h, imodel.model_id, 0, 3, *[_lib.ptr(z)] * 2, _lib.ptr(zi), *[_lib.ptr(z)] * 2,
                                              _lib.ptr(zi), _lib.ptr(zi)), "sb_topdown_gt_submit")
    same(im.predict_on_batch(ex))                                        # the next call configures the pipeline again
    m.configure(2, 64, 64, 1)                                            # a configure call on the centroid model
    refused(submit(0), "not configured")
    same(im.predict_on_batch(ex))
