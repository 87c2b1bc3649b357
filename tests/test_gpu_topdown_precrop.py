"""Top-down models whose centered-instance network was trained at an input scale s != 1, on the fused, streamed step.

CentroidCrop with precrop_resize = s resizes the full frames by s (resize_image: bilinear, half-pixel centres, cast back
to the frame dtype), multiplies the centroids by s and crops the resized frames; the instance peaks come back through
/ s + 0.5 and + crop offset / s.  The fused step does the same without storing the resized frames:
sb_crop_centered_resized (k_crop on resized texels computed on the fly) must equal FrameResizer + sb_crop_centered byte
for byte, and the fused, streamed and tracked routes must equal the staged route (fused = False) bit for bit."""
from ctypes import byref
from functools import lru_cache

import numpy as np
import pytest
from numpy.testing import assert_allclose, assert_array_equal

import reference_models as rm
from oracle import convnet, peak_finding as opf, preprocess as opre, tf_ops
from sleap_b200 import _lib
from sleap_b200.nn import tracking as T
from test_gpu_predict_pipeline import assert_same_batches, check_stream, frames_summary, variants
from test_gpu_reference_models import _matched
from test_gpu_topdown_track import CONFIGS
from track_cases import _close

pytestmark = pytest.mark.gpu

F = np.float32
NODES = list("abcd")
CROP = 64
SB_ERR_INVALID, SB_ERR_UNSUPPORTED = -1, -3


# ------------------------------------------------------------------------------------------------ the crop kernel
def _crop(imgs, cent, sinds, crop, scale=None):
    """sb_crop_centered_resized (scale given) or sb_crop_centered of host frames."""
    h = _lib.default_handle()
    B, H, W, C = imgs.shape
    out = np.zeros((len(cent), crop, crop, C), imgs.dtype)
    args = (_lib.ptr(imgs), int(imgs.dtype == np.uint8), B, H, W, C, _lib.ptr(_lib.f32(cent)), _lib.ptr(_lib.i32(sinds)), len(cent),
            crop, crop)
    if scale is None:
        h.call("sb_crop_centered", *args, _lib.ptr(out))
    else:
        h.call("sb_crop_centered_resized", *args, float(scale), _lib.ptr(out))
    return out


def _edge_centroids(Hr, Wr, crop):
    """Centroids in resized-frame coordinates: inside, on each edge and corner, hanging off every side, and wholly
    outside; fractional and whole."""
    c = crop / 2
    pts = [(Wr / 2 + 0.3, Hr / 2 - 0.6), (Wr / 3, Hr / 4), (0, 0), (Wr - 1, Hr - 1), (0, Hr / 2), (Wr - 1, Hr / 3),
           (Wr / 2, 0), (Wr / 3, Hr - 1), (-c + 3.2, Hr / 2), (Wr + c - 4.5, Hr / 3), (Wr / 3, -c + 2.7), (Wr / 4, Hr + c - 6.1),
           (-c - 10, Hr + c + 10), (Wr + 7.25, -3.5)]
    return np.asarray(pts, F)


@pytest.mark.parametrize("hw", [(250, 198), (97, 131)])
@pytest.mark.parametrize("C", [1, 3])
@pytest.mark.parametrize("dtype", [np.uint8, np.float32])
def test_crop_resized_equals_resize_then_crop(dtype, C, hw):
    from sleap_b200.nn.model import FrameResizer
    rng = np.random.default_rng(hash((hw, C)) % 2 ** 32)
    imgs = rng.integers(0, 256, size=(2,) + hw + (C,), dtype=np.uint8)
    if dtype == np.float32:
        imgs = (imgs.astype(F) / F(255) + rng.normal(0, 0.01, imgs.shape).astype(F)).astype(F)
    resizer = FrameResizer(_lib.default_handle())
    worst = 0.0
    for scale in (0.5, 0.75, 0.3):
        resized = resizer(imgs, scale)
        Hr, Wr = resized.shape[1:3]
        assert (Hr, Wr) == (int(F(hw[0]) * F(scale)), int(F(hw[1]) * F(scale)))
        for crop in (56, 65):
            pts = _edge_centroids(Hr, Wr, crop)
            cent = np.concatenate([pts, pts[::-1] + F(0.125)])
            sinds = np.repeat(np.arange(2, dtype=np.int32), len(pts))
            got = _crop(imgs, cent, sinds, crop, scale)
            want = _crop(resized, cent, sinds, crop)
            assert got.dtype == want.dtype and got.tobytes() == want.tobytes(), (scale, crop)
            assert got.any()
            oracle = tf_ops.crop_bboxes(opre.resize_image(imgs, scale), tf_ops.make_centered_bboxes(cent, crop, crop), sinds)
            worst = max(worst, float(np.abs(got.astype(np.float64) - oracle.astype(np.float64)).max()))
    print(f"sb_crop_centered_resized vs oracle resize_image + crop_bboxes ({np.dtype(dtype).name}, C={C}, {hw}): "
          f"largest difference {worst}")
    assert worst == 0.0                  # the resize and the crop round every float32 step as the oracle does


def test_crop_resized_refusals():
    h = _lib.default_handle()
    imgs = np.zeros((1, 40, 30, 1), np.uint8)
    out = np.zeros((1, 8, 8, 1), np.uint8)
    cent, sinds = np.zeros((1, 2), F), np.zeros(1, np.int32)
    for bad in (-0.5, 0.0, float("nan"), float("inf"), 0.02):          # 0.02: a 0 x 0 frame
        rc = _lib.lib().sb_crop_centered_resized(h.h, _lib.ptr(imgs), 1, 1, 40, 30, 1, _lib.ptr(cent), _lib.ptr(sinds), 1, 8, 8,
                                                 bad, _lib.ptr(out))
        assert rc == SB_ERR_INVALID, bad


# ------------------------------------------------------------------------------------------------ synthetic scaled pair
@lru_cache(maxsize=None)
def _models(precision):
    """The centroid / centered-instance UNet pair of the top-down tracker tests in one precision: centroid model at input
    scale 0.5, instance model built without a resize op (its trained scale is set per test as config_input_scale)."""
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    ccfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=2, middle_block=True, up_interpolate=True)
    cspec = dict(backbone="unet", backbone_cfg=ccfg, head_type="centroid", part_names=None, edges=None,
                 heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
    icfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=4, middle_block=True, up_interpolate=False)
    ispec = dict(backbone="unet", backbone_cfg=icfg, head_type="centered_instance", part_names=NODES, edges=None,
                 heads=[dict(name="CenteredInstanceConfmapsHead", channels=len(NODES), output_stride=4)])
    cw = A.make_synthetic_weights(A.compile_model(cspec, 1, 0.5), 41)
    iw = A.make_synthetic_weights(A.compile_model(ispec, 1), 43)
    cmodel = DeviceModel(cspec, cw, input_channels=1, input_scale=0.5, precision=precision)
    imodel = DeviceModel(ispec, iw, input_channels=1, precision=precision)
    return cmodel, imodel, ispec, iw


@pytest.fixture(scope="module")
def clip():
    """Gray clip frames with an all-black stretch (frames 12-15: no centroid), and the centroid threshold: the median over
    frames of the 5th-highest local maximum of the centroid map."""
    from scipy.ndimage import maximum_filter
    from flow_clip import clip_frames
    gray = np.ascontiguousarray(clip_frames(21)[:, :, :, :1])
    gray = np.ascontiguousarray(np.concatenate([gray[:12], np.zeros((4,) + gray.shape[1:], np.uint8), gray[12:]]))
    cmodel = _models(1)[0]
    cms = np.concatenate([cmodel.forward(gray[i:i + 5])[0] for i in range(0, 10, 5)])[..., 0]
    fifth = []
    for c in cms:
        v = np.sort(c[c == maximum_filter(c, size=3, mode="constant", cval=-np.inf)])[::-1]
        fifth.append(v[min(4, len(v) - 1)])
    return gray, float(np.median(fifth))


def _predictor(precision, scale, thr, bs, max_instances=None, chunk=64):
    from sleap_b200.nn.inference import TopDownPredictor
    cmodel, imodel, _, _ = _models(precision)
    imodel.config_input_scale = scale
    pred = TopDownPredictor(cmodel, imodel, crop_size=CROP, peak_threshold=thr, integral_refinement=True, batch_size=bs,
                            max_instances=max_instances)
    im = pred.inference_model
    im.instance_peaks.peak_threshold = 0.05
    im.instance_peaks.max_crops_per_call = chunk
    assert im.centroid_crop.precrop_resize == scale and im.instance_peaks.input_scale == scale
    assert im._can_fuse()
    return pred


KEYS = ("centroids", "centroid_vals", "instance_peaks", "instance_peak_vals")


def _fused_and_staged(im, frames):
    im.fused = True
    a = im.predict_on_batch(frames)
    im.fused = False
    b = im.predict_on_batch(frames)
    im.fused = True
    assert_array_equal(a["n_valid"], b["n_valid"])
    for k in KEYS:
        assert a[k].shape == b[k].shape, k
        assert_array_equal(a[k], b[k], err_msg=k)
    return a


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("scale", [0.5, 0.75])
def test_fused_equals_staged(clip, precision, scale):
    gray, thr = clip
    frames = np.ascontiguousarray(np.concatenate([gray[:6], gray[12:14]]))       # 8 frames, the last two black
    for max_instances, chunk in ((None, 64), (1, 64), (3, 64), (None, 5)):
        im = _predictor(precision, scale, thr, 8, max_instances, chunk).inference_model
        for x in (frames, frames.astype(F) / F(255)):
            out = _fused_and_staged(im, x)
            n = out["n_valid"]
            assert n[-2:].sum() == 0 and n[:6].sum() >= 6
            if max_instances is not None:
                assert n.max() <= max_instances
            if chunk < 64:
                assert n.sum() > chunk                                           # several instance chunks
            assert np.isfinite(out["instance_peaks"][:6]).any()


@pytest.mark.parametrize("scale", [0.5, 0.75])
def test_fused_matches_oracle(clip, scale):
    """The fused step at precision 1 against the oracle chain on the device's centroid maps: oracle local peaks, top-k,
    centroids * s, oracle resize_image + crop_bboxes, the oracle network on those crops (the device's maps on them give
    the peaks), / s + 0.5 and + crop offset / s."""
    gray, thr = clip
    imgs = np.ascontiguousarray(gray[:4])
    cmodel, imodel, ispec, iw = _models(1)
    out = _predictor(1, scale, thr, 4, max_instances=3).inference_model.predict_on_batch(imgs)
    cp, cv, csi, _ = opf.find_local_peaks(cmodel.forward(imgs)[0], thr, "integral", 5)
    cp = ((cp * F(2)).astype(F) / F(0.5) + F(0.5)).astype(F)
    keep = []
    for s in range(len(imgs)):
        idx = np.nonzero(csi == s)[0]
        if len(idx) > 3:
            idx = idx[np.argsort(-cv[idx], kind="stable")[:3]]
        keep.append(idx)
    keep = np.concatenate(keep)
    cp, cv, csi = (cp[keep] * F(scale)).astype(F), cv[keep], csi[keep]
    assert len(cp) > 0
    crops = tf_ops.crop_bboxes(opre.resize_image(imgs, scale), tf_ops.make_centered_bboxes(cp, CROP, CROP), csi)
    icms = convnet.model_forward(opre.preprocess(crops, True, 1.0, 16), ispec, iw)[0]
    dcms = imodel.forward(crops)[0]
    assert_allclose(dcms, icms, atol=1e-4 * max(1, np.abs(icms).max()), rtol=1e-4)
    wp, wv = opf.find_global_peaks(dcms, 0.05, "integral", 5)
    wp = ((wp * F(4)).astype(F) / F(scale) + F(0.5)).astype(F)
    wp = (wp + ((cp - F(CROP / 2)) / F(scale)).astype(F)[:, None, :]).astype(F)
    for s in range(len(imgs)):
        n = int(out["n_valid"][s])
        assert n == int((csi == s).sum())
        assert_allclose(out["centroids"][s, :n], cp[csi == s], atol=1e-4)
        assert_allclose(out["centroid_vals"][s, :n], cv[csi == s], atol=1e-6)
        assert_allclose(out["instance_peaks"][s, :n], wp[csi == s], atol=1e-3, equal_nan=True)
        assert_allclose(out["instance_peak_vals"][s, :n], wv[csi == s], atol=1e-6, equal_nan=True)


def test_stream_equals_per_batch(clip):
    gray, thr = clip
    for max_instances, chunk in ((None, 64), (3, 5)):
        im = _predictor(1, 0.5, thr, 4, max_instances, chunk).inference_model
        got = check_stream(im, gray, 4)                   # 25 frames: 7 batches, the last of 1; batch 3 all black
        assert got[3]["n_valid"].sum() == 0 and got[3]["instance_peaks"].shape[1] == 0
        assert sum(int(g["n_valid"].sum()) for g in got) > 30
        check_stream(im, gray[:6], 1)                     # B = 1


def test_tracker_in_stream_equals_staged(clip, monkeypatch):
    """TopDownPredictor.predict with a device tracker: the fused, streamed route (the tracker inside the step) gives the
    staged route's instances, tracks and tracking scores, and the host tracker never runs on it."""
    gray, thr = clip

    def no_host_track(*a, **k):
        raise AssertionError("Tracker.track called on the fused route")

    for name in ("simple/instance/greedy", "simplemaxtracks/centroid/hungarian"):
        kw = CONFIGS[name]
        pred = _predictor(1, 0.5, thr, 4)
        with monkeypatch.context() as mp:
            mp.setattr(T.Tracker, "track", no_host_track)
            tr_f = pred.tracker = T.Tracker.make_tracker_by_name(track_device=0, **kw)
            fused = pred.predict(gray)
        pred.inference_model.fused = False
        tr_s = pred.tracker = T.Tracker.make_tracker_by_name(track_device=0, **kw)
        staged = pred.predict(gray)
        assert sum(len(lf.instances) for lf in fused) > 20, name
        assert len(tr_f.spawned_tracks) > 1, name
        assert frames_summary(fused) == frames_summary(staged), name
        for fa, fb in zip(fused, staged):
            for xa, xb in zip(fa.instances, fb.instances):
                assert _close(float(xa.tracking_score), float(xb.tracking_score)), name
        assert [(t.name, t.spawned_on) for t in tr_f.spawned_tracks] == [(t.name, t.spawned_on) for t in tr_s.spawned_tracks]


def test_batch_independence(clip):
    gray, thr = clip
    frames = np.ascontiguousarray(gray[10:18])                    # two black frames among them
    im = _predictor(1, 0.5, thr, 8).inference_model
    full = im.predict_on_batch(frames)
    for i in range(len(frames)):
        one = im.predict_on_batch(frames[i:i + 1])
        n = int(one["n_valid"][0])
        assert int(full["n_valid"][i]) == n and full["flags"][i] == one["flags"][0]
        for k in KEYS:
            assert full[k][i, :n].tobytes() == one[k][0, :n].tobytes(), (i, k)
            assert np.isnan(full[k][i, n:]).all(), (i, k)


# ------------------------------------------------------------------------------------------------ trained fixture
@pytest.mark.parametrize("precision", [0, 1, 2])
def test_trained_scaled_instance_model(precision):
    """minimal_instance.centroid + minimal_instance.centered_instance_with_scaling (input scaling 0.5, crop 56): fused equals
    staged, the stream equals the per-batch loop, and the reference's assertions hold (two instances within 2 px)."""
    from sleap_b200.nn.inference import Predictor
    imgs, gt4 = rm.frames("minimal_instance")
    paths = [rm.model_dir("minimal_instance.centroid"), rm.model_dir("minimal_instance.centered_instance_with_scaling")]
    pred = Predictor.from_model_paths(paths, precision=precision, batch_size=2)
    im = pred.inference_model
    assert im.centroid_crop.precrop_resize == 0.5 and im.centroid_crop.crop_size == 56
    assert im._can_fuse()
    frames = np.ascontiguousarray(np.concatenate([imgs, variants(imgs[0], 3), np.zeros_like(imgs)]))    # 5 frames
    out = _fused_and_staged(im, frames)
    assert out["n_valid"][0] >= 2 and out["n_valid"][-1] == 0
    for bs in (2, 1):
        check_stream(im, frames, bs)
    got = pred.predict(imgs)
    assert len(got) == 1 and len(got[0].instances) == 2
    _matched(gt4[0].reshape(-1, 2), np.concatenate([x.numpy() for x in got[0].instances]), 2.0)


# ------------------------------------------------------------------------------------------------ refusals
def test_configure_refusals(clip):
    """A pre-crop resize that is negative, NaN, infinite or that leaves no frame is SB_ERR_INVALID, and the pipeline
    configured before stays usable."""
    from sleap_b200.nn.inference import _topdown_params
    gray, thr = clip
    im = _predictor(1, 0.5, thr, 4).inference_model
    want = im.predict_on_batch(gray[:4])
    cc, fp = im.centroid_crop, im.instance_peaks
    h = cc.keras_model.handle
    H, W, C = gray.shape[1:]
    for bad in (-1.0, float("nan"), float("inf"), 5e-4):              # 5e-4: a 0 x 0 frame
        p, _ = _topdown_params(cc, fp)
        p.precrop_resize = bad
        assert _lib.lib().sb_topdown_configure(h.h, byref(p), 4, H, W, C) == SB_ERR_INVALID, bad
        assert b"precrop_resize" in _lib.lib().sb_last_error(h.h)
        assert_same_batches([im.predict_on_batch(gray[:4])], [want])


def test_multiclass_refuses_precrop_resize():
    from sleap_b200.nn.inference import _topdown_params, topdown_multiclass_params
    from test_gpu_topdown_multiclass_step import _predictor as mc_predictor
    frames = np.random.default_rng(9).integers(0, 256, size=(2, 192, 224, 1), dtype=np.uint8)
    im = mc_predictor(1, frames).inference_model
    want = im.predict_on_batch(frames)
    cc, fp = im.centroid_crop, im.instance_peaks
    td, _ = _topdown_params(cc, fp)
    td.precrop_resize = 0.5
    p = topdown_multiclass_params(td, fp.keras_model.cm.vector_taps[fp.CLASS_VECTORS], fp.class_head, fp.dense)
    h = cc.keras_model.handle
    assert _lib.lib().sb_topdown_multiclass_configure(h.h, byref(p), 2, 192, 224, 1) == SB_ERR_UNSUPPORTED
    assert_same_batches([im.predict_on_batch(frames)], [want])
