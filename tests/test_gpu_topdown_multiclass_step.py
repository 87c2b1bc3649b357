"""The top-down multi-class (identity) step on the device: after every chunk of crops the global peaks and the class-vector
head (k_class_vectors: pooled or flattened tap, Dense + ReLU layers, Dense, softmax), after the last chunk one assignment
of each frame's crops to the classes (k_td_class_assign), one record per frame.

Grouping is checked bit for bit against the host's identity.classify_peaks_from_vectors on the device's own per-crop
probabilities and the staged path's peaks; the head against a NumPy restatement of its definition (float64 products and
sums, float32 rounding at the same points); the fused pipeline against the staged path (fused = False) on synthetic
networks in all three precisions, and on the trained fixture model through the from-features entry."""
import os
from ctypes import byref

import numpy as np
import pytest
from numpy.testing import assert_allclose

import layer_audit as la
import reference_models as rm
from test_gpu_multiclass_step import assert_bit_equal

pytestmark = pytest.mark.gpu

F32 = np.float32
NODES = list("abcd")


# ------------------------------------------------------------------------------------------------ head restated
def _dense(x, kernel, bias, relu):
    """One Dense layer as the device defines it: float64 products summed in input order, + bias, rounded once to float32."""
    k = np.asarray(kernel, np.float64)
    acc = np.zeros((len(x), k.shape[1]), np.float64)
    for i in range(k.shape[0]):
        acc = acc + x[:, i:i + 1].astype(np.float64) * k[i][None]
    z = (acc + np.asarray(bias, np.float64)).astype(F32)
    return np.where(z < 0, F32(0), z) if relu else z


def head_restated(feat, head, weights):
    """(pooled features, class probabilities) of ClassVectorsHead on feature maps (N, H, W, C)."""
    feat = np.asarray(feat, F32)
    x = feat.max(axis=(1, 2)) if head.get("global_pool", True) else feat.reshape(len(feat), -1)
    pooled = x
    for i in range(int(head.get("num_fc_layers", 1))):
        p = weights[f"pre_classification{i}_fc"]
        x = _dense(x, p["kernel"], p["bias"], True)
    z = _dense(x, weights[head["name"]]["kernel"], weights[head["name"]]["bias"], False)
    e = np.exp(z.astype(np.float64) - z.max(axis=1, keepdims=True).astype(np.float64))
    s = np.zeros(len(z), np.float64)
    for j in range(z.shape[1]):
        s = s + e[:, j]
    return pooled, (e / s[:, None]).astype(F32)


def dense_weights(n_in, n_fc, units, n_classes, seed, logit_scale=4.0):
    rng = np.random.default_rng(seed)
    w, dims = {}, [n_in] + [units] * n_fc
    for i in range(n_fc):
        w[f"pre_classification{i}_fc"] = dict(kernel=(rng.normal(0, 1, (dims[i], units)) * np.sqrt(2.0 / dims[i])).astype(F32),
                                              bias=rng.normal(0, 0.1, units).astype(F32))
    w["ClassVectorsHead"] = dict(kernel=(rng.normal(0, logit_scale, (dims[-1], n_classes)) / np.sqrt(dims[-1])).astype(F32),
                                 bias=rng.normal(0, 0.1, n_classes).astype(F32))
    return w


# ------------------------------------------------------------------------------------------------ synthetic crops
def synth_crops(seed, counts, n_classes=3, n_fc=1, units=16, global_pool=True, Hf=4, Wf=4, Cf=24, offsets=False, tie=False,
                dead=False, H=16, W=16, stride=4):
    """Per crop: confidence maps with one blob per node, a random feature map, crop offsets; the crops of frame b are
    counts[b] consecutive rows.  tie: the first two crops of the largest frame share their feature map (an exact tie);
    dead: the first crop's maps stay below every threshold used here."""
    rng = np.random.default_rng(seed)
    n = int(sum(counts))
    yy, xx = np.mgrid[0:H, 0:W].astype(F32)
    cms = np.zeros((n, H, W, len(NODES)), F32)
    for i in range(n):
        for c in range(len(NODES)):
            x0, y0 = rng.uniform(2, W - 3), rng.uniform(2, H - 3)
            cms[i, :, :, c] = np.exp(-((xx - x0) ** 2 + (yy - y0) ** 2) / F32(2 * 1.5 ** 2)) * F32(rng.uniform(0.6, 1.0))
    feats = rng.normal(0, 1, (n, Hf, Wf, Cf)).astype(F32)
    sinds = np.repeat(np.arange(len(counts)), counts).astype(np.int32)
    if tie:
        b = int(np.argmax(counts))
        i0 = int(np.sum(counts[:b]))
        feats[i0 + 1] = feats[i0]
    if dead:
        cms[0] *= F32(0.05)
    head = dict(name="ClassVectorsHead", channels=n_classes, num_fc_layers=n_fc, num_fc_units=units, global_pool=global_pool)
    n_in = Cf if global_pool else Hf * Wf * Cf
    w = dense_weights(n_in, n_fc, units, n_classes, seed + 7)
    off = rng.uniform(-0.45, 0.45, (n, H, W, 2 * len(NODES))).astype(F32) if offsets else None
    co = rng.uniform(0, 300, (n, 2)).astype(F32)
    return dict(cms=cms, feats=feats, sinds=sinds, B=len(counts), head=head, weights=w, offsets=off, crop_offsets=co, stride=stride)


CASES = {
    "more_crops_than_classes": dict(counts=[5, 3, 4], n_classes=3),
    "fewer_crops_than_classes": dict(counts=[1, 2, 2], n_classes=4),
    "frame_without_crops": dict(counts=[2, 0, 3]),
    "one_class": dict(counts=[2, 1, 3], n_classes=1),
    "seven_classes": dict(counts=[4, 7, 9], n_classes=7),
    "identical_feature_maps": dict(counts=[2, 4, 3], n_classes=3, tie=True),
    "crop_below_threshold": dict(counts=[3, 2], dead=True),
    "flatten": dict(counts=[3, 4], global_pool=False, Cf=8),
    "no_fc_layers": dict(counts=[3, 4], n_fc=0),
    "three_fc_layers": dict(counts=[3, 4], n_fc=3, units=32),
    "offsets_head": dict(counts=[3, 2, 4], offsets=True),
}
REFINE = {"refine_none": None, "refine_integral": "integral", "refine_local": "local"}


def _run_case(name, refinement="local", thr=0.3):
    from sleap_b200.nn.inference import topdown_multiclass_from_features
    case = synth_crops(sum(map(ord, name)), **CASES.get(name, dict(counts=[3, 2, 4])))
    out = topdown_multiclass_from_features(case["cms"], case["feats"], case["sinds"], case["B"], case["head"], case["weights"],
                                           case["stride"], peak_threshold=thr, refinement=refinement, offsets=case["offsets"],
                                           crop_offsets=case["crop_offsets"])
    return case, out


def _staged_peaks(case, refinement, thr):
    """TopDownMultiClassFindPeaks' peaks: find_global_peaks (with offsets when given), x output stride, + crop offsets."""
    from sleap_b200.nn import peak_finding
    if case["offsets"] is not None:
        pk, pv = peak_finding.find_global_peaks_with_offsets(case["cms"], case["offsets"], threshold=thr)
    else:
        pk, pv = peak_finding.find_global_peaks(case["cms"], threshold=thr, refinement=refinement, integral_patch_size=5)
    pk = (pk * F32(case["stride"])).astype(F32)
    return (pk + case["crop_offsets"].reshape(-1, 1, 2)).astype(F32), pv


@pytest.mark.parametrize("name", list(CASES) + list(REFINE))
def test_grouping_matches_host(name):
    from sleap_b200.nn import identity
    refinement, thr = REFINE.get(name, "local"), 0.3
    case, out = _run_case(name, refinement, thr)
    pts, pv = _staged_peaks(case, refinement, thr)
    want = identity.classify_peaks_from_vectors(pts, pv, out["class_vectors"], case["sinds"], case["B"])
    assert_bit_equal(out["instance_peaks"], want[0], f"{name}: points")
    assert_bit_equal(out["instance_peak_vals"], want[1], f"{name}: point values")
    assert_bit_equal(out["instance_scores"], want[2], f"{name}: class probabilities")
    counts = np.bincount(case["sinds"], minlength=case["B"])
    assigned = np.isfinite(out["instance_scores"]).sum(1)
    assert np.all(assigned <= np.minimum(counts, case["head"]["channels"]))
    if name == "crop_below_threshold":           # its points are NaN; it still takes part in the assignment
        assert np.isnan(pts[0]).all()
    if name == "identical_feature_maps":
        b = int(np.argmax(counts))
        i0 = int(counts[:b].sum())
        assert out["class_vectors"][i0].tobytes() == out["class_vectors"][i0 + 1].tobytes()


@pytest.mark.parametrize("name", list(CASES))
def test_head_arithmetic(name):
    from sleap_b200.nn.model import class_vectors_from_features
    case, out = _run_case(name)
    pooled, probs = head_restated(case["feats"], case["head"], case["weights"])
    assert_bit_equal(out["features"], pooled, f"{name}: pooled features")
    got = out["class_vectors"]
    assert_allclose(got, probs, rtol=1e-6, atol=0)
    exact = float(np.mean(got.view(np.uint32) == probs.view(np.uint32)))
    print(f"{name}: {exact:.4f} of the probabilities bit-equal to the restatement")
    assert_allclose(got, class_vectors_from_features(case["feats"], case["head"], case["weights"]), atol=1e-5, rtol=0)


# ------------------------------------------------------------------------------------------------ fused vs staged
def _models(precision, n_fc=3, units=64, n_classes=4):
    """A synthetic centroid model (zero biases: a black frame has no centroid) and a centered-instance model with a
    ClassVectorsHead tapping stride 16."""
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    ccfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=2, middle_block=True, up_interpolate=True)
    cspec = dict(backbone="unet", backbone_cfg=ccfg, head_type="centroid", part_names=None, edges=None,
                 heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
    icfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=4, middle_block=True, up_interpolate=False)
    classes = [f"c{i}" for i in range(n_classes)]
    ispec = dict(backbone="unet", backbone_cfg=icfg, head_type="multi_class_topdown", part_names=NODES, edges=None, classes=classes,
                 heads=[dict(name="CenteredInstanceConfmapsHead", channels=len(NODES), output_stride=4),
                        dict(name="ClassVectorsHead", channels=n_classes, output_stride=16, vector=True, num_fc_layers=n_fc,
                             num_fc_units=units, global_pool=True)])
    cw = A.make_synthetic_weights(A.compile_model(cspec, 1), 61)
    icm = A.compile_model(ispec, 1)
    iw = la.synthetic_weights(icm, 63)
    iw.update(dense_weights(icm.vector_taps["ClassVectorsHead"]["C"], n_fc, units, n_classes, 65, logit_scale=8.0))
    return DeviceModel(cspec, cw, input_channels=1, precision=precision), DeviceModel(ispec, iw, input_channels=1, precision=precision)


@pytest.fixture(scope="module")
def frames():
    imgs = np.random.default_rng(9).integers(0, 256, size=(4, 192, 224, 1), dtype=np.uint8)
    imgs[1] = 0                                      # no centroid in this frame
    return imgs


def _predictor(precision, frames, max_instances=None, max_crops_per_call=64):
    from sleap_b200.nn.inference import TopDownMultiClassPredictor
    cmodel, imodel = _models(precision)
    cms = cmodel.forward(frames)[0]
    thr = max(float(np.quantile(cms, 0.99)), 1e-3)
    pred = TopDownMultiClassPredictor(cmodel, imodel, crop_size=64, peak_threshold=thr, integral_refinement=True,
                                      batch_size=len(frames), max_instances=max_instances)
    pred.inference_model.instance_peaks.peak_threshold = 0.0
    pred.inference_model.instance_peaks.max_crops_per_call = max_crops_per_call
    return pred


def _both(im, frames):
    assert im._can_fuse()
    fused = im.predict_on_batch(frames)
    im.fused = False
    staged = im.predict_on_batch(frames)
    im.fused = True
    return fused, staged


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("max_instances,chunk", [(None, 64), (3, 64), (None, 3)])
def test_fused_matches_staged(precision, max_instances, chunk, frames):
    im = _predictor(precision, frames, max_instances, chunk).inference_model
    im.instance_peaks.return_class_vectors = True
    fused, staged = _both(im, frames)
    for k in ("centroids", "centroid_vals"):
        assert_bit_equal(fused[k], staged[k], k)
    n_crops = np.isfinite(fused["centroid_vals"]).sum(1)
    assert n_crops[1] == 0 and n_crops.sum() > len(frames), n_crops
    if chunk < 64:
        assert n_crops.sum() > chunk
    assert len(fused["class_vectors"]) == n_crops.sum()
    assert np.array_equal(np.isnan(fused["instance_scores"]), np.isnan(staged["instance_scores"])), "class assignments differ"
    assert_bit_equal(fused["instance_peaks"], staged["instance_peaks"], "points")
    assert_bit_equal(fused["instance_peak_vals"], staged["instance_peak_vals"], "point values")
    assert_allclose(fused["instance_scores"], staged["instance_scores"], atol=1e-5, rtol=0)
    assert np.array_equal(fused["flags"], im.centroid_crop.call(dict(image=frames))["flags"])


def test_batch_independence(frames):
    imgs = np.concatenate([frames, frames[::-1]])
    im = _predictor(0, imgs, 3).inference_model
    batch = im.predict_on_batch(imgs)
    for i in range(len(imgs)):
        one = im.predict_on_batch(imgs[i:i + 1])
        for k in ("instance_peaks", "instance_peak_vals", "instance_scores", "flags"):
            assert one[k][0].tobytes() == batch[k][i].tobytes(), (i, k)
        for k in ("centroids", "centroid_vals"):
            n = one[k].shape[1]
            assert one[k][0].tobytes() == batch[k][i, :n].tobytes() and np.isnan(batch[k][i, n:]).all(), (i, k)


# ------------------------------------------------------------------------------------------------ trained fixture
def _maps_and_features(m, crops):
    """Confidence maps and the ClassVectorsHead tap of a device forward, the tap read as DeviceModel._class_vectors reads it."""
    tap, raw = m.cm.vector_taps["ClassVectorsHead"], {}
    m._class_vectors = lambda buf, name: raw.setdefault(name, buf)
    try:
        cms = m.forward(crops, ["CenteredInstanceConfmapsHead", "ClassVectorsHead"])[0]
    finally:
        del m._class_vectors
    buf, c0, C = raw["ClassVectorsHead"], tap["coff"], tap["C"]
    return cms, (buf[..., c0:c0 + C] + buf[..., c0 + C:c0 + 2 * C]) if tap["planes"] == 3 else buf[..., c0:c0 + C]


@pytest.mark.parametrize("precision", [1, 0, 2])
def test_trained_fixture(precision):
    from oracle import inference as oinf
    from sleap_b200.nn.inference import Predictor, topdown_multiclass_from_features
    from sleap_b200.nn.model import head_spec
    z = np.load(os.path.join(rm.GOLDEN, "frames_tracks_2node.npz"))
    gt, names = z["points_gt"][0], [str(n) for n in z["track_names"][0]]
    d = rm.model_dir("min_tracks_2node.topdown_multiclass")
    m = Predictor.from_model_paths([d], precision=precision).confmap_model
    cfg, _, _, _ = rm.load_fixture_model("min_tracks_2node.topdown_multiclass")
    cc = oinf.centroid_crop_ground_truth_layer(z["images"], [gt[:, 1, :]], cfg["data"]["instance_cropping"]["crop_size"], 1.0)
    cms, feat = _maps_and_features(m, np.ascontiguousarray(cc["crops"]))
    sinds = np.zeros(len(feat), np.int32)
    kw = dict(refinement="local", crop_offsets=cc["crop_offsets"])
    head = head_spec(m.spec, "ClassVectorsHead")
    out = topdown_multiclass_from_features(cms, feat, sinds, 1, head, m.dense_weights, m.cm.head_strides["CenteredInstanceConfmapsHead"],
                                           peak_threshold=0.7, **kw)
    classes = m.spec["classes"]
    assert sorted(classes) == sorted(names)
    for j, c in enumerate(classes):
        assert_allclose(out["instance_peaks"][0, j], gt[names.index(c)], rtol=0.02)
        assert out["instance_scores"][0, j] > 0.99
    _, probs = head_restated(feat, head, m.dense_weights)
    assert_allclose(out["class_vectors"], probs, rtol=1e-6, atol=0)
    hi = topdown_multiclass_from_features(cms, feat, sinds, 1, head, m.dense_weights, m.cm.head_strides["CenteredInstanceConfmapsHead"],
                                          peak_threshold=1.5, **kw)
    assert np.isnan(hi["instance_peaks"]).all()


# ------------------------------------------------------------------------------------------------ errors
def test_refusals_keep_the_pipeline(frames):
    from sleap_b200._lib import MAX_CLASSES, SleapB200Error
    from sleap_b200.nn.inference import FindInstancePeaks, TopDownInferenceModel, _topdown_params, topdown_multiclass_params
    pred = _predictor(0, frames, 3)
    im = pred.inference_model
    cc, fp = im.centroid_crop, im.instance_peaks
    mc, mi = cc.keras_model, fp.keras_model
    first = im.predict_on_batch(frames)

    def same():
        again = im.predict_on_batch(frames)
        for k in first:
            assert first[k].tobytes() == again[k].tobytes(), k

    td, _ = _topdown_params(cc, fp)
    shape = frames.shape
    for bad in (dict(n_classes=MAX_CLASSES + 1), dict(tap_buffer=-1), dict(tap_planes=2)):
        p = topdown_multiclass_params(td, mi.cm.vector_taps["ClassVectorsHead"], fp.class_head, fp.dense)
        for k, v in bad.items():
            setattr(p, k, v)
        with pytest.raises(SleapB200Error):
            mc.handle.call("sb_topdown_multiclass_configure", byref(p), *shape)
        same()
    z = np.zeros(64, np.float32)
    with pytest.raises(SleapB200Error, match="is multi-class"):
        mc.handle.call("sb_infer_topdown", mc.model_id, frames.ctypes.data, 1, len(frames), *([z.ctypes.data] * 6))
    same()
    plain = TopDownInferenceModel(cc, FindInstancePeaks(mi, peak_threshold=0.0))
    plain.predict_on_batch(frames)
    with pytest.raises(SleapB200Error, match="not multi-class"):
        mc.handle.call("sb_infer_topdown_multiclass", mc.model_id, frames.ctypes.data, 1, len(frames), *([z.ctypes.data] * 7), None)
    same()                                          # the Python record reconfigures the multi-class pipeline
    # behind the Python record: the instance model's chain moves on; the centroid model's drops the pipeline it holds
    for m, fn, p, msg in ((mi, "sb_global_configure", fp.params(), "a model was reconfigured; call sb_topdown_multiclass_configure again"),
                          (mc, "sb_centroid_configure", cc.params(), "top-down pipeline not configured")):
        m.handle.call(fn, m.model_id, byref(p))
        with pytest.raises(SleapB200Error, match=msg):
            im.predict_on_batch(frames)
        mc.chain = mi.chain = None
        same()


# ------------------------------------------------------------------------------------------------ end to end
def test_predictor_fused_and_staged(frames):
    pred = _predictor(1, frames)
    fused = pred.predict(frames)
    pred.inference_model.fused = False
    staged = pred.predict(frames)
    assert len(fused) == len(staged) == len(frames)
    assert sum(len(f.instances) for f in fused) > 0
    for a, b in zip(fused, staged):
        assert a.frame_idx == b.frame_idx and len(a.instances) == len(b.instances)
        for x, y in zip(a.instances, b.instances):
            assert x.track.name == y.track.name
            assert x.numpy().tobytes() == y.numpy().tobytes()
            assert x.score == y.score
            assert abs(x.tracking_score - y.tracking_score) <= 1e-5
