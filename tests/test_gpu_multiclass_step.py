"""The bottom-up multi-class (identity) step on the device: local peaks, then k_class_group (class-map sampling, sigmoid,
per-node SciPy assignment of peaks to classes, keep rule), one record per frame.

The reference is the host chain the library ran before this step existed, composed from public calls: peaks from
sb_find_local_peaks (pinned bit-exact to the oracle), x cm_stride / class stride, probabilities from
identity.class_probabilities on the same logits, identity.classify_peaks_from_maps, x class stride (/ input_scale + 0.5).
Against it points, point values and class probabilities are bit-exact and the NaN pattern identical.  Against the CPU
oracle's peak finder the assignments are identical and the coordinates within 1e-4 px."""
import os
from ctypes import byref, c_void_p

import numpy as np
import pytest

import reference_models as rm
from oracle import peak_finding as opf
from oracle import synth

pytestmark = pytest.mark.gpu

F32 = np.float32
FIXTURE = "min_tracks_2node.bottomup_multiclass"


# ------------------------------------------------------------------------------------------------ host chain
def _truncate(peaks, vals, si, ci, max_peaks, max_node_peaks):
    """What the device keeps: the first max_peaks peaks of a frame, then the first max_node_peaks of each node (tf.where
    order throughout)."""
    keep = np.zeros(len(peaks), bool)
    for s in np.unique(si):
        idx = np.flatnonzero(si == s)[:max_peaks]
        for c in np.unique(ci[idx]):
            keep[idx[ci[idx] == c][:max_node_peaks]] = True
    return peaks[keep], vals[keep], si[keep], ci[keep]


def host_chain(cms, logits, cm_stride, cs, thr=0.2, refinement="integral", patch=5, offsets=None, input_scale=1.0,
               max_peaks=1024, max_node_peaks=32, peaks_fn=None):
    """The parent commit's host chain on the given maps.  peaks_fn: the peak finder (default: the device's)."""
    from sleap_b200.nn import identity, peak_finding
    if peaks_fn is None:
        if offsets is None:
            peaks_fn = lambda: peak_finding.find_local_peaks(cms, threshold=thr, refinement=refinement, integral_patch_size=patch)
        else:
            peaks_fn = lambda: peak_finding.find_local_peaks_with_offsets(cms, offsets, threshold=thr)
    peaks, vals, si, ci = peaks_fn()
    peaks, vals, si, ci = _truncate(np.asarray(peaks, F32).reshape(-1, 2), vals, si, ci, max_peaks, max_node_peaks)
    peaks = (peaks * F32(cm_stride)).astype(F32)
    peaks = (peaks / F32(cs)).astype(F32)
    B = cms.shape[0]
    probs = identity.class_probabilities(logits)
    pts, pv, cp = identity.classify_peaks_from_maps(probs, peaks, vals, si, ci, n_channels=cms.shape[3])
    assert pts.shape[0] == B
    pts = (pts * F32(cs)).astype(F32)
    if input_scale != 1.0:
        pts = (pts / F32(input_scale) + F32(0.5)).astype(F32)
    return pts, pv, cp


def assert_bit_equal(got, want, what):
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    gn, wn = np.isnan(got), np.isnan(want)
    assert np.array_equal(gn, wn), f"{what}: NaN pattern differs at {np.argwhere(gn != wn)[:4].tolist()}"
    g, w = got[~gn].view(np.uint32), want[~wn].view(np.uint32)
    bad = np.flatnonzero(g != w)
    assert bad.size == 0, f"{what}: {bad.size} values differ, e.g. {got[~gn][bad[0]]!r} vs {want[~wn][bad[0]]!r}"


def assert_same_as_host(out, want, what):
    assert_bit_equal(out["instance_peaks"], want[0], f"{what}: points")
    assert_bit_equal(out["instance_peak_vals"], want[1], f"{what}: point values")
    assert_bit_equal(out["instance_scores"], want[2], f"{what}: class probabilities")


# ------------------------------------------------------------------------------------------------ synthetic maps
def synth_maps(seed, B=3, H=48, W=64, n_nodes=3, n_classes=3, n_animals=3, cm_stride=2, cs=2, tie=False, empty_node=None,
               edge_x=False, offsets=False):
    """Confidence maps (B,H,W,n_nodes) at cm_stride and class-map logits (B,Hc,Wc,n_classes) at cs over an image of
    (H*cm_stride, W*cm_stride): animal a carries class a % n_classes, its logit blob rises around each of its nodes."""
    rng = np.random.default_rng(seed)
    Himg, Wimg = H * cm_stride, W * cm_stride
    Hc, Wc = Himg // cs, Wimg // cs
    xv, yv = synth.make_grid_vectors(Himg, Wimg, cm_stride)
    xc, yc = synth.make_grid_vectors(Himg, Wimg, cs)
    cms = np.zeros((B, H, W, n_nodes), F32)
    logits = np.full((B, Hc, Wc, n_classes), -3.0, F32)
    for b in range(B):
        inst = np.stack([np.stack([rng.uniform(6, Wimg - 6, n_nodes), rng.uniform(6, Himg - 6, n_nodes)], -1)
                         for _ in range(n_animals)]).astype(F32)
        if edge_x:                       # a node on the last map column: its class cell rounds onto Wc
            inst[0, 0, 0] = F32((W - 1) * cm_stride)
        cms[b] = synth.make_multi_confmaps(inst, xv, yv, sigma=1.5 * cm_stride)
        if edge_x:                       # make_multi_confmaps leaves out an animal on the image's last grid column
            cms[b] = np.maximum(cms[b], synth.make_confmaps(inst[0], xv, yv, 1.5 * cm_stride))
        for a in range(n_animals):
            g = np.zeros((Hc, Wc), F32)
            for p in inst[a]:
                g = np.maximum(g, np.exp(-((xc[None] - p[0]) ** 2 + (yc[:, None] - p[1]) ** 2) / F32(2 * (4.0 * cs) ** 2)))
            logits[b, :, :, a % n_classes] += F32(7.0) * g.astype(F32) + F32(rng.normal(0, 0.3))
        if empty_node is not None:
            cms[b, :, :, empty_node] = 0
    if tie:
        logits[..., 1] = logits[..., 0]
    off = rng.uniform(-0.45, 0.45, size=(B, H, W, 2 * n_nodes)).astype(F32) if offsets else None
    return cms, logits, off


CASES = {
    "same_stride": dict(maps=dict(cm_stride=2, cs=2)),
    "cm2_class4": dict(maps=dict(cm_stride=2, cs=4)),
    "class_cell_on_edge": dict(maps=dict(cm_stride=2, cs=4, edge_x=True), refinement=None),
    "more_animals_than_classes": dict(maps=dict(n_animals=5, n_classes=2)),
    "fewer_animals_than_classes": dict(maps=dict(n_animals=1, n_classes=4)),
    "tied_classes": dict(maps=dict(n_classes=3, tie=True)),
    "node_without_peaks": dict(maps=dict(empty_node=1)),
    "offsets": dict(maps=dict(offsets=True)),
    "refine_none": dict(maps=dict(), refinement=None),
    "refine_local": dict(maps=dict(), refinement="local"),
    "input_scale_half": dict(maps=dict(cm_stride=4, cs=2), input_scale=0.5),
    "node_over_cap": dict(maps=dict(n_animals=5, n_classes=5), max_node_peaks=3, flag=2),
    "frame_over_cap": dict(maps=dict(n_animals=5, n_classes=5), max_peaks=7, flag=1),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_from_maps_synthetic(case):
    from sleap_b200.nn.inference import bottomup_multiclass_from_maps
    cfg = CASES[case]
    mk = dict(cfg["maps"])
    cm_stride, cs = mk.get("cm_stride", 2), mk.get("cs", 2)
    cms, logits, off = synth_maps(11 + len(case), **mk)
    ref = cfg.get("refinement", "integral")
    isc = cfg.get("input_scale", 1.0)
    mp, mnp = cfg.get("max_peaks", 1024), cfg.get("max_node_peaks", 32)
    out = bottomup_multiclass_from_maps(cms, logits, cm_stride, cs, 0.2, ref, 5, offsets=off, input_scale=isc,
                                        max_peaks_per_sample=mp, max_node_peaks=mnp)
    want = host_chain(cms, logits, cm_stride, cs, 0.2, ref, 5, offsets=off, input_scale=isc, max_peaks=mp, max_node_peaks=mnp)
    assert_same_as_host(out, want, case)
    assert np.isfinite(out["instance_peaks"]).any(), "the case assigns nothing"
    if "flag" in cfg:
        assert (out["flags"] & cfg["flag"]).any(), out["flags"]
    else:
        assert not out["flags"].any(), out["flags"]
    if case == "class_cell_on_edge":
        # the last-column peak reads probability 0 for every class and is still kept (0 is its best)
        assert (out["instance_scores"] == 0).any()
    if case == "tied_classes":
        assert np.isfinite(out["instance_scores"]).any()
    if case == "node_without_peaks":
        assert np.isnan(out["instance_peaks"][:, :, 1]).all()
    # the CPU oracle's peak finder: assignments identical, coordinates within 1e-4 px
    if off is None:
        pf = lambda: opf.find_local_peaks(cms, 0.2, ref, 5)
    else:
        pf = lambda: opf.find_local_peaks_with_offsets(cms, off, 0.2)
    o = host_chain(cms, logits, cm_stride, cs, 0.2, ref, 5, offsets=off, input_scale=isc, max_peaks=mp, max_node_peaks=mnp,
                   peaks_fn=pf)
    assert np.array_equal(np.isnan(out["instance_peaks"]), np.isnan(o[0]))
    np.testing.assert_allclose(out["instance_peaks"], o[0], atol=1e-4, equal_nan=True)
    assert_bit_equal(out["instance_peak_vals"], o[1], f"{case}: oracle point values")


# ------------------------------------------------------------------------------------------------ trained fixture model
def _predictor(precision, **kw):
    from sleap_b200.nn.inference import BottomUpMultiClassPredictor, Predictor
    pred = Predictor.from_model_paths([rm.model_dir(FIXTURE)], precision=precision, **kw)
    assert isinstance(pred, BottomUpMultiClassPredictor)
    return pred


def _device_host_chain(layer, imgs):
    m = layer.keras_model
    names = [layer.CMS, layer.CLASS_MAPS] + ([layer.OFFSETS] if layer.has_offsets else [])
    outs = m.forward(layer._prep(imgs), names)
    return host_chain(outs[0], outs[1], layer.cm_output_stride, layer.class_maps_output_stride, layer.peak_threshold,
                      layer.refinement, layer.integral_patch_size, offsets=outs[2] if layer.has_offsets else None,
                      input_scale=layer.input_scale, max_peaks=layer.max_peaks_per_sample, max_node_peaks=layer.max_node_peaks)


def _tracks_frames():
    return np.load(os.path.join(rm.GOLDEN, "frames_tracks_2node.npz"))["images"]


def _clip(n):
    from flow_clip import clip_frames
    return clip_frames(n)


@pytest.mark.parametrize("precision", [0, 1, 2])
def test_trained_model_matches_host_chain(precision):
    pred = _predictor(precision)
    layer = pred.inference_model.inference_layer
    for what, imgs in (("frames_tracks_2node", _tracks_frames()), ("clip[:24]", _clip(24))):
        for i in range(0, len(imgs), 8):
            batch = imgs[i:i + 8]
            out = pred.inference_model.predict_on_batch(batch)
            assert_same_as_host(out, _device_host_chain(layer, batch), f"{what} batch {i // 8} precision {precision}")
            assert not out["flags"].any()
    out = pred.inference_model.predict_on_batch(_clip(8))
    assert np.isfinite(out["instance_peaks"]).any()


@pytest.mark.parametrize("precision", [0, 1, 2])
def test_predict_through_pipelined_loop(precision):
    from sleap_b200.io.video import Video
    pred = _predictor(precision, batch_size=5)
    clip = _clip(23)
    frames = pred.predict(Video.from_numpy(clip))
    assert [f.frame_idx for f in frames] == list(range(23))
    for i in range(0, 23, 5):
        out = pred.inference_model.predict_on_batch(clip[i:i + 5])
        for j, f in enumerate(frames[i:i + 5]):
            got = {inst.track.name: inst for inst in f.instances}
            for k, name in enumerate(pred.classes):
                pts = out["instance_peaks"][j, k]
                if np.all(np.isnan(pts)):
                    assert name not in got
                    continue
                assert_bit_equal(got[name].numpy(), pts, f"frame {i + j} class {name}")
    assert sum(len(f.instances) for f in frames) > 0


# ------------------------------------------------------------------------------------------------ pipeline
def _collect_all(layer, batches):
    m = layer.keras_model
    outs = []
    for s, b in enumerate(batches):
        m.handle.call("sb_multiclass_submit", m.model_id, b.ctypes.data_as(c_void_p), len(b), s % 2)
        if s % 2 == 1 or s == len(batches) - 1:
            for t in range(s - s % 2, s + 1):
                pts, vals, probs, fl = layer._outputs(len(batches[t]))
                m.handle.call("sb_multiclass_collect", m.model_id, t % 2, len(batches[t]), pts.ctypes.data_as(c_void_p),
                              vals.ctypes.data_as(c_void_p), probs.ctypes.data_as(c_void_p), fl.ctypes.data_as(c_void_p))
                outs.append({"instance_peaks": pts, "instance_peak_vals": vals, "instance_scores": probs, "flags": fl})
    return outs


@pytest.mark.parametrize("overlap", [True, False])
def test_back_to_back_submits(overlap, monkeypatch):
    if not overlap:
        monkeypatch.setenv("SB_DISABLE_POST_OVERLAP", "1")
    pred = _predictor(0)
    layer = pred.inference_model.inference_layer
    clip = np.ascontiguousarray(_clip(24))
    batches = [np.ascontiguousarray(clip[i:i + 4]) for i in range(0, 24, 4)]
    layer._configure(4, *clip.shape[1:])
    got = _collect_all(layer, batches)
    for s, b in enumerate(batches):
        want = pred.inference_model.predict_on_batch(b)
        assert_same_as_host(got[s], (want["instance_peaks"], want["instance_peak_vals"], want["instance_scores"]), f"step {s}")
    gen = list(pred.inference_model.predict_batches(clip, 4))
    for s, b in enumerate(batches):
        want = pred.inference_model.predict_on_batch(b)
        assert_same_as_host(gen[s], (want["instance_peaks"], want["instance_peak_vals"], want["instance_scores"]), f"loop {s}")


def test_bottomup_and_multiclass_models_alternate_on_one_handle():
    from sleap_b200.nn.inference import BottomUpPredictor, Predictor
    mc = _predictor(0)
    bu = Predictor.from_model_paths([rm.model_dir("minimal_instance.bottomup")], precision=0)
    assert isinstance(bu, BottomUpPredictor)
    assert bu.inference_model.bottomup_layer.keras_model.handle is mc.inference_model.inference_layer.keras_model.handle
    bu_imgs, _ = rm.frames("minimal_instance")
    bu_frames = np.ascontiguousarray(np.concatenate([bu_imgs] * 8))
    rng = np.random.default_rng(5)
    bu_frames = np.ascontiguousarray(np.clip(bu_frames.astype(np.int16) + rng.integers(-3, 4, bu_frames.shape), 0, 255).astype(np.uint8))
    mc_frames = np.ascontiguousarray(_clip(16))
    g_bu = bu.inference_model.predict_batches(bu_frames, 2)
    g_mc = mc.inference_model.predict_batches(mc_frames, 4)
    steps = []
    for _ in range(4):
        steps.append(("bu", next(g_bu)))
        steps.append(("mc", next(g_mc)))
    for k in range(4):
        want_bu = bu.inference_model.predict_on_batch(bu_frames[2 * k:2 * k + 2])
        got_bu = steps[2 * k][1]
        for key in ("instance_peaks", "instance_peak_vals", "instance_scores"):
            assert_bit_equal(got_bu[key], want_bu[key], f"bottom-up step {k} {key}")
        assert np.array_equal(got_bu["n_valid"], want_bu["n_valid"])
        want_mc = mc.inference_model.predict_on_batch(mc_frames[4 * k:4 * k + 4])
        assert_same_as_host(steps[2 * k + 1][1], (want_mc["instance_peaks"], want_mc["instance_peak_vals"],
                                                  want_mc["instance_scores"]), f"multi-class step {k}")


def test_maps_on_request():
    pred = _predictor(1)
    layer = pred.inference_model.inference_layer
    layer.return_confmaps, layer.return_class_maps = True, True
    imgs = _tracks_frames()
    out = pred.inference_model.predict_on_batch(imgs)
    assert out["confmaps"].shape[-1] == layer.n_nodes and out["class_maps"].shape[-1] == layer.n_classes
    cs, isc = F32(layer.class_maps_output_stride), F32(layer.input_scale)
    n = 0
    for b, k, c in np.argwhere(np.isfinite(out["instance_scores"])):
        x, y = out["instance_peaks"][b, k, c]
        col, row = int(np.rint((x - F32(0.5)) * isc / cs)), int(np.rint((y - F32(0.5)) * isc / cs))
        assert out["class_maps"][b, row, col, k] == out["instance_scores"][b, k, c]
        n += 1
    assert n > 0
    # the pipelined loop falls back to per-batch calls and still returns the maps
    gen = list(pred.inference_model.predict_batches(imgs, 1))
    assert "class_maps" in gen[0]


# ------------------------------------------------------------------------------------------------ errors
def test_errors():
    from sleap_b200._lib import SleapB200Error
    pred = _predictor(0)
    layer = pred.inference_model.inference_layer
    m = layer.keras_model
    imgs = np.ascontiguousarray(_tracks_frames())
    B, H, W = imgs.shape[:3]
    C = imgs.shape[3] if imgs.ndim == 4 else 1
    fresh = _predictor(0).inference_model.inference_layer
    fresh.keras_model.configure(1, H, W, C)
    pts, vals, probs, fl = fresh._outputs(1)
    with pytest.raises(SleapB200Error):                           # infer before configure
        fresh.keras_model.handle.call("sb_infer_multiclass", fresh.keras_model.model_id, imgs.ctypes.data_as(c_void_p), 1, 1,
                                      pts.ctypes.data_as(c_void_p), vals.ctypes.data_as(c_void_p),
                                      probs.ctypes.data_as(c_void_p), fl.ctypes.data_as(c_void_p))
    with pytest.raises(SleapB200Error):                           # submit before configure
        fresh.keras_model.handle.call("sb_multiclass_submit", fresh.keras_model.model_id, imgs.ctypes.data_as(c_void_p), 1, 0)
    layer._configure(1, H, W, C)

    def configure(**kw):
        p = layer.params()
        for k, v in kw.items():
            setattr(p, k, v)
        m.handle.call("sb_multiclass_configure", m.model_id, byref(p))

    heads = set(m.cm.head_buffers.values())
    internal = next(i for i in range(1, m.cm.n_buffers) if i not in heads)
    with pytest.raises(SleapB200Error):                           # class maps: wrong channel count
        configure(n_classes=layer.n_classes + 1)
    with pytest.raises(SleapB200Error):                           # class maps: a buffer that is no f32 head output
        configure(class_maps_buffer=internal)
    with pytest.raises(SleapB200Error):                           # too many classes
        configure(n_classes=129)
    configure()
    out = np.zeros(64, np.uint8)
    with pytest.raises(SleapB200Error):                           # the record exchange is the PAF chain's
        m.handle.call("sb_gather_init", m.model_id, 0, 1, 2, out.ctypes.data_as(c_void_p))
    m.chain = None
    res = pred.inference_model.predict_on_batch(imgs)             # a refused configure leaves a usable model after a good one
    assert np.isfinite(res["instance_peaks"]).any()
