"""GPU parity of the network forward (fp32 CUDA-core path: <=1e-4; fp16 tensor-core path: fp16
tolerance) against the torch-CPU oracle, and of the fused predictors end to end."""
import numpy as np
import pytest
from numpy.testing import assert_allclose, assert_array_equal

from oracle import convnet, paf_grouping as opg, peak_finding as opf, preprocess as opre, synth

pytestmark = pytest.mark.gpu


def _mk(spec, in_ch, seed, input_scale=1.0, precision=1):
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    cm = A.compile_model(spec, in_ch, input_scale)
    w = A.make_synthetic_weights(cm, seed)
    rng = np.random.default_rng(seed + 1)
    for L in cm.layers:   # non-trivial biases / BN statistics so every epilogue term is exercised
        if L["kind"] in ("conv", "tconv"):
            w[L["name"]]["bias"] = rng.normal(0, 0.1, size=L["cout"]).astype(np.float32)
        else:
            c = L["c"]
            w[L["name"]] = dict(gamma=rng.uniform(0.5, 1.5, c).astype(np.float32), beta=rng.normal(0, 0.1, c).astype(np.float32),
                                mean=rng.normal(0, 0.1, c).astype(np.float32), var=rng.uniform(0.5, 1.5, c).astype(np.float32))
    return DeviceModel(spec, w, input_channels=in_ch, input_scale=input_scale, precision=precision), w, cm


def _unet_spec(cfg, heads):
    return dict(backbone="unet", backbone_cfg=cfg, head_type="multi_instance", heads=heads, part_names=None, edges=None)


def _oracle_forward(imgs, spec, w, in_ch, input_scale, max_stride):
    x = opre.preprocess(imgs, ensure_gray=(in_ch == 1), input_scale=input_scale, pad_stride=max_stride)
    return convnet.model_forward(x, spec, w)


HEADS2 = [dict(name="MultiInstanceConfmapsHead", channels=5, output_stride=2),
          dict(name="PartAffinityFieldsHead", channels=8, output_stride=4)]

UNET_CASES = {
    "tconv": dict(filters=8, filters_rate=2, max_stride=16, output_stride=2, middle_block=True, up_interpolate=False),
    "interp": dict(filters=8, filters_rate=1.5, max_stride=8, output_stride=2, middle_block=True, up_interpolate=True),
    "nomiddle": dict(filters=4, filters_rate=2, max_stride=4, output_stride=2, middle_block=False, up_interpolate=False),
    "stem": dict(filters=8, filters_rate=2, max_stride=16, output_stride=2, middle_block=True, up_interpolate=True, stem_stride=2),
}


@pytest.mark.parametrize("name", list(UNET_CASES))
def test_unet_forward_fp32(name):
    cfg = UNET_CASES[name]
    spec = _unet_spec(cfg, HEADS2)
    model, w, cm = _mk(spec, 1, 3, precision=1)
    rng = np.random.default_rng(0)
    imgs = rng.integers(0, 256, size=(2, 61, 75, 1), dtype=np.uint8)      # needs bottom/right padding
    got = model.forward(imgs)
    want = _oracle_forward(imgs, spec, w, 1, 1.0, cfg["max_stride"])
    for g, x in zip(got, want):
        assert g.shape == x.shape
        assert_allclose(g, x, atol=1e-4 * max(1.0, np.abs(x).max()), rtol=1e-4)


def test_unet_forward_resize_and_rgb():
    cfg = UNET_CASES["tconv"]
    spec = _unet_spec(cfg, HEADS2)
    rng = np.random.default_rng(1)
    model, w, cm = _mk(spec, 1, 4, input_scale=0.5, precision=1)
    imgs = rng.integers(0, 256, size=(2, 96, 128, 3), dtype=np.uint8)     # rgb -> gray -> resize 0.5 -> pad
    got = model.forward(imgs)
    want = _oracle_forward(imgs, spec, w, 1, 0.5, cfg["max_stride"])
    for g, x in zip(got, want):
        assert_allclose(g, x, atol=2e-4 * max(1.0, np.abs(x).max()), rtol=1e-3)
    model3, w3, _ = _mk(spec, 3, 5, precision=1)
    gray = rng.uniform(0, 1, size=(1, 64, 64, 1)).astype(np.float32)        # gray float -> rgb
    got = model3.forward(gray)
    want = _oracle_forward(gray, spec, w3, 3, 1.0, cfg["max_stride"])
    for g, x in zip(got, want):
        assert_allclose(g, x, atol=1e-4 * max(1.0, np.abs(x).max()), rtol=1e-4)


def test_unet_forward_resize_fp16_first_layer_on_tensor_cores():
    """input_scale != 1 (and rgb -> gray): PREPROCESS runs as its own kernel and the first 3x3 conv takes the Toeplitz
    tensor-core form from the preprocessed one-channel buffer (sb_entry.cu, buffer view route) instead of k_conv_direct."""
    from ctypes import byref, c_int, c_void_p
    import torch
    from sleap_b200 import _lib
    cfg = dict(filters=16, filters_rate=2, max_stride=16, output_stride=2, middle_block=True, up_interpolate=False)
    spec = _unet_spec(cfg, HEADS2)
    model, w, cm = _mk(spec, 1, 6, input_scale=0.5, precision=0)
    imgs = np.random.default_rng(3).integers(0, 256, size=(2, 256, 320, 3), dtype=np.uint8)   # rgb -> gray -> resize 0.5
    got = model.forward(imgs)
    want = _oracle_forward(imgs, spec, w, 1, 0.5, cfg["max_stride"])
    for g, x in zip(got, want):
        assert np.abs(g - x).max() <= 2e-2 * np.abs(x).max()
    h = model.handle
    dev = torch.zeros((2, 256, 320, 3), dtype=torch.uint8, device="cuda")
    op_ms = np.zeros(64, np.float32); op_kind = np.zeros(64, np.int32); op_fl = np.zeros(64, np.float64)
    n_ops = c_int(0)
    h.call("sb_model_profile_ops", model.model_id, c_void_p(dev.data_ptr()), 2, 64, _lib.ptr(op_ms), _lib.ptr(op_kind), _lib.ptr(op_fl), byref(n_ops))
    assert 2 not in list(op_kind[:n_ops.value]), list(op_kind[:n_ops.value])       # no conv left on the CUDA-core kernel


def test_hourglass_forward_fp32():
    spec = dict(backbone="hourglass", head_type="multi_instance", part_names=None, edges=None,
                backbone_cfg=dict(stem_stride=4, max_stride=32, output_stride=4, stem_filters=8, filters=16, filter_increase=8, stacks=2),
                heads=[dict(name="MultiInstanceConfmapsHead", channels=6, output_stride=4),
                       dict(name="PartAffinityFieldsHead", channels=10, output_stride=4)])
    model, w, cm = _mk(spec, 3, 7, precision=1)
    imgs = np.random.default_rng(2).integers(0, 256, size=(2, 96, 64, 3), dtype=np.uint8)
    got = model.forward(imgs)
    want = _oracle_forward(imgs, spec, w, 3, 1.0, 32)
    for g, x in zip(got, want):
        assert_allclose(g, x, atol=1e-4 * max(1.0, np.abs(x).max()), rtol=1e-4)


def test_hourglass_forward_fp16():
    """conv -> ReLU -> BN affine epilogue of the tensor-core path (hourglass), additive skips, nearest x2."""
    spec = dict(backbone="hourglass", head_type="multi_instance", part_names=None, edges=None,
                backbone_cfg=dict(stem_stride=4, max_stride=32, output_stride=4, stem_filters=16, filters=32, filter_increase=32, stacks=2),
                heads=[dict(name="MultiInstanceConfmapsHead", channels=6, output_stride=4),
                       dict(name="PartAffinityFieldsHead", channels=10, output_stride=4)])
    model, w, cm = _mk(spec, 3, 17, precision=0)
    imgs = np.random.default_rng(2).integers(0, 256, size=(2, 512, 640, 3), dtype=np.uint8)
    got = model.forward(imgs)
    want = _oracle_forward(imgs, spec, w, 3, 1.0, 32)
    for g, x in zip(got, want):
        err = np.abs(g - x).max() / max(1e-6, np.abs(x).max())
        assert err < 2e-2, err


@pytest.mark.parametrize("name", ["tconv", "interp"])
def test_unet_forward_fp16(name):
    cfg = dict(UNET_CASES[name], filters=16, max_stride=16)
    spec = _unet_spec(cfg, HEADS2)
    model, w, cm = _mk(spec, 1, 9, precision=0)
    imgs = np.random.default_rng(3).integers(0, 256, size=(2, 128, 160, 1), dtype=np.uint8)
    got = model.forward(imgs)
    want = _oracle_forward(imgs, spec, w, 1, 1.0, 16)
    for g, x in zip(got, want):
        err = np.abs(g - x).max() / max(1e-6, np.abs(x).max())
        assert err < 2e-2, err      # fp16 activations through ~20 layers, fp32 accumulation


def _c4_small():
    cfg = dict(filters=8, filters_rate=2, max_stride=32, output_stride=4, middle_block=True, up_interpolate=False)
    heads = [dict(name="MultiInstanceConfmapsHead", channels=13, output_stride=4),
             dict(name="PartAffinityFieldsHead", channels=24, output_stride=8)]
    spec = _unet_spec(cfg, heads)
    spec["part_names"], spec["edges"] = synth.FLIES13_NODES, synth.FLIES13_EDGES
    return spec


@pytest.mark.parametrize("precision", [1, 0])
def test_bottomup_predictor_end_to_end(precision):
    """Fused device pipeline == oracle post-processing applied to the very maps the device produced."""
    from sleap_b200.nn.inference import BottomUpPredictor
    spec = _c4_small()
    model, w, cm = _mk(spec, 1, 21, precision=precision)
    # make the random net emit a sane number of peaks: rescale the head like bench.py does
    imgs = np.random.default_rng(5).integers(0, 256, size=(3, 256, 256, 1), dtype=np.uint8)
    pred = BottomUpPredictor(model, synth.FLIES13_NODES, synth.FLIES13_EDGES, peak_threshold=0.2, batch_size=3,
                             max_peaks_per_sample=4096, max_node_peaks=64, max_instances_per_frame=128)
    layer = pred.inference_model.bottomup_layer
    cms, pafs = model.forward(imgs)
    thr = float(np.quantile(cms, 0.9995))
    layer.peak_threshold = thr
    layer.return_paf_graph = True
    out = pred.inference_model.predict_on_batch(imgs)
    p, v, si, ci = opf.find_local_peaks(cms, thr, "integral", 5)
    assert 10 < len(p) < 3 * 4096
    p = (p * np.float32(4)).astype(np.float32)
    B = 3
    peaks = [p[si == b] for b in range(B)]; vals = [v[si == b] for b in range(B)]; chans = [ci[si == b] for b in range(B)]
    oscorer = opg.PAFScorer(synth.FLIES13_NODES, synth.FLIES13_EDGES, 8)
    winst, wps, wisc, wei, wepi, wls = oscorer.predict(pafs, peaks, vals, chans)
    for b in range(B):
        assert out["flags"][b] == 0
        assert_array_equal(out["peak_channel_inds"][b], chans[b])
        assert_array_equal(out["edge_peak_inds"][b], wepi[b])
        assert_allclose(out["line_scores"][b], wls[b], atol=1e-4, rtol=0, equal_nan=True)
        n = out["n_valid"][b]
        assert n == len(winst[b])
        assert_array_equal(np.isnan(out["instance_peaks"][b, :n]), np.isnan(winst[b]))
        assert_allclose(out["instance_peaks"][b, :n], winst[b], atol=4e-4, rtol=0, equal_nan=True)
        assert_allclose(out["instance_scores"][b, :n], wisc[b], atol=1e-4, rtol=0)
        assert np.all(np.isnan(out["instance_peaks"][b, n:]))
    frames = pred.predict(imgs, make_labels=True)
    assert len(frames) == 3 and frames[0].frame_idx == 0


def test_single_instance_predictor():
    from sleap_b200.nn.inference import SingleInstancePredictor
    cfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=2, middle_block=True, up_interpolate=True)
    spec = dict(backbone="unet", backbone_cfg=cfg, head_type="single_instance", part_names=list("abcde"), edges=None,
                heads=[dict(name="SingleInstanceConfmapsHead", channels=5, output_stride=2)])
    model, w, cm = _mk(spec, 1, 31, precision=1)
    imgs = np.random.default_rng(6).integers(0, 256, size=(4, 128, 128, 1), dtype=np.uint8)
    cms = model.forward(imgs)[0]
    thr = float(np.median(cms.max(axis=(1, 2))))      # about half of the (sample, channel) maxima pass
    pred = SingleInstancePredictor(model, peak_threshold=thr, integral_refinement=True, batch_size=4)
    out = pred.inference_model.predict_on_batch(imgs)
    wp, wv = opf.find_global_peaks(cms, thr, "integral", 5)
    wp = wp * np.float32(2)
    assert out["instance_peaks"].shape == (4, 1, 5, 2)
    assert_array_equal(np.isnan(out["instance_peaks"][:, 0]), np.isnan(wp))
    assert_allclose(out["instance_peaks"][:, 0], wp, atol=2e-4, equal_nan=True)
    assert_array_equal(out["instance_peak_vals"][:, 0], wv)


def test_topdown_predictor():
    from sleap_b200.nn.inference import TopDownPredictor
    from oracle import tf_ops
    ccfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=2, middle_block=True, up_interpolate=True)
    cspec = dict(backbone="unet", backbone_cfg=ccfg, head_type="centroid", part_names=None, edges=None,
                 heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
    icfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=4, middle_block=True, up_interpolate=False)
    ispec = dict(backbone="unet", backbone_cfg=icfg, head_type="centered_instance", part_names=list("abcd"), edges=None,
                 heads=[dict(name="CenteredInstanceConfmapsHead", channels=4, output_stride=4)])
    cmodel, cw, _ = _mk(cspec, 1, 41, input_scale=0.5, precision=1)
    imodel, iw, _ = _mk(ispec, 1, 43, precision=1)
    imgs = np.random.default_rng(7).integers(0, 256, size=(2, 256, 256, 1), dtype=np.uint8)
    ccms = cmodel.forward(imgs)[0]
    flat = np.sort(ccms.reshape(-1))
    thr = float(flat[-40])
    pred = TopDownPredictor(cmodel, imodel, crop_size=64, peak_threshold=thr, integral_refinement=True, batch_size=2,
                            max_instances=3)
    pred.inference_model.instance_peaks.peak_threshold = -1e9     # keep every node so all paths are compared
    out = pred.inference_model.predict_on_batch(imgs)
    # oracle chain on the device's centroid maps
    cp, cv, csi, _ = opf.find_local_peaks(ccms, thr, "integral", 5)
    cp = (cp * np.float32(2)) / np.float32(0.5) + np.float32(0.5)
    keep = []
    for s in range(2):
        idx = np.nonzero(csi == s)[0]
        if len(idx) > 3:
            idx = idx[np.argsort(-cv[idx], kind="stable")[:3]]
        keep.append(idx)
    keep = np.concatenate(keep)
    cp, cv, csi = cp[keep], cv[keep], csi[keep]
    assert len(cp) > 0
    bb = tf_ops.make_centered_bboxes(cp, 64, 64)
    crops = tf_ops.crop_bboxes(imgs, bb, csi)
    icms = convnet.model_forward(opre.preprocess(crops, True, 1.0, 16), ispec, iw)[0]
    dcms = imodel.forward(crops)[0]
    assert_allclose(dcms, icms, atol=1e-4 * max(1, np.abs(icms).max()), rtol=1e-4)
    wp, wv = opf.find_global_peaks(dcms, -1e9, "integral", 5)
    wp = wp * np.float32(4) + (cp - np.float32(32))[:, None, :]
    for s in range(2):
        n = int(out["n_valid"][s])
        assert n == int((csi == s).sum())
        assert_allclose(out["centroids"][s, :n], cp[csi == s], atol=1e-4)
        assert_allclose(out["instance_peaks"][s, :n], wp[csi == s], atol=5e-4, equal_nan=True)
    # the fused device pipeline (sb_infer_topdown, default) and the stage-by-stage path (CentroidCrop -> FindInstancePeaks
    # through host memory) run the same kernels on the same data: identical results, with and without the top-k cut
    assert pred.inference_model._can_fuse()
    for mi in (3, None, 1):
        pred.inference_model.centroid_crop.max_instances = mi
        pred.inference_model.fused = True
        a = pred.inference_model.predict_on_batch(imgs)
        pred.inference_model.fused = False
        b = pred.inference_model.predict_on_batch(imgs)
        assert_array_equal(a["n_valid"], b["n_valid"])
        for k in ("centroids", "centroid_vals", "instance_peaks", "instance_peak_vals"):
            assert_array_equal(np.nan_to_num(a[k], nan=-7.0), np.nan_to_num(b[k], nan=-7.0))
    assert int(a["n_valid"].max()) == 1


def test_tc_path_matches_direct_fp16(monkeypatch):
    """wgmma implicit-GEMM convs vs the CUDA-core kernels on identical fp16 activations / weights:
    only the fp32 accumulation order differs."""
    cfg = dict(filters=64, filters_rate=2, max_stride=8, output_stride=2, middle_block=True, up_interpolate=False)
    heads = [dict(name="MultiInstanceConfmapsHead", channels=13, output_stride=2),
             dict(name="PartAffinityFieldsHead", channels=24, output_stride=4)]
    spec = _unet_spec(cfg, heads)
    imgs = np.random.default_rng(11).integers(0, 256, size=(2, 128, 144, 1), dtype=np.uint8)
    tc_model, w, cm = _mk(spec, 1, 13, precision=0)
    got_tc = tc_model.forward(imgs)
    launches_tc = tc_model.handle.gpu_launches()
    monkeypatch.setenv("SB_DISABLE_TC", "1")
    dm, _, _ = _mk(spec, 1, 13, precision=0)
    got_direct = dm.forward(imgs)
    monkeypatch.delenv("SB_DISABLE_TC")
    want = _oracle_forward(imgs, spec, w, 1, 1.0, 8)
    for a, b, x in zip(got_tc, got_direct, want):
        scale = np.abs(x).max()
        assert np.abs(a - b).max() / scale < 3e-3, np.abs(a - b).max() / scale
        assert np.abs(a - x).max() / scale < 2e-2
    assert launches_tc > 0


@pytest.mark.parametrize("variant", [None, "0", "1", "2", "4"])
@pytest.mark.parametrize("cin,cout", [(16, 16), (64, 32), (128, 64), (256, 128), (512, 256)])
def test_tc_tconv_layers(cin, cout, variant, monkeypatch):
    """Conv2DTranspose(k3, s2) on the tensor cores, against the CUDA-core kernel on the same fp16 activations, with
    SB_FORCE_VARIANT = variant: None autotuned; 0 / 1 the four sub-pixel phase launches in the streaming / resident form
    (a phase the form does not take stays autotuned); 2 the phase launches in their autotuned forms (no phase takes the
    halo form); 4 the fused form where it is eligible."""
    from conv_forms import tconv_layer
    layer = tconv_layer(cin, cout, (88, 72), 2)          # tconv input grid 44 x 36 -> output 88 x 72, fp16
    if variant is not None:
        monkeypatch.setenv("SB_FORCE_VARIANT", variant)
    got = layer()[0]
    monkeypatch.delenv("SB_FORCE_VARIANT", raising=False)
    monkeypatch.setenv("SB_DISABLE_TC", "1")
    want = layer()[0]
    assert np.abs(want).max() > 0.1
    assert_allclose(got, want, atol=3e-3 * max(1.0, np.abs(want).max()), rtol=3e-3)


@pytest.mark.parametrize("variant,no_first_view", [("2", None), ("3", None), ("4", None), ("5", None), ("2", "1")])
def test_tc_forced_variants_unet(variant, no_first_view, monkeypatch):
    """The whole fp16 UNet (transposed convs, fused max-pool, concat-by-slice outputs) with SB_FORCE_VARIANT = variant,
    against the CUDA-core path: 2 / 3 the halo / wide form wherever it is eligible and the phase launches; 4 the autotuned
    launch forms and the fused transposed convs; 5 the autotuned launch forms and the phase launches.  no_first_view:
    SB_DISABLE_FIRST_VIEW, so the first layer runs on k_conv_first instead of its Toeplitz view (None: autotuned)."""
    cfg = dict(filters=32, filters_rate=2, max_stride=8, output_stride=2, middle_block=True, up_interpolate=False)
    heads = [dict(name="MultiInstanceConfmapsHead", channels=13, output_stride=2),
             dict(name="PartAffinityFieldsHead", channels=24, output_stride=4)]
    spec = _unet_spec(cfg, heads)
    imgs = np.random.default_rng(12).integers(0, 256, size=(2, 288, 304, 1), dtype=np.uint8)
    monkeypatch.setenv("SB_FORCE_VARIANT", variant)
    if no_first_view:
        monkeypatch.setenv("SB_DISABLE_FIRST_VIEW", no_first_view)
    tc_model, w, cm = _mk(spec, 1, 17, precision=0)
    got_tc = tc_model.forward(imgs)
    monkeypatch.delenv("SB_FORCE_VARIANT")
    monkeypatch.delenv("SB_DISABLE_FIRST_VIEW", raising=False)
    monkeypatch.setenv("SB_DISABLE_TC", "1")
    dm, _, _ = _mk(spec, 1, 17, precision=0)
    got_direct = dm.forward(imgs)
    for a, b in zip(got_tc, got_direct):
        scale = np.abs(b).max()
        assert np.abs(a - b).max() / scale < 3e-3, np.abs(a - b).max() / scale


@pytest.mark.parametrize("variant", [None, "0", "1", "2", "3", "4", "5", "6", "7", "8", "9"])
@pytest.mark.parametrize("cin,cout,k,hw", [(16, 16, 3, (40, 48)), (32, 32, 3, (40, 48)), (64, 64, 3, (53, 70)),
                                           (128, 128, 3, (40, 48)), (256, 128, 3, (53, 70)), (128, 256, 3, (40, 48)), (128, 64, 3, (53, 70)),
                                           (256, 512, 3, (40, 48)), (64, 13, 1, (40, 48)), (128, 24, 1, (40, 48)),
                                           (24, 24, 3, (40, 48)), (48, 36, 3, (40, 48)), (96, 48, 3, (53, 70)),
                                           (192, 96, 3, (40, 48)), (24, 13, 1, (40, 48)),
                                           (32, 32, 5, (40, 48)), (64, 48, 7, (53, 70)), (128, 64, 5, (40, 48)), (16, 16, 7, (40, 48)),
                                           (192, 384, 3, (10, 10)), (384, 384, 3, (5, 7)), (64, 64, 3, (12, 20)), (96, 24, 1, (3, 3))])
def test_tc_single_layers(cin, cout, k, hw, variant, monkeypatch):
    """Each swizzle mode / chunk count / N-tile shape of the tensor-core conv on its own, autotuned (None) and with each
    launch form 0-3 forced (SB_FORCE_VARIANT; a form that is not eligible for the layer leaves it autotuned).  4 (the
    fused transposed conv) and 5-9 name no launch form of a conv: the layer must run its autotuned forms."""
    if variant is not None:
        monkeypatch.setenv("SB_FORCE_VARIANT", variant)
    import torch
    import torch.nn.functional as F
    from ctypes import byref, c_int, c_void_p
    from sleap_b200 import _lib
    from conv_forms import conv_layer
    layer = conv_layer(cin, cout, hw, 2, k=k, relu=False, f32_out=True)
    B, H, W, _ = layer.imgs.shape

    def op_kinds(h, mid):
        """the per-op profile's kinds: the layer must run on the tensor-core path (kind 1), not on the CUDA-core fallback"""
        dev = torch.zeros((B, H, W, 1), dtype=torch.uint8, device="cuda")
        op_ms = np.zeros(16, np.float32); op_kind = np.zeros(16, np.int32); op_fl = np.zeros(16, np.float64)
        n_ops = c_int(0)
        h.call("sb_model_profile_ops", mid, c_void_p(dev.data_ptr()), B, 16, _lib.ptr(op_ms), _lib.ptr(op_kind), _lib.ptr(op_fl),
               byref(n_ops))
        return list(op_kind[:n_ops.value])
    (mids, outs), kinds = layer.run(ids=[1, 2], probe=op_kinds)
    assert kinds[-1] == 1, kinds
    # reference from the *device's* fp16 intermediate so only this layer is under test
    x = torch.from_numpy(mids).permute(0, 3, 1, 2)
    w16 = torch.from_numpy(layer.w1.astype(np.float16).astype(np.float32)).permute(3, 2, 0, 1)
    y = F.conv2d(x, w16, torch.from_numpy(layer.b1), padding=k // 2).permute(0, 2, 3, 1).numpy()
    assert_allclose(outs, y, atol=2e-3 * max(1.0, np.abs(y).max()), rtol=2e-3)


@pytest.mark.filterwarnings("ignore:device capacity reached")
def test_predictor_reconfigures_between_frame_sizes():
    """One predictor, two videos of different size / batch / capacity (ADVICE r1: the submit/collect slots and the pinned
    staging were sized once): results equal a fresh predictor's, in both directions (grow and shrink)."""
    from sleap_b200.nn.inference import BottomUpPredictor
    spec = _c4_small()
    model, w, cm = _mk(spec, 1, 29, precision=0)
    rng = np.random.default_rng(5)
    small = rng.integers(0, 256, size=(6, 128, 160, 1), dtype=np.uint8)
    big = rng.integers(0, 256, size=(5, 256, 320, 1), dtype=np.uint8)
    thr = float(np.quantile(model.forward(big[:2])[0], 0.998))
    kw = dict(peak_threshold=thr, max_peaks_per_sample=4096, max_node_peaks=64, min_line_scores=-100.0)

    def fresh(imgs, bs, cap):
        m2, _, _ = _mk(spec, 1, 29, precision=0)
        return BottomUpPredictor(m2, synth.FLIES13_NODES, synth.FLIES13_EDGES, batch_size=bs, max_instances_per_frame=cap, **kw).predict(
            imgs, make_labels=False)

    pred = BottomUpPredictor(model, synth.FLIES13_NODES, synth.FLIES13_EDGES, batch_size=2, max_instances_per_frame=32, **kw)
    for imgs, bs, cap in ((small, 2, 32), (big, 4, 32), (small, 2, 32)):
        pred.batch_size = bs
        got = pred.predict(imgs, make_labels=False)
        want = fresh(imgs, bs, cap)
        assert len(got) == len(want)
        for g, x in zip(got, want):
            assert_array_equal(g["n_valid"], x["n_valid"])
            assert_array_equal(np.nan_to_num(g["instance_peaks"], nan=-1), np.nan_to_num(x["instance_peaks"], nan=-1))
    # growing the instance capacity re-sizes the staging records as well
    pred.inference_model.bottomup_layer.max_instances = 128
    pred.batch_size = 4
    got = pred.predict(big, make_labels=False)
    want = fresh(big, 4, 128)
    for g, x in zip(got, want):
        assert_array_equal(g["n_valid"], x["n_valid"])
        assert_array_equal(np.nan_to_num(g["instance_peaks"], nan=-1), np.nan_to_num(x["instance_peaks"], nan=-1))


def test_pipelined_predict_matches_per_batch():
    """submit/collect double buffering returns exactly what predict_on_batch returns, batch by batch."""
    from sleap_b200.nn.inference import BottomUpPredictor
    spec = _c4_small()
    model, w, cm = _mk(spec, 1, 23, precision=0)
    imgs = np.random.default_rng(8).integers(0, 256, size=(10, 256, 256, 1), dtype=np.uint8)
    cms, _ = model.forward(imgs[:2])
    thr = float(np.quantile(cms, 0.9995))
    pred = BottomUpPredictor(model, synth.FLIES13_NODES, synth.FLIES13_EDGES, peak_threshold=thr, batch_size=4,
                             max_peaks_per_sample=4096, max_node_peaks=64, max_instances_per_frame=128)
    want = [pred.inference_model.predict_on_batch(imgs[i:i + 4]) for i in range(0, 10, 4)]
    got = pred.predict(imgs, make_labels=False)
    assert len(got) == 3
    for g, x in zip(got, want):
        assert_array_equal(g["n_valid"], x["n_valid"])
        assert_array_equal(np.nan_to_num(g["instance_peaks"], nan=-1), np.nan_to_num(x["instance_peaks"], nan=-1))
        assert_array_equal(np.nan_to_num(g["instance_scores"], nan=-1), np.nan_to_num(x["instance_scores"], nan=-1))
    assert list(got[2]["frame_ind"]) == [8, 9]
    merged = pred.inference_model.predict(imgs, batch_size=4)
    assert merged["instance_peaks"].shape[0] == 10


@pytest.mark.parametrize("variant", [None, "0", "1", "2", "3"])
@pytest.mark.parametrize("cout,hw,as_float", [(16, (64, 128), False), (16, (38, 136), False), (8, (48, 256), False),
                                              (32, (64, 128), True), (24, (36, 160), False)])
def test_first_layer_toeplitz_view(cout, hw, as_float, variant, monkeypatch):
    """First conv (1 input channel) as a Toeplitz GEMM on the stock tensor-core kernel (sb_entry.cu,
    toeplitz_prepare) vs the torch-CPU fp32 conv on the fp16-rounded operands it consumes, and vs the
    CUDA-core k_conv_first (SB_DISABLE_FIRST_VIEW=1).  Covers every kernel variant, widths whose group
    count is not a tile multiple, float frames, and the bottom zero pad (H not a multiple of the stride)."""
    from ctypes import byref, c_int, c_void_p
    import torch
    from sleap_b200 import _lib
    from sleap_b200.nn import oplist as ol
    H, W = hw
    B = 3
    rng = np.random.default_rng(cout * 100 + H)
    w0 = (rng.standard_normal((3, 3, 1, cout)) * 0.5).astype(np.float32)
    b0 = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    blob = np.concatenate([w0.reshape(-1), b0]).astype(np.float32)
    recs = [ol.buffer_record(0, 1, 1, 0, 1), ol.buffer_record(1, 1, cout, 0, 0), ol.preprocess_record(0, 1, 1.0, 4),
            ol.conv_record(0, 0, 1, 1, 0, cout, 3, 1, True, 0, w0.size)]
    ops = np.ascontiguousarray(np.stack(recs).astype(np.int32))
    if as_float:
        imgs = rng.random((B, H, W, 1)).astype(np.float32)
        xin = imgs
    else:
        imgs = rng.integers(0, 256, size=(B, H, W, 1), dtype=np.uint8)
        xin = imgs.astype(np.float32) * np.float32(1.0 / 255.0)
    Hn = -(-H // 4) * 4

    def run():
        h = _lib.Handle(0)
        mid = c_int(-1)
        h.call("sb_load_model", _lib.ptr(ops), ops.shape[0], _lib.ptr(blob), int(blob.size), 0, byref(mid))
        h.call("sb_model_configure", mid.value, B, H, W, 1)
        out = np.zeros((B, Hn, W, cout), np.float32)
        ids = np.asarray([1], np.int32)
        ptrs = (c_void_p * 1)(out.ctypes.data)
        h.call("sb_model_forward", mid.value, _lib.ptr(imgs), int(not as_float), B, 1, _lib.ptr(ids), ptrs)
        n = h.gpu_launches()
        h.close()
        return out, n

    if variant is not None:
        monkeypatch.setenv("SB_FORCE_VARIANT", variant)
    got, _ = run()
    monkeypatch.setenv("SB_DISABLE_FIRST_VIEW", "1")
    direct, _ = run()
    monkeypatch.delenv("SB_DISABLE_FIRST_VIEW")
    x16 = torch.from_numpy(np.pad(xin, ((0, 0), (0, Hn - H), (0, 0), (0, 0)))).half().float().permute(0, 3, 1, 2)
    w16 = torch.from_numpy(w0).half().float().permute(3, 2, 0, 1)
    want = torch.relu(torch.nn.functional.conv2d(x16, w16, torch.from_numpy(b0), padding=1)).permute(0, 2, 3, 1).numpy()
    scale = max(1.0, float(np.abs(want).max()))
    assert_allclose(got, want, atol=1.5e-3 * scale, rtol=0)          # fp16 output rounding (2^-11 relative)
    assert_allclose(got, direct, atol=4e-3 * scale, rtol=0)          # direct kernel keeps fp32 pixels / weights


@pytest.mark.gpu
def test_load_model_rejects_second_preprocess_op():
    """The network has one input stage: an op list with a second PREPROCESS op is refused at load time."""
    from ctypes import byref, c_int
    from sleap_b200 import _lib
    from sleap_b200.nn import oplist as ol
    blob = np.zeros(9 * 8 + 8, np.float32)
    recs = [ol.buffer_record(0, 1, 1, 0, 1), ol.buffer_record(1, 1, 8, 0, 0), ol.preprocess_record(0, 1, 1.0, 1),
            ol.conv_record(0, 0, 1, 1, 0, 8, 3, 1, True, 0, 72)]
    h = _lib.Handle(0)
    try:
        mid = c_int(-1)
        ops = np.ascontiguousarray(np.stack(recs).astype(np.int32))
        h.call("sb_load_model", _lib.ptr(ops), ops.shape[0], _lib.ptr(blob), int(blob.size), 0, byref(mid))
        ops = np.ascontiguousarray(np.stack(recs + [ol.preprocess_record(0, 1, 1.0, 1)]).astype(np.int32))
        with pytest.raises(_lib.SleapB200Error, match="second preprocess"):
            h.call("sb_load_model", _lib.ptr(ops), ops.shape[0], _lib.ptr(blob), int(blob.size), 0, byref(mid))
    finally:
        h.close()


@pytest.mark.parametrize("hw,as_float,relu", [((64, 64), False, True), ((34, 1056), False, True), ((96, 520), True, True),
                                              ((40, 516), False, False)])
def test_conv01_fused_first_block(hw, as_float, relu, monkeypatch):
    """k_conv01 (sb_conv01.cu): frame -> conv0 (1 -> 16) -> conv1 (16 -> 16) -> 2x2 max-pool in ONE kernel, against
    (a) torch fp32 convs on the operands the tensor cores consume (fp16 pixels / weights, fp16-rounded intermediate) and
    (b) the two separate tensor-core launches (SB_FORCE_CONV01=0).  Partial edge tiles (W not a multiple of 16,
    H not a multiple of 8), float frames, bottom zero padding, no-ReLU."""
    from ctypes import byref, c_int, c_void_p
    import torch
    import torch.nn.functional as F
    from sleap_b200 import _lib
    from sleap_b200.nn import oplist as ol
    H, W = hw
    B = 3
    rng = np.random.default_rng(H * 7 + W)
    w0 = (rng.standard_normal((3, 3, 1, 16)) * 0.5).astype(np.float32); b0 = (rng.standard_normal(16) * 0.1).astype(np.float32)
    w1 = (rng.standard_normal((3, 3, 16, 16)) * np.sqrt(2.0 / 144)).astype(np.float32); b1 = (rng.standard_normal(16) * 0.1).astype(np.float32)
    blob = np.concatenate([w0.reshape(-1), b0, w1.reshape(-1), b1]).astype(np.float32)
    o1 = w0.size + 16
    # buffers: 0 input, 1 conv0 out (stride 1), 2 conv1 out (stride 1), 3 pooled (stride 2), 4 copy of pooled as f32 via 1x1 identity conv
    eye = np.eye(16, dtype=np.float32).reshape(1, 1, 16, 16)
    blob = np.concatenate([blob, eye.reshape(-1), np.zeros(16, np.float32)])
    o2 = o1 + w1.size + 16
    recs = [ol.buffer_record(0, 1, 1, 0, 1), ol.buffer_record(1, 1, 16, 0, 0), ol.buffer_record(2, 1, 16, 0, 0), ol.buffer_record(3, 2, 16, 0, 0),
            ol.buffer_record(4, 2, 16, 1, 0), ol.preprocess_record(0, 1, 1.0, 4),
            ol.conv_record(0, 0, 1, 1, 0, 16, 3, 1, relu, 0, w0.size),
            ol.conv_record(1, 0, 16, 2, 0, 16, 3, 1, relu, o1, o1 + w1.size, pool_buf=3, pool_coff=0),
            ol.pool_record(2, 0, 16, 3, 0, fused=True),
            ol.conv_record(3, 0, 16, 4, 0, 16, 1, 1, False, o2, o2 + 256)]
    ops = np.ascontiguousarray(np.stack(recs).astype(np.int32))
    if as_float:
        imgs = rng.random((B, H, W, 1)).astype(np.float32); xin = imgs
    else:
        imgs = rng.integers(0, 256, size=(B, H, W, 1), dtype=np.uint8); xin = imgs.astype(np.float32) * np.float32(1.0 / 255.0)
    Hn, Wn = -(-H // 4) * 4, -(-W // 4) * 4

    def run(fused):
        monkeypatch.setenv("SB_FORCE_CONV01", "1" if fused else "0")
        h = _lib.Handle(0)
        mid = c_int(-1)
        h.call("sb_load_model", _lib.ptr(ops), ops.shape[0], _lib.ptr(blob), int(blob.size), 0, byref(mid))
        h.call("sb_model_configure", mid.value, B, H, W, 1)
        out = np.zeros((B, Hn // 2, Wn // 2, 16), np.float32)
        ids = np.asarray([4], np.int32)
        ptrs = (c_void_p * 1)(out.ctypes.data)
        for _ in range(2):                                   # twice: ring / barrier state must be reusable across launches
            h.call("sb_model_forward", mid.value, _lib.ptr(imgs), int(not as_float), B, 1, _lib.ptr(ids), ptrs)
        n = h.gpu_launches()
        h.close()
        return out, n

    got, n_fused = run(True)
    sep, n_sep = run(False)
    assert n_fused < n_sep                                   # the fused block really ran (one launch instead of view + conv0 + conv1)
    act = (lambda t: torch.relu(t)) if relu else (lambda t: t)
    x = torch.from_numpy(np.pad(xin, ((0, 0), (0, Hn - H), (0, Wn - W), (0, 0)))).half().float().permute(0, 3, 1, 2)
    y0 = act(F.conv2d(x, torch.from_numpy(w0).half().float().permute(3, 2, 0, 1), torch.from_numpy(b0), padding=1)).half().float()
    y1 = act(F.conv2d(y0, torch.from_numpy(w1).half().float().permute(3, 2, 0, 1), torch.from_numpy(b1), padding=1)).half().float()
    want = F.max_pool2d(y1, 2).permute(0, 2, 3, 1).numpy()
    scale = max(1.0, float(np.abs(want).max()))
    assert_allclose(got, want, atol=2.5e-3 * scale, rtol=0)      # one fp16 ulp of the intermediate propagated through 144 taps
    assert_allclose(got, sep, atol=2.5e-3 * scale, rtol=0)
    assert np.mean(np.abs(got - want) > 1e-3 * scale) < 1e-3     # ... and only on a handful of values


@pytest.mark.parametrize("cin,cout,hw,as_float,bn", [(3, 32, (64, 96), False, True), (1, 16, (70, 130), False, False), (3, 128, (96, 64), True, True)])
def test_tc_stem_7x7_stride2(cin, cout, hw, as_float, bn):
    """Hourglass stem (hourglass.py:49-100): 7x7 stride-2 SAME convolution on 1 / 3 input channels as a 4x4 convolution over
    the space-to-depth view of the frame on the tensor-core path (sb_entry.cu, stem_prepare), conv -> ReLU -> BN affine.
    Reference: torch conv2d with TF SAME padding (2 before, 3 after for even sizes) on the fp16-rounded operands."""
    from ctypes import byref, c_int, c_void_p
    import torch
    import torch.nn.functional as F
    from sleap_b200 import _lib
    from sleap_b200.nn import oplist as ol
    H, W = hw
    B = 2
    rng = np.random.default_rng(cin * 100 + cout)
    w0 = (rng.standard_normal((7, 7, cin, cout)) * np.sqrt(2.0 / (49 * cin))).astype(np.float32)
    b0 = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    sc = rng.uniform(0.5, 1.5, cout).astype(np.float32); sh = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    eye = np.eye(cout, dtype=np.float32).reshape(-1)
    blob = np.concatenate([w0.reshape(-1), b0, sc, sh, eye, np.zeros(cout, np.float32)]).astype(np.float32)
    ob, osc, osh, oe = w0.size, w0.size + cout, w0.size + 2 * cout, w0.size + 3 * cout
    recs = [ol.buffer_record(0, 1, cin, 0, 1), ol.buffer_record(1, 2, cout, 0, 0), ol.buffer_record(2, 2, cout, 1, 0),
            ol.preprocess_record(0, cin, 1.0, 2),
            ol.conv_record(0, 0, cin, 1, 0, cout, 7, 2, True, 0, ob, bn_scale_off=osc if bn else -1, bn_shift_off=osh if bn else -1),
            ol.conv_record(1, 0, cout, 2, 0, cout, 1, 1, False, oe, oe + cout * cout)]
    ops = np.ascontiguousarray(np.stack(recs).astype(np.int32))
    if as_float:
        imgs = rng.random((B, H, W, cin)).astype(np.float32); xin = imgs
    else:
        imgs = rng.integers(0, 256, size=(B, H, W, cin), dtype=np.uint8); xin = imgs.astype(np.float32) * np.float32(1.0 / 255.0)
    Hn, Wn = -(-H // 2) * 2, -(-W // 2) * 2
    h = _lib.default_handle()
    mid = c_int(-1)
    h.call("sb_load_model", _lib.ptr(ops), ops.shape[0], _lib.ptr(blob), int(blob.size), 0, byref(mid))
    h.call("sb_model_configure", mid.value, B, H, W, cin)
    out = np.zeros((B, Hn // 2, Wn // 2, cout), np.float32)
    ids = np.asarray([2], np.int32)
    ptrs = (c_void_p * 1)(out.ctypes.data)
    h.call("sb_model_forward", mid.value, _lib.ptr(imgs), int(not as_float), B, 1, _lib.ptr(ids), ptrs)
    dev = torch.zeros((B, H, W, cin), dtype=torch.uint8, device="cuda")
    op_ms = np.zeros(8, np.float32); op_kind = np.zeros(8, np.int32); op_fl = np.zeros(8, np.float64)
    n_ops = c_int(0)
    h.call("sb_model_profile_ops", mid.value, c_void_p(dev.data_ptr()), B, 8, _lib.ptr(op_ms), _lib.ptr(op_kind), _lib.ptr(op_fl), byref(n_ops))
    assert op_kind[1] == 1, list(op_kind[:n_ops.value])                   # the stem ran on the tensor-core path
    x = torch.from_numpy(np.pad(xin, ((0, 0), (0, Hn - H), (0, Wn - W), (0, 0)))).half().float().permute(0, 3, 1, 2)
    x = F.pad(x, (2, 3, 2, 3))                                               # TF SAME for k = 7, s = 2 on even sizes
    y = torch.relu(F.conv2d(x, torch.from_numpy(w0).half().float().permute(3, 2, 0, 1), torch.from_numpy(b0), stride=2))
    if bn:
        y = y * torch.from_numpy(sc).view(1, -1, 1, 1) + torch.from_numpy(sh).view(1, -1, 1, 1)
    want = y.half().float().permute(0, 2, 3, 1).numpy()
    assert_allclose(out, want, atol=2e-3 * max(1.0, float(np.abs(want).max())), rtol=2e-3)
