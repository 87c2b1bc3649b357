"""GPU parity of the ResNet (v1 + UpsamplingStack) and LEAP backbones against the torch-CPU oracle written from the
reference source (tests/backbone_oracle.py), in the three precisions, and end to end through Predictor.from_model_paths.

Bars: fp32 CUDA-core path <= 1e-4 * max, fp16 tensor-core path <= 5e-3 * max, precision 2 <= 5e-5 * max."""
import json
import os

import numpy as np
import pytest
from numpy.testing import assert_allclose, assert_array_equal

from oracle import paf_grouping as opg, peak_finding as opf, preprocess as opre, synth
import backbone_oracle as bo

pytestmark = pytest.mark.gpu

BAR = {0: 5e-3, 1: 1e-4, 2: 5e-5}
HEADS = [dict(name="MultiInstanceConfmapsHead", channels=5, output_stride=4),
         dict(name="PartAffinityFieldsHead", channels=8, output_stride=8)]


def _resnet_spec(max_stride=32, weights="frozen", up="tconv_concat", heads=HEADS):
    ups = {
        "tconv_concat": dict(method="transposed_conv", skip_connections="concatenate", block_stride=2, filters=64, filters_rate=1,
                             refine_convs=2, batch_norm=True, transposed_conv_kernel_size=4),
        "interp_add": dict(method="interpolation", skip_connections="add", block_stride=2, filters=64, filters_rate=1,
                           refine_convs=1, batch_norm=False, transposed_conv_kernel_size=4),
        "tconv_add_nobn": dict(method="transposed_conv", skip_connections="add", block_stride=2, filters=32, filters_rate=2,
                               refine_convs=1, batch_norm=False, transposed_conv_kernel_size=4),
    }
    cfg = dict(version="ResNet50", weights=weights, max_stride=max_stride, output_stride=4, upsampling=ups[up])
    return dict(backbone="resnet", backbone_cfg=cfg, head_type="multi_instance", heads=heads, part_names=None, edges=None)


def _leap_spec(interp=False):
    cfg = dict(max_stride=8, output_stride=2, filters=16, filters_rate=2, up_interpolate=interp, stacks=1)
    heads = [dict(name="MultiInstanceConfmapsHead", channels=5, output_stride=2),
             dict(name="PartAffinityFieldsHead", channels=8, output_stride=4)]
    return dict(backbone="leap", backbone_cfg=cfg, head_type="multi_instance", heads=heads, part_names=None, edges=None)


def _weights(cm, seed):
    """Synthetic weights with non-trivial biases and BN statistics (every fold / epilogue term exercised); the last BN
    of each residual branch is scaled down so that 16 blocks of He-normal weights keep activations well inside fp16."""
    from sleap_b200.nn import architectures as A
    w = A.make_synthetic_weights(cm, seed)
    rng = np.random.default_rng(seed + 1)
    for L in cm.layers:
        if L["kind"] in ("conv", "tconv"):
            w[L["name"]]["bias"] = rng.normal(0, 0.1, size=L["cout"]).astype(np.float32)
        else:
            c = L["c"]
            g = 0.3 if L["name"].endswith("_3_bn") else 1.0
            w[L["name"]] = dict(gamma=(g * rng.uniform(0.5, 1.5, c)).astype(np.float32), beta=rng.normal(0, 0.1, c).astype(np.float32),
                                mean=rng.normal(0, 0.1, c).astype(np.float32), var=rng.uniform(0.5, 1.5, c).astype(np.float32))
    return w


def _model(spec, in_ch, seed, precision):
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    w = _weights(A.compile_model(spec, in_ch), seed)
    return DeviceModel(spec, w, input_channels=in_ch, precision=precision), w


def _oracle(imgs, spec, w, in_ch):
    x = opre.preprocess(imgs, ensure_gray=(in_ch == 1), pad_stride=spec["backbone_cfg"]["max_stride"])
    return bo.model_forward(x, spec, w)


def _check(got, want, precision):
    for g, x in zip(got, want):
        assert g.shape == x.shape
        err = np.abs(g - x).max() / np.abs(x).max()
        assert err <= BAR[precision], err


@pytest.mark.parametrize("precision", [1, 0, 2])
@pytest.mark.parametrize("up", ["tconv_concat", "interp_add", "tconv_add_nobn"])
def test_resnet50_forward(up, precision):
    """Pad-3 stem after ImageNet preprocessing, zero-padded 3x3 / s2 pool, stride-2 1x1 convs, residual adds (projection
    and identity shortcuts), k4 transposed convs with / without BN, concat and add skips, bilinear upsampling."""
    spec = _resnet_spec(up=up)
    model, w = _model(spec, 3, 11, precision)
    imgs = np.random.default_rng(2).integers(0, 256, size=(2, 150, 160, 3), dtype=np.uint8)   # bottom padding to 160
    _check(model.forward(imgs), _oracle(imgs, spec, w, 3), precision)


@pytest.mark.parametrize("precision", [1, 0, 2])
def test_resnet50_max_stride16_random_weights(precision):
    """max_stride 16: conv5 keeps stride 1 (its dilation only reaches 1x1 convs); no ImageNet preprocessing."""
    spec = _resnet_spec(max_stride=16, weights="random")
    model, w = _model(spec, 1, 12, precision)
    imgs = np.random.default_rng(3).integers(0, 256, size=(2, 160, 160, 1), dtype=np.uint8)
    _check(model.forward(imgs), _oracle(imgs, spec, w, 1), precision)


def test_resnet50_gray_float_frames_tiled():
    """A grayscale float frame into a pretrained ResNet: tile_channels (1 -> 3) + caffe normalisation."""
    spec = _resnet_spec()
    model, w = _model(spec, 3, 13, 1)
    imgs = np.random.default_rng(4).uniform(0, 1, size=(1, 128, 128, 1)).astype(np.float32)
    _check(model.forward(imgs), _oracle(imgs, spec, w, 3), 1)


@pytest.mark.parametrize("precision", [1, 0, 2])
@pytest.mark.parametrize("interp", [False, True])
def test_leap_forward(interp, precision):
    spec = _leap_spec(interp)
    model, w = _model(spec, 1, 14, precision)
    imgs = np.random.default_rng(5).integers(0, 256, size=(2, 96, 112, 1), dtype=np.uint8)
    _check(model.forward(imgs), _oracle(imgs, spec, w, 1), precision)


def test_resnet_fused_residual_matches_unfused_store():
    """Asking for a fused conv's own output makes that forward store it and run the ADD op instead of the epilogue add;
    the heads agree with the fused run to fp16 rounding."""
    from ctypes import c_void_p
    from sleap_b200._lib import ptr
    spec = _resnet_spec(up="interp_add")
    model, w = _model(spec, 3, 15, 0)
    imgs = np.random.default_rng(6).integers(0, 256, size=(1, 128, 128, 3), dtype=np.uint8)
    fused = model.forward(imgs)
    rec = next(r for r in model.cm.records if r[0] == 1 and r[11] & 128)          # a CONV carrying a residual
    own = int(rec[6])
    brec = next(r for r in model.cm.records if r[0] == 0 and r[1] == own)
    outs = [np.zeros_like(f) for f in fused] + [np.zeros((1, 128 // int(brec[2]), 128 // int(brec[2]), int(brec[3])), np.float32)]
    ids = np.asarray([model.cm.head_buffers[h["name"]] for h in spec["heads"]] + [own], np.int32)
    ptrs = (c_void_p * len(outs))(*[o.ctypes.data for o in outs])
    model.handle.call("sb_model_forward", model.model_id, ptr(np.ascontiguousarray(imgs)), 1, 1, len(outs), ptr(ids), ptrs)
    assert np.abs(outs[-1]).max() > 0
    for g, x in zip(outs, fused):
        assert np.abs(g - x).max() <= 5e-3 * np.abs(x).max()


def _write_model_dir(d, spec, cfg_model, w, in_ch):
    from sleap_b200.nn.model import save_weights_npz
    os.makedirs(d, exist_ok=True)
    cfg = {"model": cfg_model, "data": {"preprocessing": {"input_scaling": 1.0, "pad_to_stride": None, "ensure_rgb": in_ch == 3,
                                                          "ensure_grayscale": in_ch == 1},
                                        "labels": {"skeletons": []}}}
    with open(os.path.join(d, "training_config.json"), "w") as f:
        json.dump(cfg, f)
    save_weights_npz(os.path.join(d, "best_model.npz"), w)


def _resnet_cfg_model(heads_cfg):
    return {"backbone": {"resnet": dict(version="ResNet50", weights="frozen", max_stride=32, output_stride=4,
                                        upsampling=dict(method="transposed_conv", skip_connections="concatenate", block_stride=2,
                                                        filters=64, filters_rate=1, refine_convs=2, batch_norm=True,
                                                        transposed_conv_kernel_size=4)),
                         "unet": None, "hourglass": None, "leap": None, "pretrained_encoder": None},
            "heads": heads_cfg}


def test_resnet_bottomup_from_model_paths(tmp_path):
    """A ResNet50 bottom-up model folder (training_config.json + best_model.npz with Keras layer names) through the public
    predictor: the device output equals the oracle post-processing of the device's own maps."""
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.inference import Predictor
    nodes, edges = synth.FLIES13_NODES, synth.FLIES13_EDGES
    heads_cfg = {"multi_instance": {"confmaps": {"part_names": nodes, "sigma": 2.5, "output_stride": 4},
                                    "pafs": {"edges": [list(e) for e in edges], "sigma": 5, "output_stride": 8}}}
    cfg_model = _resnet_cfg_model(heads_cfg)
    spec = A.spec_from_config(cfg_model)
    w = _weights(A.compile_model(spec, 3), 21)
    _write_model_dir(str(tmp_path / "bu"), spec, cfg_model, w, 3)
    imgs = np.random.default_rng(7).integers(0, 256, size=(2, 192, 192, 3), dtype=np.uint8)
    pred = Predictor.from_model_paths(str(tmp_path / "bu"), peak_threshold=0.2, batch_size=2, max_peaks_per_sample=4096,
                                      max_node_peaks=64, max_instances_per_frame=128)
    model = pred.inference_model.bottomup_layer.keras_model
    cms, pafs = model.forward(imgs)
    thr = float(np.quantile(cms, 0.999))
    layer = pred.inference_model.bottomup_layer
    layer.peak_threshold = thr
    layer.return_paf_graph = True
    out = pred.inference_model.predict_on_batch(imgs)
    p, v, si, ci = opf.find_local_peaks(cms, thr, "integral", 5)
    assert len(p) > 4
    p = (p * np.float32(4)).astype(np.float32)
    peaks = [p[si == b] for b in range(2)]; vals = [v[si == b] for b in range(2)]; chans = [ci[si == b] for b in range(2)]
    winst, wps, wisc, wei, wepi, wls = opg.PAFScorer(nodes, edges, 8).predict(pafs, peaks, vals, chans)
    for b in range(2):
        assert out["flags"][b] == 0
        assert_array_equal(out["peak_channel_inds"][b], chans[b])
        n = out["n_valid"][b]
        assert n == len(winst[b])
        assert_allclose(out["instance_peaks"][b, :n], winst[b], atol=4e-4, rtol=0, equal_nan=True)
        assert_allclose(out["instance_scores"][b, :n], wisc[b], atol=1e-4, rtol=0)
    assert len(pred.predict(imgs, make_labels=True)) == 2


def _fetch(model, imgs, buf_ids):
    """Forward pass returning whole op-list buffers (fp16 buffers converted to float32)."""
    from ctypes import c_void_p
    from sleap_b200._lib import ptr
    imgs = np.ascontiguousarray(imgs)
    B, H, W, C = imgs.shape
    model.configure(B, H, W, C)
    outs = []
    for bid in buf_ids:
        rec = next(r for r in model.cm.records if r[0] == 0 and r[1] == bid)
        nh, nw = model.net_hw(H, W)
        outs.append(np.zeros((B, nh // int(rec[2]), nw // int(rec[2]), int(rec[3])), np.float32))
    ptrs = (c_void_p * len(outs))(*[o.ctypes.data for o in outs])
    model.handle.call("sb_model_forward", model.model_id, ptr(imgs), int(imgs.dtype == np.uint8), B, len(outs),
                      ptr(np.asarray(buf_ids, np.int32)), ptrs)
    return outs


def _op_kinds(model, B, H, W, C):
    """Per-op kind of one forward pass (sb_model_profile_ops): 1 tensor-core conv, 2 CUDA-core conv, 0 other."""
    from ctypes import byref, c_int, c_void_p
    import torch
    from sleap_b200 import _lib
    model.configure(B, H, W, C)
    dev = torch.zeros((B, H, W, C), dtype=torch.uint8, device="cuda")
    n = len(model.cm.records)
    ms, kind, fl = np.zeros(n, np.float32), np.zeros(n, np.int32), np.zeros(n, np.float64)
    cnt = c_int(0)
    model.handle.call("sb_model_profile_ops", model.model_id, c_void_p(dev.data_ptr()), B, n, _lib.ptr(ms), _lib.ptr(kind),
                      _lib.ptr(fl), byref(cnt))
    return kind[:cnt.value]


@pytest.mark.parametrize("precision", [1, 0, 2])
def test_resnet_gray_trained_fed_rgb_frames(precision):
    """A pretrained ResNet trained on grayscale frames (1-channel Keras input) fed colour frames: rgb -> gray, then
    tile_channels, then caffe normalisation -- against the oracle fed the rgb_to_grayscale frames."""
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    spec = _resnet_spec()
    w = _weights(A.compile_model(spec, 1), 16)
    model = DeviceModel(spec, w, input_channels=1, precision=precision)
    imgs = np.random.default_rng(8).integers(0, 256, size=(2, 128, 160, 3), dtype=np.uint8)
    _check(model.forward(imgs), _oracle(imgs, spec, w, 1), precision)


@pytest.mark.parametrize("case", ["rgb_u8", "rgb_float", "gray_u8_tiled", "gray_model_rgb_u8", "random_weights_gray_u8"])
def test_resnet_stem_on_tensor_cores_matches_cuda_cores(case, monkeypatch):
    """The pad-3 ResNet stem (7x7 / s2) through the space-to-depth view with the ImageNet preprocessing folded in, against
    PREPROCESS + the CUDA-core conv on the same fp16 path (<= 2e-3 of the max); the op runs on the tensor cores."""
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    spec = _resnet_spec(weights="random" if case.startswith("random") else "frozen")
    in_ch = 1 if case in ("gray_model_rgb_u8", "random_weights_gray_u8") else 3
    w = _weights(A.compile_model(spec, in_ch), 17)
    rng = np.random.default_rng(9)
    fc = 1 if case in ("gray_u8_tiled", "random_weights_gray_u8") else 3
    imgs = (rng.uniform(0, 1, size=(2, 150, 176, fc)).astype(np.float32) if case == "rgb_float"
            else rng.integers(0, 256, size=(2, 150, 176, fc), dtype=np.uint8))          # bottom / right padding to 160 x 192
    tc = DeviceModel(spec, w, input_channels=in_ch, precision=0)
    stem = next(i for i, r in enumerate(tc.cm.records) if r[0] == ol_CONV)
    stem_out = int(tc.cm.records[stem][6])
    got = _fetch(tc, imgs, [stem_out])[0]
    assert _op_kinds(tc, 2, 150, 176, fc)[stem - tc.cm.n_buffers] == 1        # the stem ran on the tensor cores
    monkeypatch.setenv("SB_DISABLE_STEM_VIEW", "1")
    cc = DeviceModel(spec, w, input_channels=in_ch, precision=0)
    want = _fetch(cc, imgs, [stem_out])[0]
    assert _op_kinds(cc, 2, 150, 176, fc)[stem - cc.cm.n_buffers] == 2
    assert np.abs(got - want).max() <= 2e-3 * np.abs(want).max()


ol_CONV = 1


@pytest.mark.parametrize("up", ["tconv_concat", "tconv_add_nobn"])
def test_resnet_fp16_forms_engage(up, monkeypatch):
    """Every conv of an fp16 ResNet runs on the tensor cores (stem view, stride-2 1x1, k4 transposed convs included), and
    each fused residual ADD saves one launch against SB_DISABLE_RES_FUSION=1."""
    spec = _resnet_spec(up=up)
    model, w = _model(spec, 3, 18, 0)
    kinds = _op_kinds(model, 2, 160, 160, 3)
    ops = [r for r in model.cm.records if r[0] != 0]
    conv_kinds = [int(k) for k, r in zip(kinds, ops) if r[0] in (1, 2)]
    assert conv_kinds and all(k == 1 for k in conv_kinds), conv_kinds
    assert any(r[0] == 1 and r[10] == 2 and r[9] == 1 for r in ops) and any(r[0] == 2 and r[9] == 4 for r in ops)
    n_res = sum(1 for r in ops if r[0] == 1 and r[11] & 128)
    imgs = np.random.default_rng(10).integers(0, 256, size=(2, 160, 160, 3), dtype=np.uint8)
    fused = model.forward(imgs)
    l0 = model.handle.gpu_launches(); model.forward(imgs); l_fused = model.handle.gpu_launches() - l0
    monkeypatch.setenv("SB_DISABLE_RES_FUSION", "1")
    plain, _ = _model(spec, 3, 18, 0)
    unf = plain.forward(imgs)
    l0 = plain.handle.gpu_launches(); plain.forward(imgs); l_plain = plain.handle.gpu_launches() - l0
    assert n_res >= 16 and l_plain - l_fused == n_res, (l_plain, l_fused, n_res)
    for a, b in zip(fused, unf):
        assert np.abs(a - b).max() <= 5e-3 * np.abs(b).max()


def test_resnet_topdown_from_model_paths(tmp_path):
    """Centroid UNet + centered-instance pretrained ResNet (trained on grayscale, fed colour frames) through
    Predictor.from_model_paths: centroids and instance peaks equal the oracle chain on the device's own maps, and the
    instance net on the crops (3-channel caffe preprocessing after rgb -> gray) matches the ResNet oracle."""
    from oracle import tf_ops
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.inference import Predictor
    ccfg = {"backbone": {"unet": dict(filters=8, filters_rate=2, max_stride=16, output_stride=2, middle_block=True,
                                      up_interpolate=True, stacks=1, stem_stride=None),
                         "hourglass": None, "resnet": None, "leap": None, "pretrained_encoder": None},
            "heads": {"centroid": {"anchor_part": None, "sigma": 2.5, "output_stride": 2}}}
    icfg = _resnet_cfg_model({"centered_instance": {"anchor_part": None, "part_names": list("abcd"), "sigma": 2.5,
                                                    "output_stride": 4}})
    cspec, ispec = A.spec_from_config(ccfg), A.spec_from_config(icfg)
    cw, iw = _weights(A.compile_model(cspec, 1), 31), _weights(A.compile_model(ispec, 1), 32)
    for d, spec, cfgm, w in (("c", cspec, ccfg, cw), ("i", ispec, icfg, iw)):
        _write_model_dir(str(tmp_path / d), spec, cfgm, w, 1)
        cfg_path = tmp_path / d / "training_config.json"
        cfg = json.loads(cfg_path.read_text())
        cfg["data"]["instance_cropping"] = {"center_on_part": None, "crop_size": 64}
        cfg_path.write_text(json.dumps(cfg))
    imgs = np.random.default_rng(11).integers(0, 256, size=(2, 192, 224, 3), dtype=np.uint8)
    pred = Predictor.from_model_paths([str(tmp_path / "c"), str(tmp_path / "i")], batch_size=2, max_instances=3, precision=1)
    cmodel, imodel = pred.centroid_model, pred.confmap_model
    assert imodel.cm.input_channels == 1
    ccms = cmodel.forward(imgs)[0]
    thr = float(np.sort(ccms.reshape(-1))[-40])
    pred.inference_model.centroid_crop.peak_threshold = thr
    pred.inference_model.instance_peaks.peak_threshold = -1e9
    out = pred.inference_model.predict_on_batch(imgs)
    cp, cv, csi, _ = opf.find_local_peaks(ccms, thr, "integral", 5)
    cp = cp * np.float32(2)
    keep = []
    for s in range(2):
        idx = np.nonzero(csi == s)[0]
        if len(idx) > 3:
            idx = idx[np.argsort(-cv[idx], kind="stable")[:3]]
        keep.append(idx)
    keep = np.concatenate(keep)
    cp, cv, csi = cp[keep], cv[keep], csi[keep]
    assert len(cp) > 0
    crops = tf_ops.crop_bboxes(imgs, tf_ops.make_centered_bboxes(cp, 64, 64), csi)
    dcms = imodel.forward(crops)[0]
    ocms = bo.model_forward(opre.preprocess(crops, ensure_gray=True, pad_stride=32), ispec, iw)[0]
    assert np.abs(dcms - ocms).max() <= 1e-4 * np.abs(ocms).max()
    wp, wv = opf.find_global_peaks(dcms, -1e9, "integral", 5)
    wp = wp * np.float32(4) + (cp - np.float32(32))[:, None, :]
    for s in range(2):
        n = int(out["n_valid"][s])
        assert n == int((csi == s).sum())
        assert_allclose(out["centroids"][s, :n], cp[csi == s], atol=1e-4)
        assert_allclose(out["instance_peaks"][s, :n], wp[csi == s], atol=5e-4, equal_nan=True)
