"""Precision 2 (split-fp16 activations / weights, three tensor-core products per term, fp32 accumulate): the wgmma
conv path must reproduce the fp32 torch-CPU oracle to the north-star tolerance (1e-4 of the map; measured ~1e-6), so
that peak indices / instance assignments of the tensor-core path agree with the fp32 reference network."""
import numpy as np
import pytest
from numpy.testing import assert_allclose

from oracle import convnet, paf_grouping as opg, peak_finding as opf, preprocess as opre, synth

pytestmark = pytest.mark.gpu

from test_gpu_model import HEADS2, UNET_CASES, _mk, _oracle_forward, _unet_spec  # noqa: E402

TOL = 5e-5     # of max(1, |map|max); measured 2.4e-5 at C4 full size on an H100.  The split arithmetic itself
               # is good to ~1e-6 (numpy emulation); what is left is the tensor core's fp32 accumulator, which truncates
               # instead of rounding: a bias of ~n_steps * 2^-25 per accumulation chain (DESIGN.md 5.7)


def _check(got, want, tol=TOL):
    worst = 0.0
    for g, x in zip(got, want):
        assert g.shape == x.shape
        worst = max(worst, float(np.abs(g - x).max() / max(1.0, np.abs(x).max())))
    assert worst <= tol, worst
    return worst


@pytest.mark.parametrize("name", list(UNET_CASES))
def test_unet_forward_split_small(name):
    """Same nets / frames as test_unet_forward_fp32 (8-filter nets: 24-channel split tensors on the tensor cores, the 4-filter
    net's 12-channel tensors and every first conv on the CUDA-core kernels with split stores; stand-alone pool,
    bilinear upsample, 7x7 stem from the fp32 frame buffer)."""
    cfg = UNET_CASES[name]
    spec = _unet_spec(cfg, HEADS2)
    model, w, cm = _mk(spec, 1, 3, precision=2)
    imgs = np.random.default_rng(0).integers(0, 256, size=(2, 61, 75, 1), dtype=np.uint8)
    got = model.forward(imgs)
    want = _oracle_forward(imgs, spec, w, 1, 1.0, cfg["max_stride"])
    _check(got, want)


@pytest.mark.parametrize("name", ["tconv", "interp"])
def test_unet_forward_split(name):
    """16-filter nets at 128x160 (the fp16 test's shapes): fused pools, concat slices, transposed convs / bilinear."""
    cfg = dict(UNET_CASES[name], filters=16, max_stride=16)
    spec = _unet_spec(cfg, HEADS2)
    model, w, cm = _mk(spec, 1, 9, precision=2)
    imgs = np.random.default_rng(3).integers(0, 256, size=(2, 128, 160, 1), dtype=np.uint8)
    got = model.forward(imgs)
    want = _oracle_forward(imgs, spec, w, 1, 1.0, cfg["max_stride"])
    _check(got, want)


def test_unet_forward_split_resize_and_rgb():
    cfg = UNET_CASES["tconv"]
    spec = _unet_spec(cfg, HEADS2)
    rng = np.random.default_rng(1)
    model, w, cm = _mk(spec, 1, 4, input_scale=0.5, precision=2)
    imgs = rng.integers(0, 256, size=(2, 96, 128, 3), dtype=np.uint8)     # rgb -> gray -> resize 0.5 -> pad (fp32 frame buffer)
    got = model.forward(imgs)
    want = _oracle_forward(imgs, spec, w, 1, 0.5, cfg["max_stride"])
    _check(got, want, 2e-4)                                               # same bar as the fp32 path's resize test
    model3, w3, _ = _mk(spec, 3, 5, precision=2)
    gray = rng.uniform(0, 1, size=(1, 64, 64, 1)).astype(np.float32)      # gray float -> rgb
    _check(model3.forward(gray), _oracle_forward(gray, spec, w3, 3, 1.0, cfg["max_stride"]))


def test_hourglass_forward_split():
    """conv -> ReLU -> BN affine epilogue, additive skips, nearest x2, 7x7 stride-2 stem, three-channel frames."""
    spec = dict(backbone="hourglass", head_type="multi_instance", part_names=None, edges=None,
                backbone_cfg=dict(stem_stride=4, max_stride=32, output_stride=4, stem_filters=16, filters=32, filter_increase=32, stacks=2),
                heads=[dict(name="MultiInstanceConfmapsHead", channels=6, output_stride=4),
                       dict(name="PartAffinityFieldsHead", channels=10, output_stride=4)])
    model, w, cm = _mk(spec, 3, 17, precision=2)
    imgs = np.random.default_rng(2).integers(0, 256, size=(2, 160, 192, 3), dtype=np.uint8)
    got = model.forward(imgs)
    want = _oracle_forward(imgs, spec, w, 3, 1.0, 32)
    _check(got, want)


def test_bottomup_predictor_split_matches_fp32_path():
    """C4-shaped bottom-up model (16 filters, stride 32 -> 4, 13 nodes / 12 edges) at 256^2: precision 2 and the fp32
    CUDA-core path give the same peak indices and instance assignments, coordinates / scores within 1e-4."""
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.inference import BottomUpPredictor
    from sleap_b200.nn.model import DeviceModel
    spec = dict(backbone="unet", head_type="multi_instance", part_names=synth.FLIES13_NODES, edges=synth.FLIES13_EDGES,
                backbone_cfg=dict(filters=16, filters_rate=2, max_stride=32, output_stride=4, middle_block=True, up_interpolate=False),
                heads=[dict(name="MultiInstanceConfmapsHead", channels=13, output_stride=4),
                       dict(name="PartAffinityFieldsHead", channels=24, output_stride=8)])
    cm = A.compile_model(spec, 1)
    w = A.make_synthetic_weights(cm, 1)
    imgs = np.random.default_rng(0).integers(0, 256, size=(2, 256, 256, 1), dtype=np.uint8)
    outs = {}
    for prec in (1, 2):
        model = DeviceModel(spec, w, input_channels=1, precision=prec)
        dcms, dpafs = model.forward(imgs)
        if prec == 1:
            thr = float(np.quantile(dcms, 0.999))
        pred = BottomUpPredictor(model, synth.FLIES13_NODES, synth.FLIES13_EDGES, peak_threshold=thr, batch_size=2,
                                 max_peaks_per_sample=2048, max_node_peaks=64, max_instances_per_frame=128)
        outs[prec] = (dcms, dpafs, pred.inference_model.predict_on_batch(imgs))
    (c1, p1, o1), (c2, p2, o2) = outs[1], outs[2]
    assert np.abs(c1 - c2).max() <= 1e-4 * max(1.0, np.abs(c1).max())
    assert np.abs(p1 - p2).max() <= 1e-4 * max(1.0, np.abs(p1).max())
    assert np.array_equal(o1["n_valid"], o2["n_valid"])
    for b in range(2):
        n = int(o1["n_valid"][b])
        assert np.array_equal(np.isnan(o1["instance_peaks"][b, :n]), np.isnan(o2["instance_peaks"][b, :n]))
        assert_allclose(o1["instance_peaks"][b, :n], o2["instance_peaks"][b, :n], atol=1e-3, equal_nan=True)
        assert_allclose(o1["instance_scores"][b, :n], o2["instance_scores"][b, :n], atol=1e-4, equal_nan=True)
