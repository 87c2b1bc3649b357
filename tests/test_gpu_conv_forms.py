"""The kernel forms of the tensor-core convolution (sb_conv_tc.cu) give bit-identical outputs.

SB_FORCE_VARIANT=n forces form n (0 streaming k_conv_wg, 1 persistent k_conv_wg_p with resident weights) on every launch
where it is eligible; the persistent form issues the same wgmma sequence as the streaming one, so each forced run must
equal the form-0 run exactly (np.array_equal), whatever the autotuner would pick."""
from ctypes import byref, c_int, c_void_p

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

FORMS = ("0", "1")
PICKED = {"1": "-> resident"}


def _forms(run, monkeypatch, capfd, expect_picked=()):
    """run() under each forced form; returns the outputs of form 0 and asserts the others are equal to them."""
    monkeypatch.setenv("SB_DEBUG", "1")
    outs = {}
    for f in FORMS:
        monkeypatch.setenv("SB_FORCE_VARIANT", f)
        capfd.readouterr()
        outs[f] = run()
        err = capfd.readouterr().err
        if f in expect_picked:
            assert PICKED[f] in err, f"form {f} never ran"
    for f in FORMS[1:]:
        for a, b in zip(outs["0"], outs[f]):
            assert np.array_equal(a, b), (f, float(np.abs(a.astype(np.float64) - b).max()))
    return outs["0"]


def _single_layer(cin, cout, k, hw, B):
    from sleap_b200 import _lib
    from sleap_b200.nn import oplist as ol
    rng = np.random.default_rng(cin + cout)
    H, W = hw
    recs = [ol.buffer_record(0, 1, 1, 0, 1), ol.buffer_record(1, 1, cin, 0, 0), ol.buffer_record(2, 1, cout, 1, 0),
            ol.preprocess_record(0, 1, 1.0, 1)]
    w0 = (rng.standard_normal((3, 3, 1, cin)) * 0.5).astype(np.float32)
    b0 = rng.normal(0, 0.1, cin).astype(np.float32)
    w1 = (rng.standard_normal((k, k, cin, cout)) * np.sqrt(2.0 / (k * k * cin))).astype(np.float32)
    b1 = rng.normal(0, 0.1, cout).astype(np.float32)
    blob = np.concatenate([w0.reshape(-1), b0, w1.reshape(-1), b1]).astype(np.float32)
    o1 = w0.size + cin
    recs.append(ol.conv_record(0, 0, 1, 1, 0, cin, 3, 1, True, 0, w0.size))
    recs.append(ol.conv_record(1, 0, cin, 2, 0, cout, k, 1, False, o1, o1 + w1.size))
    ops = np.ascontiguousarray(np.stack(recs).astype(np.int32))
    imgs = rng.uniform(0, 1, size=(B, H, W, 1)).astype(np.float32)

    def run():
        h = _lib.Handle(0)
        mid = c_int(-1)
        h.call("sb_load_model", _lib.ptr(ops), ops.shape[0], _lib.ptr(blob), int(blob.size), 0, byref(mid))
        h.call("sb_model_configure", mid.value, B, H, W, 1)
        outs = np.zeros((B, H, W, cout), np.float32)
        ids = np.asarray([2], np.int32)
        ptrs = (c_void_p * 1)(outs.ctypes.data)
        h.call("sb_model_forward", mid.value, _lib.ptr(imgs), 0, B, 1, _lib.ptr(ids), ptrs)
        h.close()
        return [outs]
    return run


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("cin,cout,k,hw", [(16, 16, 3, (40, 48)), (32, 32, 3, (40, 48)), (64, 64, 3, (53, 70)),
                                           (128, 128, 3, (40, 48)), (256, 128, 3, (53, 70)), (128, 256, 3, (40, 48)), (128, 64, 3, (53, 70)),
                                           (256, 512, 3, (40, 48)), (64, 13, 1, (40, 48)), (128, 24, 1, (40, 48)),
                                           (24, 24, 3, (40, 48)), (48, 36, 3, (40, 48)), (96, 48, 3, (53, 70)),
                                           (192, 96, 3, (40, 48)), (24, 13, 1, (40, 48)),
                                           (32, 32, 5, (40, 48)), (64, 48, 7, (53, 70)), (128, 64, 5, (40, 48)), (16, 16, 7, (40, 48)),
                                           (192, 384, 3, (10, 10)), (384, 384, 3, (5, 7)), (64, 64, 3, (12, 20)), (96, 24, 1, (3, 3))])
def test_forms_single_layers(cin, cout, k, hw, B, monkeypatch, capfd):
    out = _forms(_single_layer(cin, cout, k, hw, B), monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


def _model_run(spec, in_ch, imgs, precision, seed=3):
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    cm = A.compile_model(spec, in_ch)
    w = A.make_synthetic_weights(cm, seed)
    rng = np.random.default_rng(seed + 1)
    for L in cm.layers:          # non-trivial biases / BN statistics: every epilogue term is exercised
        if L["kind"] in ("conv", "tconv"):
            w[L["name"]]["bias"] = rng.normal(0, 0.1, size=L["cout"]).astype(np.float32)
        else:
            c = L["c"]
            g = 0.3 if L["name"].endswith("_3_bn") else 1.0
            w[L["name"]] = dict(gamma=(g * rng.uniform(0.5, 1.5, c)).astype(np.float32), beta=rng.normal(0, 0.1, c).astype(np.float32),
                                mean=rng.normal(0, 0.1, c).astype(np.float32), var=rng.uniform(0.5, 1.5, c).astype(np.float32))

    def run():
        return [np.asarray(x) for x in DeviceModel(spec, w, input_channels=in_ch, precision=precision).forward(imgs)]
    return run


@pytest.mark.parametrize("precision", [0, 2])
@pytest.mark.parametrize("B", [1, 3])
def test_forms_unet(B, precision, monkeypatch, capfd):
    """UNet with output stride 4: pooled convs whose full-resolution output is dead (stores skipped), k3 transposed convs,
    16 -> 512 channels; the 96 x 64 frame leaves the deepest maps (3 x 2 at stride 32) smaller than one tile."""
    cfg = dict(filters=16, filters_rate=2, max_stride=32, output_stride=4, middle_block=True, up_interpolate=False)
    heads = [dict(name="MultiInstanceConfmapsHead", channels=13, output_stride=4),
             dict(name="PartAffinityFieldsHead", channels=24, output_stride=8)]
    spec = dict(backbone="unet", backbone_cfg=cfg, head_type="multi_instance", heads=heads, part_names=None, edges=None)
    imgs = np.random.default_rng(21).integers(0, 256, size=(B, 96, 64, 1), dtype=np.uint8)
    out = _forms(_model_run(spec, 1, imgs, precision), monkeypatch, capfd, expect_picked=("1",))
    assert all(np.isfinite(o).all() and np.abs(o).max() > 0 for o in out)


@pytest.mark.parametrize("B", [1, 3])
def test_forms_resnet(B, monkeypatch, capfd):
    """ResNet50: residual 1x1 convs with the ADD in their epilogue, stride-2 1x1 convs, k4 transposed convs."""
    ups = dict(method="transposed_conv", skip_connections="concatenate", block_stride=2, filters=64, filters_rate=1,
               refine_convs=2, batch_norm=True, transposed_conv_kernel_size=4)
    cfg = dict(version="ResNet50", weights="frozen", max_stride=32, output_stride=4, upsampling=ups)
    heads = [dict(name="MultiInstanceConfmapsHead", channels=5, output_stride=4),
             dict(name="PartAffinityFieldsHead", channels=8, output_stride=8)]
    spec = dict(backbone="resnet", backbone_cfg=cfg, head_type="multi_instance", heads=heads, part_names=None, edges=None)
    imgs = np.random.default_rng(22).integers(0, 256, size=(B, 128, 96, 3), dtype=np.uint8)
    out = _forms(_model_run(spec, 3, imgs, 0), monkeypatch, capfd, expect_picked=("1",))
    assert all(np.isfinite(o).all() and np.abs(o).max() > 0 for o in out)
