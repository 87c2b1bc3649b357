"""The fused transposed-conv form (k_tconv_wg_hw, form 4 in sb_conv_tc.cu) is byte-identical to the four phase launches of
the streaming form 0.

SB_FORCE_VARIANT=4 forces the fused form where it is eligible (k3 / k4 stride-2 transposed convs with C_in > 32, N tiles
of at most 128 channels covering C_out, fp16 output in the fast-epilogue shape); each case asserts from the SB_DEBUG
autotune lines that it actually ran, and compares the raw bits of every requested tensor with the SB_FORCE_VARIANT=0 run.
The cases cover several K chunks, a zero-filled last chunk (C_in = 96), several N tiles (C_out = 256 against form 0's
N = 256 tile, and 128 -> 256), maps that are not a multiple of the 16 x 16 input item and maps smaller than one item."""
from ctypes import byref, c_int, c_void_p

import numpy as np
import pytest

from test_gpu_conv_halo import _same_bits

pytestmark = pytest.mark.gpu


def _fused_vs_phases(run, monkeypatch, capfd):
    """run() with the fused form forced and with the streaming phase launches forced; the outputs must be equal bit for bit."""
    monkeypatch.setenv("SB_DEBUG", "1")
    outs = {}
    for f in ("0", "4"):
        monkeypatch.setenv("SB_FORCE_VARIANT", f)
        capfd.readouterr()
        outs[f] = run()
        err = capfd.readouterr().err
        assert ("-> tconv-fused" in err) == (f == "4"), "the fused form did not run exactly when forced"
    for a, b in zip(outs["0"], outs["4"]):
        assert _same_bits(a, b), float(np.abs(a.astype(np.float64) - b).max())
    return outs["0"]


def _tconv_layer(cin, cout, hw, B, out_slice=False, in_slice=False):
    """frame (H x W) -> conv0 (3x3, 1 -> cin) -> 2x2 max-pool -> tconv (k3 s2, cin -> cout, ReLU, the layer under test) on
    the H / 2 x W / 2 grid -> fp16 output at H x W.  out_slice / in_slice: the tconv writes / reads a channel slice of a
    wider concat buffer."""
    from sleap_b200 import _lib
    from sleap_b200.nn import oplist as ol
    rng = np.random.default_rng(5 * cin + cout)
    H, W = hw
    in_off, in_tot = (8, cin + 24) if in_slice else (0, cin)
    out_off, out_tot = (16, cout + 48) if out_slice else (0, cout)
    recs = [ol.buffer_record(0, 1, 1, 0, 1), ol.buffer_record(1, 1, cin, 0, 0), ol.buffer_record(2, 2, in_tot, 0, 0),
            ol.buffer_record(3, 1, out_tot, 0, 0), ol.preprocess_record(0, 1, 1.0, 2)]
    w0 = (rng.standard_normal((3, 3, 1, cin)) * 0.5).astype(np.float32)
    b0 = rng.normal(0, 0.1, cin).astype(np.float32)
    w1 = (rng.standard_normal((3, 3, cin, cout)) * np.sqrt(2.0 / (4 * cin))).astype(np.float32)
    b1 = rng.normal(0, 0.1, cout).astype(np.float32)
    blob = np.concatenate([w0.reshape(-1), b0, w1.reshape(-1), b1]).astype(np.float32)
    o1 = w0.size + cin
    recs.append(ol.conv_record(0, 0, 1, 1, 0, cin, 3, 1, True, 0, w0.size))
    recs.append(ol.pool_record(1, 0, cin, 2, in_off))
    recs.append(ol.tconv_record(2, in_off, cin, 3, out_off, cout, o1, o1 + w1.size))
    ops = np.ascontiguousarray(np.stack(recs).astype(np.int32))
    imgs = rng.uniform(0, 1, size=(B, H, W, 1)).astype(np.float32)

    def run():
        h = _lib.Handle(0)
        mid = c_int(-1)
        h.call("sb_load_model", _lib.ptr(ops), ops.shape[0], _lib.ptr(blob), int(blob.size), 0, byref(mid))
        h.call("sb_model_configure", mid.value, B, H, W, 1)
        out = np.zeros((B, H, W, out_tot), np.float32)
        ptrs = (c_void_p * 1)(out.ctypes.data)
        h.call("sb_model_forward", mid.value, _lib.ptr(imgs), 0, B, 1, _lib.ptr(np.asarray([3], np.int32)), ptrs)
        h.close()
        return [out[..., out_off:out_off + cout]]      # only the tconv's slice of a concat buffer is written
    return run


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("cin,cout", [(512, 256), (256, 128), (128, 64), (96, 48), (128, 256)])
def test_tconv_fused_single_layers(cin, cout, B, monkeypatch, capfd):
    """Input grid 44 x 37: partial items in both directions."""
    out = _fused_vs_phases(_tconv_layer(cin, cout, (88, 74), B), monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


@pytest.mark.parametrize("cin,cout,hw", [(256, 128, (12, 20)), (128, 64, (4, 4)), (512, 256, (30, 18))])
def test_tconv_fused_smaller_than_one_item(cin, cout, hw, monkeypatch, capfd):
    out = _fused_vs_phases(_tconv_layer(cin, cout, hw, 3), monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


@pytest.mark.parametrize("cin,cout", [(256, 128), (96, 48), (128, 256)])
def test_tconv_fused_concat_slices(cin, cout, monkeypatch, capfd):
    """The tconv reads a channel slice of one concat buffer and writes a slice of another."""
    out = _fused_vs_phases(_tconv_layer(cin, cout, (64, 80), 2, out_slice=True, in_slice=True), monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


def test_tconv_fused_c4_unet(monkeypatch, capfd):
    """The benchmark's C4 UNet at 2 x 256 x 256, whose three k3 decoder tconvs take the fused form: every output map
    byte-identical."""
    import bench
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    spec = bench.c4_spec()
    w = A.make_synthetic_weights(A.compile_model(spec, 1), bench.SEED)
    imgs = np.random.default_rng(29).integers(0, 256, size=(2, 256, 256, 1), dtype=np.uint8)

    def run():
        return [np.asarray(x) for x in DeviceModel(spec, w, input_channels=1, precision=0).forward(imgs)]
    out = _fused_vs_phases(run, monkeypatch, capfd)
    assert all(np.isfinite(o).all() and np.abs(o).max() > 0 for o in out)


def test_tconv_fused_resnet50_k4(monkeypatch, capfd):
    """ResNet50 at 2 x 128 x 96 with 4x4 transposed-conv upsampling: its k4 phases (filter columns dx of 0 and -1 / +1, box
    start rows -1 and 0) take the fused form."""
    from test_gpu_conv_forms import _model_run
    ups = dict(method="transposed_conv", skip_connections="concatenate", block_stride=2, filters=64, filters_rate=1,
               refine_convs=2, batch_norm=True, transposed_conv_kernel_size=4)
    cfg = dict(version="ResNet50", weights="frozen", max_stride=32, output_stride=4, upsampling=ups)
    heads = [dict(name="MultiInstanceConfmapsHead", channels=5, output_stride=4),
             dict(name="PartAffinityFieldsHead", channels=8, output_stride=8)]
    spec = dict(backbone="resnet", backbone_cfg=cfg, head_type="multi_instance", heads=heads, part_names=None, edges=None)
    imgs = np.random.default_rng(31).integers(0, 256, size=(2, 128, 96, 3), dtype=np.uint8)
    out = _fused_vs_phases(_model_run(spec, 3, imgs, 0), monkeypatch, capfd)
    assert all(np.isfinite(o).all() and np.abs(o).max() > 0 for o in out)
