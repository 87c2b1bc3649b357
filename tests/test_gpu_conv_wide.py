"""The wide form of the tensor-core convolution (k_conv_wg_hw, form 3 in sb_conv_tc.cu) is byte-identical to the streaming
form 0.

SB_FORCE_VARIANT=3 forces the wide form where it is eligible (3x3 stride-1 convs with C_in > 32, N tiles of at most 128
channels covering C_out, in the fp16 fast-epilogue shape without a residual); each case asserts from the SB_DEBUG autotune
lines that it actually ran, and compares the raw bits of every requested tensor with the SB_FORCE_VARIANT=0 run.  The
cases cover several K chunks, a zero-filled last chunk (C_in = 96), several N tiles (C_out = 256 / 512 against form 0's
N = 256 tiles), maps that are not a multiple of the 16 x 16 / 16 x 32 item and maps smaller than one item."""
import numpy as np
import pytest

from test_gpu_conv_halo import _layer, _same_bits

pytestmark = pytest.mark.gpu

PAIRS = [(64, 128), (128, 128), (256, 128), (128, 64), (96, 48), (128, 256), (512, 256), (256, 512)]


def _wide_vs_streaming(run, monkeypatch, capfd):
    """run() with the wide form forced and with the streaming form forced; the outputs must be equal bit for bit."""
    monkeypatch.setenv("SB_DEBUG", "1")
    outs = {}
    for f in ("0", "3"):
        monkeypatch.setenv("SB_FORCE_VARIANT", f)
        capfd.readouterr()
        outs[f] = run()
        err = capfd.readouterr().err
        if f == "3":
            assert "-> wide" in err, "the wide form never ran"
    for a, b in zip(outs["0"], outs["3"]):
        assert _same_bits(a, b), float(np.abs(a.astype(np.float64) - b).max())
    return outs["0"]


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("cin,cout", PAIRS)
def test_wide_single_layers(cin, cout, B, monkeypatch, capfd):
    out = _wide_vs_streaming(_layer(cin, cout, (40, 53), B), monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


@pytest.mark.parametrize("cin,cout", [(128, 128), (96, 48)])
def test_wide_no_relu(cin, cout, monkeypatch, capfd):
    out = _wide_vs_streaming(_layer(cin, cout, (24, 40), 2, relu=False), monkeypatch, capfd)
    assert (out[0] < 0).any()


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("pool", ["dead", "alive"])
@pytest.mark.parametrize("cin,cout", [(64, 128), (128, 64), (256, 256)])
def test_wide_pooled(cin, cout, pool, B, monkeypatch, capfd):
    """Fused 2x2 max-pool with conv1's own output dead (stores skipped) and requested; 36 x 50 leaves partial items."""
    out = _wide_vs_streaming(_layer(cin, cout, (36, 50), B, pool=pool), monkeypatch, capfd)
    assert all(np.abs(o).max() > 0 for o in out)


@pytest.mark.parametrize("cin,cout,hw", [(128, 128, (6, 10)), (128, 64, (12, 20)), (256, 512, (4, 4))])
def test_wide_smaller_than_one_item(cin, cout, hw, monkeypatch, capfd):
    out = _wide_vs_streaming(_layer(cin, cout, hw, 3), monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


@pytest.mark.parametrize("cin,cout,pool", [(128, 128, None), (96, 48, "alive"), (128, 256, None)])
def test_wide_concat_slices(cin, cout, pool, monkeypatch, capfd):
    """conv1 reads a channel slice of one concat buffer and writes a slice of another."""
    out = _wide_vs_streaming(_layer(cin, cout, (40, 48), 2, pool=pool, out_slice=True, in_slice=True), monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


def test_wide_c4_unet(monkeypatch, capfd):
    """The benchmark's C4 UNet (16 -> 512 channels) at 2 x 256 x 256: every output map byte-identical."""
    import bench
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    spec = bench.c4_spec()
    w = A.make_synthetic_weights(A.compile_model(spec, 1), bench.SEED)
    imgs = np.random.default_rng(23).integers(0, 256, size=(2, 256, 256, 1), dtype=np.uint8)

    def run():
        return [np.asarray(x) for x in DeviceModel(spec, w, input_channels=1, precision=0).forward(imgs)]
    out = _wide_vs_streaming(run, monkeypatch, capfd)
    assert all(np.isfinite(o).all() and np.abs(o).max() > 0 for o in out)


def test_wide_resnet50(monkeypatch, capfd):
    """ResNet50 at 2 x 128 x 96: its BN-folded 3x3 bottleneck convs (64-512 channels) take the wide form."""
    from test_gpu_conv_forms import _model_run
    ups = dict(method="transposed_conv", skip_connections="concatenate", block_stride=2, filters=64, filters_rate=1,
               refine_convs=2, batch_norm=True, transposed_conv_kernel_size=4)
    cfg = dict(version="ResNet50", weights="frozen", max_stride=32, output_stride=4, upsampling=ups)
    heads = [dict(name="MultiInstanceConfmapsHead", channels=5, output_stride=4),
             dict(name="PartAffinityFieldsHead", channels=8, output_stride=8)]
    spec = dict(backbone="resnet", backbone_cfg=cfg, head_type="multi_instance", heads=heads, part_names=None, edges=None)
    imgs = np.random.default_rng(22).integers(0, 256, size=(2, 128, 96, 3), dtype=np.uint8)
    out = _wide_vs_streaming(_model_run(spec, 3, imgs, 0), monkeypatch, capfd)
    assert all(np.isfinite(o).all() and np.abs(o).max() > 0 for o in out)
