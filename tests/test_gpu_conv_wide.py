"""The wide form of the tensor-core convolution (k_conv_wg_hw, form 3 in sb_conv_tc.cu) is byte-identical to the streaming
form 0 where it is eligible: 3x3 stride-1 convs with C_in > 32, N tiles of at most 128 channels covering C_out, in the
fp16 fast-epilogue shape without a residual (conv_forms.forced_equal).  The cases cover several K chunks, a zero-filled
last chunk (C_in = 96), several N tiles (C_out = 256 / 512 against form 0's N = 256 tiles), maps that are not a
multiple of the 16 x 16 / 16 x 32 item and maps smaller than one item."""
import numpy as np
import pytest

from conv_forms import c4_run, conv_layer, forced_equal, resnet50_run

pytestmark = pytest.mark.gpu

PAIRS = [(64, 128), (128, 128), (256, 128), (128, 64), (96, 48), (128, 256), (512, 256), (256, 512)]


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("cin,cout", PAIRS)
def test_wide_single_layers(cin, cout, B, monkeypatch, capfd):
    out = forced_equal(conv_layer(cin, cout, (40, 53), B), 3, monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


@pytest.mark.parametrize("cin,cout", [(128, 128), (96, 48)])
def test_wide_no_relu(cin, cout, monkeypatch, capfd):
    out = forced_equal(conv_layer(cin, cout, (24, 40), 2, relu=False), 3, monkeypatch, capfd)
    assert (out[0] < 0).any()


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("pool", ["dead", "alive"])
@pytest.mark.parametrize("cin,cout", [(64, 128), (128, 64), (256, 256)])
def test_wide_pooled(cin, cout, pool, B, monkeypatch, capfd):
    """Fused 2x2 max-pool with conv1's own output dead (stores skipped) and requested; 36 x 50 leaves partial items."""
    out = forced_equal(conv_layer(cin, cout, (36, 50), B, pool=pool), 3, monkeypatch, capfd)
    assert all(np.abs(o).max() > 0 for o in out)


@pytest.mark.parametrize("cin,cout,hw", [(128, 128, (6, 10)), (128, 64, (12, 20)), (256, 512, (4, 4))])
def test_wide_smaller_than_one_item(cin, cout, hw, monkeypatch, capfd):
    out = forced_equal(conv_layer(cin, cout, hw, 3), 3, monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


@pytest.mark.parametrize("cin,cout,pool", [(128, 128, None), (96, 48, "alive"), (128, 256, None)])
def test_wide_concat_slices(cin, cout, pool, monkeypatch, capfd):
    """conv1 reads a channel slice of one concat buffer and writes a slice of another."""
    out = forced_equal(conv_layer(cin, cout, (40, 48), 2, pool=pool, out_slice=True, in_slice=True), 3, monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


def test_wide_c4_unet(monkeypatch, capfd):
    """The benchmark's C4 UNet: every output map byte-identical."""
    out = forced_equal(c4_run(23), 3, monkeypatch, capfd)
    assert all(np.isfinite(o).all() and np.abs(o).max() > 0 for o in out)


def test_wide_resnet50(monkeypatch, capfd):
    """ResNet50 at 2 x 128 x 96: its BN-folded 3x3 bottleneck convs (64-512 channels) take the wide form."""
    out = forced_equal(resnet50_run(2, 22), 3, monkeypatch, capfd)
    assert all(np.isfinite(o).all() and np.abs(o).max() > 0 for o in out)
