"""The fused transposed-conv form (k_tconv_wg_hw, form 4 in sb_conv_tc.cu) is byte-identical to the four phase launches of
the streaming form 0 where it is eligible: k3 / k4 stride-2 transposed convs with C_in > 32, N tiles of at most 128
channels covering C_out, fp16 output in the fast-epilogue shape (conv_forms.forced_equal, which also asserts that the
fused form runs exactly when forced).  The cases cover several K chunks, a zero-filled last chunk (C_in = 96), several N
tiles (C_out = 256 against form 0's N = 256 tile, and 128 -> 256), maps that are not a multiple of the 16 x 16 input
item and maps smaller than one item."""
import numpy as np
import pytest

from conv_forms import c4_run, forced_equal, resnet50_run, tconv_layer

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("cin,cout", [(512, 256), (256, 128), (128, 64), (96, 48), (128, 256)])
def test_tconv_fused_single_layers(cin, cout, B, monkeypatch, capfd):
    """Input grid 44 x 37: partial items in both directions."""
    out = forced_equal(tconv_layer(cin, cout, (88, 74), B), 4, monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


@pytest.mark.parametrize("cin,cout,hw", [(256, 128, (12, 20)), (128, 64, (4, 4)), (512, 256, (30, 18))])
def test_tconv_fused_smaller_than_one_item(cin, cout, hw, monkeypatch, capfd):
    out = forced_equal(tconv_layer(cin, cout, hw, 3), 4, monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


@pytest.mark.parametrize("cin,cout", [(256, 128), (96, 48), (128, 256)])
def test_tconv_fused_concat_slices(cin, cout, monkeypatch, capfd):
    """The tconv reads a channel slice of one concat buffer and writes a slice of another."""
    out = forced_equal(tconv_layer(cin, cout, (64, 80), 2, out_slice=True, in_slice=True), 4, monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


def test_tconv_fused_c4_unet(monkeypatch, capfd):
    """The benchmark's C4 UNet, whose three k3 decoder tconvs take the fused form: every output map byte-identical."""
    out = forced_equal(c4_run(29), 4, monkeypatch, capfd)
    assert all(np.isfinite(o).all() and np.abs(o).max() > 0 for o in out)


def test_tconv_fused_resnet50_k4(monkeypatch, capfd):
    """ResNet50 at 2 x 128 x 96 with 4x4 transposed-conv upsampling: its k4 phases (filter columns dx of 0 and -1 / +1, box
    start rows -1 and 0) take the fused form."""
    out = forced_equal(resnet50_run(2, 31), 4, monkeypatch, capfd)
    assert all(np.isfinite(o).all() and np.abs(o).max() > 0 for o in out)
