"""The halo form of the tensor-core convolution (k_conv_wg_h, form 2 in sb_conv_tc.cu) is byte-identical to the streaming
form 0 where it is eligible: 3x3 stride-1 convs, C_in <= 64, C_out 16..64 in the fp16 fast-epilogue shape
(conv_forms.forced_equal)."""
import numpy as np
import pytest

from conv_forms import c4_run, conv_layer, forced_equal

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("cin,cout", [(16, 16), (16, 32), (24, 48), (32, 32), (32, 64), (48, 16), (64, 64), (64, 32)])
def test_halo_single_layers(cin, cout, B, monkeypatch, capfd):
    """Maps that are not a multiple of the 16 x 16 / 16 x 8 item in either direction."""
    out = forced_equal(conv_layer(cin, cout, (40, 53), B), 2, monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


@pytest.mark.parametrize("cin,cout", [(16, 32), (64, 64)])
def test_halo_no_relu(cin, cout, monkeypatch, capfd):
    out = forced_equal(conv_layer(cin, cout, (24, 40), 2, relu=False), 2, monkeypatch, capfd)
    assert (out[0] < 0).any()


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("pool", ["dead", "alive"])
@pytest.mark.parametrize("cin,cout", [(16, 16), (32, 32), (24, 48), (64, 64)])
def test_halo_pooled(cin, cout, pool, B, monkeypatch, capfd):
    """Fused 2x2 max-pool with conv1's own output dead (stores skipped) and requested; 36 x 50 leaves partial items."""
    out = forced_equal(conv_layer(cin, cout, (36, 50), B, pool=pool), 2, monkeypatch, capfd)
    assert all(np.abs(o).max() > 0 for o in out)


@pytest.mark.parametrize("cin,cout,hw", [(16, 32, (6, 10)), (64, 64, (4, 4)), (32, 48, (14, 12))])
def test_halo_smaller_than_one_item(cin, cout, hw, monkeypatch, capfd):
    out = forced_equal(conv_layer(cin, cout, hw, 3), 2, monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


@pytest.mark.parametrize("cin,cout,pool", [(32, 32, None), (16, 64, "alive"), (48, 32, None)])
def test_halo_concat_slices(cin, cout, pool, monkeypatch, capfd):
    """conv1 reads a channel slice of one concat buffer and writes a slice of another."""
    out = forced_equal(conv_layer(cin, cout, (40, 48), 2, pool=pool, out_slice=True, in_slice=True), 2, monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


def test_halo_c4_unet(monkeypatch, capfd):
    """The benchmark's C4 UNet: every output map byte-identical."""
    out = forced_equal(c4_run(23), 2, monkeypatch, capfd)
    assert all(np.isfinite(o).all() and np.abs(o).max() > 0 for o in out)
