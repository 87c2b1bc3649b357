"""The halo form's patch loader (stage_halo_patch in sb_conv_tc.cu) deals each item's 16-byte pieces over the 128 threads of
the producer warpgroup.  Forced form 2 against forced form 0, raw bits (conv_forms.forced_equal), at the shapes where that
split matters: 8-channel planes beyond C_in inside the K chunk, piece counts that 128 does not divide, maps narrower than
the 18-pixel patch or shorter than one item, and the full-size encoder layers, where each CTA wraps its ring of patch
slots many times."""
import numpy as np
import pytest

from conv_forms import conv_layer, forced_equal

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cin,cout", [(24, 32), (24, 64), (40, 16), (40, 48), (56, 32)])
def test_loader_planes_beyond_cin(cin, cout, monkeypatch, capfd):
    """C_in 24 stages 4 planes (KC 32), the last all zero fill; C_in 40 and 56 stage 8 (KC 64), 3 and 1 beyond C_in."""
    out = forced_equal(conv_layer(cin, cout, (40, 53), 2), 2, monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


@pytest.mark.parametrize("cin,cout", [(16, 48), (16, 16), (32, 48), (64, 16)])
def test_loader_uneven_piece_counts(cin, cout, monkeypatch, capfd):
    """Items of 360, 648, 720 and 2,592 pieces: the last round of cp.async leaves part of the 128 loaders idle."""
    out = forced_equal(conv_layer(cin, cout, (34, 46), 3, pool="alive"), 2, monkeypatch, capfd)
    assert all(np.abs(o).max() > 0 for o in out)


@pytest.mark.parametrize("cin,cout,hw", [(16, 32, (6, 10)), (24, 48, (5, 15)), (64, 64, (20, 12)), (32, 16, (7, 9))])
def test_loader_small_maps(cin, cout, hw, monkeypatch, capfd):
    """Maps narrower than 16 columns and shorter than one item: most of each patch is zero fill."""
    out = forced_equal(conv_layer(cin, cout, hw, 3), 2, monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


@pytest.mark.parametrize("cin,cout,hw,pool", [(16, 32, (512, 512), None), (32, 32, (512, 512), "dead"),
                                              (32, 64, (256, 256), None)])
def test_loader_full_size_layers(cin, cout, hw, pool, monkeypatch, capfd):
    """The C4 UNet's second-block convs (16 -> 32 and 32 -> 32 + pool, full output dead, at 512²) and its 32 -> 64 conv at
    256², 8 frames: about 62 items per CTA, so the ring of patch slots wraps many times."""
    out = forced_equal(conv_layer(cin, cout, hw, 8, pool=pool), 2, monkeypatch, capfd)
    assert all(np.abs(o).max() > 0 for o in out)


def test_loader_c4_unet_full_frames(monkeypatch, capfd):
    """The benchmark's C4 UNet at 8 x 1024 x 1024 with the benchmark's weights: every output map byte-identical."""
    import bench
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    spec = bench.c4_spec()
    w = A.make_synthetic_weights(A.compile_model(spec, 1), bench.SEED)
    imgs = np.random.default_rng(29).integers(0, 256, size=(8, 1024, 1024, 1), dtype=np.uint8)

    def run():
        return [np.asarray(x) for x in DeviceModel(spec, w, input_channels=1, precision=0).forward(imgs)]
    out = forced_equal(run, 2, monkeypatch, capfd)
    assert all(np.isfinite(o).all() and np.abs(o).max() > 0 for o in out)
