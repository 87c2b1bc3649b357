"""The resident-weight form of the tensor-core convolution (k_conv_wg_p, form 1 in sb_conv_tc.cu) is bit-identical to the
streaming form 0: it issues the same wgmma sequence, so each forced run must equal the form-0 run exactly, whatever the
autotuner would pick (conv_forms.forced_equal)."""
import numpy as np
import pytest

from conv_forms import conv_layer, forced_equal, model_run, resnet50_run

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("cin,cout,k,hw", [(16, 16, 3, (40, 48)), (32, 32, 3, (40, 48)), (64, 64, 3, (53, 70)),
                                           (128, 128, 3, (40, 48)), (256, 128, 3, (53, 70)), (128, 256, 3, (40, 48)), (128, 64, 3, (53, 70)),
                                           (256, 512, 3, (40, 48)), (64, 13, 1, (40, 48)), (128, 24, 1, (40, 48)),
                                           (24, 24, 3, (40, 48)), (48, 36, 3, (40, 48)), (96, 48, 3, (53, 70)),
                                           (192, 96, 3, (40, 48)), (24, 13, 1, (40, 48)),
                                           (32, 32, 5, (40, 48)), (64, 48, 7, (53, 70)), (128, 64, 5, (40, 48)), (16, 16, 7, (40, 48)),
                                           (192, 384, 3, (10, 10)), (384, 384, 3, (5, 7)), (64, 64, 3, (12, 20)), (96, 24, 1, (3, 3))])
def test_forms_single_layers(cin, cout, k, hw, B, monkeypatch, capfd):
    """fp32 output without ReLU; form 1 runs where it is eligible."""
    out = forced_equal(conv_layer(cin, cout, hw, B, k=k, relu=False, f32_out=True), 1, monkeypatch, capfd, check_ran=False)
    assert np.abs(out[0]).max() > 0


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
    out = forced_equal(model_run(spec, 1, imgs, precision), 1, monkeypatch, capfd)
    assert all(np.isfinite(o).all() and np.abs(o).max() > 0 for o in out)


@pytest.mark.parametrize("B", [1, 3])
def test_forms_resnet(B, monkeypatch, capfd):
    out = forced_equal(resnet50_run(B, 22), 1, monkeypatch, capfd)
    assert all(np.isfinite(o).all() and np.abs(o).max() > 0 for o in out)
