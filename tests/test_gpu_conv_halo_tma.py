"""The halo-patch forms (2 and 3 in sb_conv_tc.cu) load each patch as one TMA box of a 5-D map {8 channels, W, H, C_in / 8,
frames}, and rely on its bounds for the zero fill: the channel-group bound for the planes beyond C_in, the H / W bounds
for SAME padding.  Forced form 2 / 3 against forced form 0, raw bits (conv_forms.forced_equal), where a wrong bound would
read real data: the channels after an input slice in the same buffer, the next frame's first rows below a frame's last
item, and maps as wide as the 18-pixel box or one pixel narrower."""
import numpy as np
import pytest

from conv_forms import Layer, conv_layer, forced_equal

pytestmark = pytest.mark.gpu

# (form, C_in, C_out): C_in is not a multiple of the 64-channel K chunk, so the last chunk's box reaches past C_in
SHAPES = [(2, 40, 32), (3, 72, 64)]


def sliced_input_layer(cin, cout, hw, B, in_off=8, after=24):
    """frame -> conv0 (3x3, 1 -> in_off + cin + after channels, all written and mostly nonzero) -> conv1 (3x3) reading
    only channels [in_off, in_off + cin) of conv0's buffer."""
    from sleap_b200.nn import oplist as ol
    rng = np.random.default_rng(11 * cin + cout)
    H, W = hw
    ctot = in_off + cin + after
    recs = [ol.buffer_record(0, 1, 1, 0, 1), ol.buffer_record(1, 1, ctot, 0, 0), ol.buffer_record(2, 1, cout, 0, 0),
            ol.preprocess_record(0, 1, 1.0, 1)]
    w0 = (rng.standard_normal((3, 3, 1, ctot)) * 0.5).astype(np.float32)
    b0 = rng.uniform(0.2, 0.5, ctot).astype(np.float32)           # positive: the neighbour channels survive the ReLU
    w1 = (rng.standard_normal((3, 3, cin, cout)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)
    b1 = rng.normal(0, 0.1, cout).astype(np.float32)
    blob = np.concatenate([w0.reshape(-1), b0, w1.reshape(-1), b1]).astype(np.float32)
    o1 = w0.size + ctot
    recs.append(ol.conv_record(0, 0, 1, 1, 0, ctot, 3, 1, True, 0, w0.size))
    recs.append(ol.conv_record(1, in_off, cin, 2, 0, cout, 3, 1, True, o1, o1 + w1.size))
    imgs = rng.uniform(0, 1, size=(B, H, W, 1)).astype(np.float32)
    return Layer(recs, blob, imgs, {2: (B, H, W, cout)}, [2], {}, w1, b1)


@pytest.mark.parametrize("form,cin,cout", SHAPES)
def test_channels_after_input_slice(form, cin, cout, monkeypatch, capfd):
    """The input is channels [8, 8 + C_in) of a buffer whose 24 channels after the slice are nonzero."""
    out = forced_equal(sliced_input_layer(cin, cout, (20, 37), 2), form, monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


@pytest.mark.parametrize("form,cin,cout", SHAPES)
def test_last_item_below_frame(form, cin, cout, monkeypatch, capfd):
    """H = 37: the last item row's patch reaches past H.  The frames after the first are 100 times brighter, so rows of the
    next frame read in place of the zero fill would change the first frame's bottom rows."""
    layer = conv_layer(cin, cout, (37, 40), 3)
    layer.imgs[1:] *= 100.0
    out = forced_equal(layer, form, monkeypatch, capfd)
    assert np.abs(out[0][0]).max() > 0


@pytest.mark.parametrize("W", [18, 17])
@pytest.mark.parametrize("form,cin,cout", SHAPES)
def test_map_as_wide_as_the_box(form, cin, cout, W, monkeypatch, capfd):
    """W = 18 is exactly the box width; at W = 17 the box is one pixel wider than the map."""
    out = forced_equal(conv_layer(cin, cout, (29, W), 2), form, monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0
