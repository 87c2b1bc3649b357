"""The fused first block k_conv01 (sb_conv01.cu) at the geometries of its 64x16 image-row items and its conv0 -> conv1
plane ring: widths at, below and between multiples of the 64-pixel item, heights off the 16-row item, three frames, and
a map on which every CTA walks many items and so wraps the ring many times."""
import numpy as np
import pytest
from numpy.testing import assert_allclose

from test_gpu_first_block import _first_block, _reference, _run

pytestmark = pytest.mark.gpu

CASES = {
    "width_64": ((16, 64), 1, False, True),            # exactly one item
    "width_100": ((48, 100), 2, False, True),          # last item column half outside the image
    "width_200": ((40, 200), 1, True, True),
    "width_below_64": ((32, 40), 1, False, False),
    "height_36": ((36, 128), 2, False, True),          # last item row partly below the image
    "b3": ((64, 192), 3, False, True),
    "ring_wraps": ((1024, 1024), 2, False, True),      # ~16 items per CTA on a 132-SM part
}


@pytest.mark.parametrize("case", list(CASES))
def test_first_block_rows(case, monkeypatch):
    (H, W), B, as_float, relu = CASES[case]
    ops, blob, imgs, xin, weights = _first_block(H, W, B, as_float, relu, seed=H * 37 + W + B)
    got, n_fused = _run(ops, blob, imgs, as_float, True, monkeypatch)
    sep, n_sep = _run(ops, blob, imgs, as_float, False, monkeypatch)
    assert n_fused < n_sep                               # the fused kernel really ran
    assert np.array_equal(got[0], got[1])                # the second launch computes the same thing
    want = _reference(xin, weights, relu)
    scale = max(1.0, float(np.abs(want).max()))
    assert_allclose(got[1], want, atol=2.5e-3 * scale, rtol=0)   # one fp16 ulp of the intermediate through 144 taps
    assert_allclose(got[1], sep[1], atol=2.5e-3 * scale, rtol=0)
    assert np.mean(np.abs(got[1] - want) > 1e-3 * scale) < 1e-3
