"""C4 at BASELINE.json's full size (bottom-up UNet+PAF, 1024x1024x1, 8 frames per GPU): properties that do not need a
CPU run of the whole batch -- order independence, duplicate-frame equality, the fused device pipeline against the
oracle post-processing of the device's own maps, and one frame of the fp16 network against the fp32 oracle network.
"""
import os
import sys

import numpy as np
import pytest
from numpy.testing import assert_allclose, assert_array_equal

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

pytestmark = pytest.mark.gpu

# fp16-activation network vs fp32 network, max |error| / max |map| at C4 full size (fp16 rounding of the activations).
FP16_GATE = 5e-3


def _c4():
    import bench
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.inference import BottomUpPredictor
    from sleap_b200.nn.model import DeviceModel
    spec = bench.c4_spec()
    weights = A.make_synthetic_weights(A.compile_model(spec, 1), bench.SEED)
    calib = bench.make_frames(2, 500)
    m0 = DeviceModel(spec, weights, input_channels=1, precision=0)
    cms0, pafs0 = m0.forward(calib)
    weights = bench.calibrate_heads(weights, cms0, pafs0, len(calib))
    model = DeviceModel(spec, weights, input_channels=1, precision=0)
    pred = BottomUpPredictor(model, bench.NODES, bench.EDGES, peak_threshold=0.2, batch_size=8, max_peaks_per_sample=1024,
                             max_node_peaks=32, max_instances_per_frame=32)
    return bench, spec, weights, model, pred


def _per_frame(out):
    rows = []
    for b in range(len(out["n_valid"])):
        n = int(out["n_valid"][b])
        rows.append((n, np.nan_to_num(out["instance_peaks"][b, :n], nan=-1.0), np.nan_to_num(out["instance_scores"][b, :n], nan=-1.0)))
    return rows


def test_c4_full_size_properties():
    from oracle import convnet, paf_grouping as opg, peak_finding as opf, preprocess as opre
    bench, spec, weights, model, pred = _c4()
    frames = bench.make_frames(8, 4242)
    out = pred.inference_model.predict_on_batch(frames)
    assert out["instance_peaks"].shape[0] == 8 and int(out["n_valid"].sum()) > 0 and not out["flags"].any()
    # (1) order independence: every frame's result is the same wherever it sits in the batch
    rev = pred.inference_model.predict_on_batch(frames[::-1].copy())
    for a, b in zip(_per_frame(out), _per_frame(rev)[::-1]):
        assert a[0] == b[0]
        assert_array_equal(a[1], b[1])
        assert_array_equal(a[2], b[2])
    # (2) a batch of duplicates returns eight identical results
    dup = _per_frame(pred.inference_model.predict_on_batch(np.repeat(frames[3:4], 8, axis=0)))
    for d in dup[1:]:
        assert d[0] == dup[0][0]
        assert_array_equal(d[1], dup[0][1])
    assert dup[0][0] == _per_frame(out)[3][0]
    assert_array_equal(dup[0][1], _per_frame(out)[3][1])
    # (3) fused pipeline == oracle post-processing of the device's own maps (indices / assignments exact)
    cms, pafs = model.forward(frames[:2])
    p, v, si, ci = opf.find_local_peaks(cms, 0.2, "integral", 5)
    p = (p * np.float32(4)).astype(np.float32)
    winst, _, wisc, *_ = opg.PAFScorer(bench.NODES, bench.EDGES, 8).predict(
        pafs, [p[si == b] for b in range(2)], [v[si == b] for b in range(2)], [ci[si == b] for b in range(2)])
    for b in range(2):
        n = int(out["n_valid"][b])
        assert n == len(winst[b])
        assert_array_equal(np.isnan(out["instance_peaks"][b, :n]), np.isnan(winst[b]))
        assert_allclose(out["instance_peaks"][b, :n], winst[b], atol=4e-4, rtol=0, equal_nan=True)
        assert_allclose(out["instance_scores"][b, :n], wisc[b], atol=1e-4, rtol=0)
    # (4) one frame of the fp16 tensor-core network against the fp32 oracle network (torch CPU)
    x = opre.preprocess(frames[:1], ensure_gray=True, input_scale=1.0, pad_stride=32)
    ocms, opafs = convnet.model_forward(x, spec, weights)
    for got, want in ((cms[:1], ocms), (pafs[:1], opafs)):
        assert np.abs(got - want).max() <= FP16_GATE * np.abs(want).max()


def test_c4_fp16_parity_on_bench_frames():
    """The benchmarked path (fp16 activations, tensor-core convs) against the strict fp32 CUDA path and the fp32 CPU oracle on
    the bench's own 8 frames: map errors are gated at FP16_GATE of the map maximum; the fp32 path itself meets
    north_star's 1e-4 against the oracle."""
    bench, spec, weights, model, pred = _c4()
    from sleap_b200 import _lib
    frames = bench.make_frames(8, 0)
    r = bench.c4_parity(spec, weights, _lib.default_handle(), frames, pred, model, n_oracle=1)
    print(r)
    assert r["oracle"]["fp32_path_max_rel_cm"] <= 1e-4 and r["oracle"]["fp32_path_max_rel_paf"] <= 1e-4
    assert r["max_rel_cm"] <= FP16_GATE and r["max_rel_paf"] <= FP16_GATE
    assert r["oracle"]["fp16_path_max_rel_cm"] <= FP16_GATE and r["oracle"]["fp16_path_max_rel_paf"] <= FP16_GATE
    assert r["peak_index_match"] >= 0.9 and r["instance_assignment_match"] >= 0.8
    assert r["max_offset_err_px"] <= 0.25


def test_c4_split_precision_parity_on_bench_frames():
    """Precision 2 (split fp16 pairs on the tensor-core kernels) on the bench's own 8 frames at full size: north_star's
    tolerance -- confidence maps / PAFs within 1e-4 of the map maximum against the fp32 CUDA path and the fp32 CPU oracle
    (measured on an H100: 2.4e-5 / 2.5e-5), sub-pixel offsets within 1e-3 px, >= 99 % of the peaks and >= 90 % of the instances identical."""
    from sleap_b200 import _lib
    from sleap_b200.nn.inference import BottomUpPredictor
    from sleap_b200.nn.model import DeviceModel
    bench, spec, weights, _, _ = _c4()
    m2 = DeviceModel(spec, weights, input_channels=1, precision=2)
    p2 = BottomUpPredictor(m2, bench.NODES, bench.EDGES, peak_threshold=0.2, batch_size=8, max_peaks_per_sample=1024,
                           max_node_peaks=32, max_instances_per_frame=32)
    frames = bench.make_frames(8, 0)
    r = bench.c4_parity(spec, weights, _lib.default_handle(), frames, p2, m2, n_oracle=1, tag="split")
    print(r)
    assert r["max_rel_cm"] <= 1e-4 and r["max_rel_paf"] <= 1e-4
    assert r["oracle"]["split_path_max_rel_cm"] <= 1e-4 and r["oracle"]["split_path_max_rel_paf"] <= 1e-4
    # one of ~560 peaks sits within the remaining 6e-4 absolute error of the 0.2 threshold on these random-weight maps and may
    # flip (it then changes the grouping of its frame): 53 / 53 or 50 / 53 instances identical depending on the calibration run
    assert r["peak_index_match"] >= 0.99
    assert r["instance_assignment_match"] >= 0.9 and r["frames_identical_grouping"] >= 0.75
    assert r["max_offset_err_px"] <= 1e-3 and r["max_instance_score_err"] <= 1e-3


def test_c4_analytic_maps_bit_exact():
    """Network-bypassing entry at C4 map size, B=8, 5 instances per frame: indices / candidate lists / assignments bit-exact,
    coordinates and scores <= 1e-4 (north_star's bar)."""
    import bench
    from sleap_b200 import _lib
    r = bench.analytic_parity(_lib.default_handle(), n_frames=8, n_instances=5)
    print(r)
    assert r["peak_indices_bit_exact"] and r["instance_assignments_bit_exact"]
    assert r["instances"] >= 8 and r["peaks"] >= 8 * 13
    assert r["max_peak_xy_err_px"] <= 4e-4 and r["max_line_score_err"] <= 1e-4 and r["max_instance_score_err"] <= 1e-4
