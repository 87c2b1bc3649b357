"""Post-processing kernels (sb_post.cu, sb_topdown.cu) at the shapes, capacities and branches the comfortable-size
parity tests do not reach, against the oracle restatement: indices, candidate lists and assignments bit-exact,
coordinates and scores within 1e-4 (times the output stride where the oracle's points are scaled after rounding)."""
import numpy as np
import pytest
from numpy.testing import assert_allclose, assert_array_equal

from oracle import convnet, paf_grouping as opg, peak_finding as opf, preprocess as opre, tf_ops

pytestmark = pytest.mark.gpu

TOL = 1e-4
FLAG_NODE_PEAKS_TRUNCATED, FLAG_INSTANCES_TRUNCATED = 2, 4


@pytest.fixture(scope="module")
def pf():
    from sleap_b200.nn import peak_finding
    return peak_finding


def _blobs(H, W, pts, vals, sigma=1.2):
    """One channel: max of Gaussian blobs of height vals[i] centred on pts[i] = (x, y)."""
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float32)
    m = np.zeros((H, W), np.float32)
    for (x, y), v in zip(pts, vals):
        m = np.maximum(m, np.float32(v) * np.exp(-((xx - x) ** 2 + (yy - y) ** 2) / np.float32(2 * sigma ** 2)))
    return m.astype(np.float32)


def _border_cms(seed, B, H, W, C):
    """Peaks next to every border and corner (sub-pixel centres), some inside; light noise."""
    rng = np.random.default_rng(seed)
    cms = np.zeros((B, H, W, C), np.float32)
    edge = [(0.2, 0.3), (W - 1.3, 0.4), (0.4, H - 1.2), (W - 1.1, H - 1.4), (W / 2 + 0.3, 0.1), (0.1, H / 2 + 0.4),
            (W - 1.0, H / 2 - 0.3), (W / 2 - 0.2, H - 1.0), (1.6, 2.3), (W - 2.7, H - 2.2)]
    for b in range(B):
        for c in range(C):
            inner = rng.uniform([4, 4], [W - 5, H - 5], size=(3, 2))
            pts = np.concatenate([np.asarray(edge, np.float32), inner]) + rng.uniform(-0.2, 0.2, size=(len(edge) + 3, 2))
            pts = np.clip(pts, 0, [W - 1, H - 1])
            cms[b, :, :, c] = _blobs(H, W, pts, rng.uniform(0.5, 1.0, len(pts)))
    return (cms + rng.normal(0, 0.01, cms.shape)).astype(np.float32)


def _same_local(a, b):
    for x, y in zip(a, b):
        assert_array_equal(x, y)


# ---------------------------------------------------------------------------------------------------------------------
# refinement patches
@pytest.mark.parametrize("patch", [9, 11, 13])
@pytest.mark.parametrize("scan", ["vector", "scalar"])
def test_local_refinement_patches(pf, patch, scan, monkeypatch):
    """Patch 9 / 11 use sample rows 2 and 3 of refine_offset_warp, 13 the scalar refine_offset in k_local_emit."""
    if scan == "scalar":
        monkeypatch.setenv("SB_DISABLE_SCAN_V", "1")
    cms = _border_cms(patch, 2, 40, 52, 3)
    want = opf.find_local_peaks(cms, 0.2, "integral", patch)
    got = pf.find_local_peaks(cms, 0.2, "integral", patch)
    assert len(want[0]) > 20
    for k in (1, 2, 3):
        assert_array_equal(got[k], want[k])
    assert_array_equal(np.isnan(got[0]), np.isnan(want[0]))
    assert_allclose(got[0], want[0], atol=TOL, rtol=0, equal_nan=True)


@pytest.mark.parametrize("patch", [9, 11, 13])
def test_global_refinement_patches(pf, patch):
    cms = _border_cms(100 + patch, 3, 36, 44, 5)
    for b in range(3):          # one global maximum per (sample, channel), each against a different border
        for c in range(5):
            x, y = [(0, 0), (43, 17), (20, 35), (0, 35), (43, 0)][(b + c) % 5]
            cms[b, y, x, c] = 2.0
    want = opf.find_global_peaks(cms, 0.2, "integral", patch)
    got = pf.find_global_peaks(cms, 0.2, "integral", patch)
    assert_array_equal(got[1], want[1])
    assert_array_equal(np.isnan(got[0]), np.isnan(want[0]))
    assert_allclose(got[0], want[0], atol=TOL, rtol=0, equal_nan=True)


# ---------------------------------------------------------------------------------------------------------------------
# ordered scan (k_local_scan) == atomic vector scan (k_local_scan_v)
def _both_scans(pf, monkeypatch, cms, threshold, refinement=None, max_peaks=None):
    monkeypatch.delenv("SB_DISABLE_SCAN_V", raising=False)
    a = pf._local(cms, threshold, refinement, 5, None, None, max_peaks_per_sample=max_peaks)
    monkeypatch.setenv("SB_DISABLE_SCAN_V", "1")
    b = pf._local(cms, threshold, refinement, 5, None, None, max_peaks_per_sample=max_peaks)
    monkeypatch.delenv("SB_DISABLE_SCAN_V")
    _same_local(a, b)
    return a


def _tall_centroid_map():
    """1 x 1024 x 1024 x 1: an isolated peak on every row (adjacent rows 37 columns apart, so every row-chunk boundary is
    straddled), vertical and horizontal two-pixel plateaus across every 4th row boundary, pixels exactly at the
    threshold 0.25 and pixels one ulp above it."""
    H = W = 1024
    rng = np.random.default_rng(4)
    m = rng.uniform(0.0, 0.1, size=(H, W)).astype(np.float32)
    ys = np.arange(H)
    m[ys, 1 + (37 * ys) % 500] = rng.uniform(0.3, 1.0, H).astype(np.float32)
    for y in range(3, H - 1, 4):
        x = 600 + (y % 300)
        m[y, x] = m[y + 1, x] = np.float32(0.7)          # vertical plateau across the y | y + 1 boundary
        m[y, x + 100] = m[y, x + 101] = np.float32(0.6)  # horizontal plateau
    m[::16, 1010] = np.float32(0.25)                     # exactly the threshold: not a peak (strict >)
    m[5::16, 1015] = np.nextafter(np.float32(0.25), np.float32(1))          # one ulp above: a peak
    return m[None, :, :, None].astype(np.float32)


def test_scans_agree_on_tall_centroid_map(pf, monkeypatch):
    cms = _tall_centroid_map()
    got = _both_scans(pf, monkeypatch, cms, 0.25, "integral")
    want = opf.find_local_peaks(cms, 0.25, "integral", 5)
    assert len(want[0]) == 1024 + 64
    for k in (1, 2, 3):
        assert_array_equal(got[k], want[k])
    assert_allclose(got[0], want[0], atol=TOL, rtol=0)
    cut = _both_scans(pf, monkeypatch, cms, 0.25, None, max_peaks=100)          # truncation keeps tf.where order
    full = opf.find_local_peaks(cms, 0.25, None, 5)
    assert_array_equal(cut[0], full[0][:100])
    assert_array_equal(cut[1], full[1][:100])


def _edge_case_cms(shape):
    B, H, W, C = shape
    cms = _border_cms(sum(shape), B, H, W, C)
    cms[0, 10, 10:12, 0] = 0.95                         # plateau: no peak
    cms[-1, H // 2, W // 2, C - 1] = np.float32(0.2)    # exactly the threshold
    return cms


def _check_local_and_truncation(cms, got, want, full, cut, cap):
    for k in (1, 2, 3):
        assert_array_equal(got[k], want[k])
    assert_allclose(got[0], want[0], atol=TOL, rtol=0, equal_nan=True)
    for b in range(cms.shape[0]):                       # the cut keeps each sample's first peaks in tf.where order
        sel = full[2] == b
        k = int((cut[2] == b).sum())
        assert k == min(int(sel.sum()), cap)
        assert_array_equal(cut[0][cut[2] == b], full[0][sel][:k])


@pytest.mark.parametrize("shape", [(2, 37, 53, 3), (1, 61, 47, 5), (3, 33, 31, 1)])
def test_ordered_scan_odd_rows_match_oracle(pf, shape):
    """W * C % 4 != 0: only the ordered scan (k_local_scan) can take these maps."""
    cms = _edge_case_cms(shape)
    want = opf.find_local_peaks(cms, 0.2, "local", 5)
    got = pf.find_local_peaks(cms, 0.2, "local", 5)
    cap = max(1, len(want[0]) // 2 // shape[0])
    full = pf._local(cms, 0.2, None, 5, None, None)
    cut = pf._local(cms, 0.2, None, 5, None, None, max_peaks_per_sample=cap)
    _check_local_and_truncation(cms, got, want, full, cut, cap)


def test_scans_agree_and_match_oracle(pf, monkeypatch):
    """W * C % 4 == 0: the vector scan by default, the ordered scan under SB_DISABLE_SCAN_V=1; identical outputs, also
    under a max_peaks_per_sample cut."""
    shape = (2, 64, 64, 13)
    B = shape[0]
    cms = _edge_case_cms(shape)
    got = _both_scans(pf, monkeypatch, cms, 0.2, "local")
    want = opf.find_local_peaks(cms, 0.2, "local", 5)
    n = len(want[0]) // 2
    cut = _both_scans(pf, monkeypatch, cms, 0.2, None, max_peaks=max(1, n // B))
    full = pf._local(cms, 0.2, None, 5, None, None)
    _check_local_and_truncation(cms, got, want, full, cut, max(1, n // B))


# ---------------------------------------------------------------------------------------------------------------------
# global peaks
@pytest.mark.parametrize("C", [1, 3, 7, 13, 24, 100, 255, 256])
def test_global_channels_and_chunk_ties(pf, C):
    """C that does not divide 256 leaves threads of k_global_partial idle; equal maxima sit in different row chunks
    (first row and first column with the maximum win, independently)."""
    rng = np.random.default_rng(C)
    B, H, W = 2, 300, 24
    cms = rng.uniform(0, 0.5, size=(B, H, W, C)).astype(np.float32)
    for b in range(B):
        for c in range(C):
            y1, y2 = rng.choice(H, 2, replace=False)
            x1, x2 = rng.choice(W, 2, replace=False)
            cms[b, y1, x1, c] = cms[b, y2, x2, c] = np.float32(0.9)
            if c % 3 == 0:
                cms[b, H - 1, W - 1, c] = np.float32(0.9)
    cms[0, :, :, 0] = 0.1                                # below threshold: NaN point
    for ref in (None, "integral"):
        want = opf.find_global_peaks(cms, 0.2, ref, 5)
        got = pf.find_global_peaks(cms, 0.2, ref, 5)
        assert_array_equal(got[1], want[1])
        assert_array_equal(np.isnan(got[0]), np.isnan(want[0]))
        assert_allclose(got[0], want[0], atol=TOL, rtol=0, equal_nan=True)
    rough = opf.find_global_peaks_rough(cms, 0.2)
    assert_array_equal(np.nan_to_num(pf.find_global_peaks_rough(cms, 0.2)[0], nan=-1), np.nan_to_num(rough[0], nan=-1))


def test_global_257_channels_raises(pf):
    from sleap_b200._lib import SleapB200Error
    with pytest.raises(SleapB200Error, match="C > 256"):
        pf.find_global_peaks(np.zeros((1, 8, 8, 257), np.float32), 0.2)


# ---------------------------------------------------------------------------------------------------------------------
# LSAP against SciPy
def _lsap_cases():
    rng = np.random.default_rng(12)
    mats = []
    sizes = [(n, m) for n in (1, 2, 7, 16, 31, 64) for m in (1, 5, 16, 33, 64)] + [(128, 128), (100, 128), (128, 90), (127, 3)]
    for n, m in sizes:
        mats.append(rng.normal(size=(n, m)).astype(np.float32))
        mats.append(rng.integers(-2, 3, size=(n, m)).astype(np.float32))          # many ties
        mats.append(rng.integers(0, 2, size=(n, m)).astype(np.float32))           # 0 / 1
    for n, m in [(8, 8), (64, 64), (40, 64), (64, 40), (128, 128)]:
        mats.append(np.full((n, m), 0.5, np.float32))                             # all equal
        a = rng.normal(size=(n, m)).astype(np.float32)
        a[rng.uniform(size=a.shape) < 0.2] = np.nan                               # scattered NaN
        mats.append(a)
        b = rng.integers(-1, 2, size=(n, m)).astype(np.float32)
        b[rng.uniform(size=b.shape) < 0.3] = np.nan
        mats.append(b)
    for n, m in [(20, 30), (30, 20), (64, 64)]:
        a = rng.normal(size=(n, m)).astype(np.float32); a[3, :] = np.nan          # NaN row
        mats.append(a)
        a = rng.normal(size=(n, m)).astype(np.float32); a[:, 5] = np.nan          # NaN column
        mats.append(a)
        a = rng.normal(size=(n, m)).astype(np.float32); a[:, : min(n, m) // 2] = np.nan   # infeasible in one orientation
        mats.append(a)
        a = rng.normal(size=(n, m)).astype(np.float32); a[: min(n, m) // 2 + 1, :] = np.nan
        mats.append(a)
    return mats


def test_lsap_matches_scipy_at_production_sizes():
    from scipy.optimize import linear_sum_assignment
    from sleap_b200.nn import paf_grouping as pg
    mats = _lsap_cases()
    sols = pg._lsap_scores(mats)
    n_empty = 0
    for i, (mat, (r, c, s)) in enumerate(zip(mats, sols)):
        cost = np.where(np.isnan(mat), np.float32(np.inf), -mat).astype(np.float32)
        try:
            wr, wc = linear_sum_assignment(cost)
        except ValueError:
            wr = wc = np.zeros((0,), np.int64)
            n_empty += 1
        assert_array_equal(r, wr, err_msg=f"case {i} {mat.shape}")
        assert_array_equal(c, wc, err_msg=f"case {i} {mat.shape}")
        assert_array_equal(s, mat[wr, wc], err_msg=f"case {i} {mat.shape}")
    assert 0 < n_empty < len(mats) // 4


# ---------------------------------------------------------------------------------------------------------------------
# the fused bottom-up chain at capacity
NODES = ["a", "b", "c"]
EDGES = [("a", "b"), ("b", "c")]


def _crowded_maps(seed=0):
    """Node a: 120 peaks on a jittered grid; b: 60 of them shifted right, c: 40 of those shifted down; PAFs point
    along the edges, with noise so that some line scores fall below 0.25 or 0.5."""
    rng = np.random.default_rng(seed)
    H = W = 160                                              # confidence maps at stride 4
    gy, gx = np.divmod(np.arange(120), 12)
    a = np.stack([6 + 12.5 * gx, 5 + 15 * gy], 1) + rng.uniform(-0.4, 0.4, size=(120, 2))
    b = a[rng.permutation(120)[:60]] + [4.0, 0.5] + rng.uniform(-0.4, 0.4, size=(60, 2))
    c = b[rng.permutation(60)[:40]] + [0.3, 5.0] + rng.uniform(-0.4, 0.4, size=(40, 2))
    cms = np.stack([_blobs(H, W, p, rng.uniform(0.4, 1.0, len(p)), 1.0) for p in (a, b, c)], -1)[None]
    Hp = Wp = 80                                             # PAFs at stride 8
    pafs = rng.normal(0, 0.45, size=(1, Hp, Wp, 4)).astype(np.float32)
    pafs[..., 0] += 1.0                                      # edge a -> b points along +x
    pafs[..., 3] += 1.0                                      # edge b -> c along +y
    return cms.astype(np.float32), pafs.astype(np.float32)


def _oracle_bottomup(cms, pafs, scorer_kw, keep_node_peaks=None):
    p, v, si, ci = opf.find_local_peaks(cms, 0.2, "integral", 5)
    p = (p * np.float32(4)).astype(np.float32)
    if keep_node_peaks is not None:                          # the first K peaks of every node, in tf.where order
        rank = np.array([int((ci[:i] == ci[i]).sum()) for i in range(len(ci))])
        sel = rank < keep_node_peaks
        p, v, ci = p[sel], v[sel], ci[sel]
    return opg.PAFScorer(NODES, EDGES, 8, **scorer_kw).predict(pafs, [p], [v], [ci]), (p, v, ci)


def _device_bottomup(cms, pafs, scorer_kw, **kw):
    from sleap_b200.nn import paf_grouping as pg
    from sleap_b200.nn.inference import bottomup_from_maps
    return bottomup_from_maps(cms, pafs, pg.PAFScorer(NODES, EDGES, 8, **scorer_kw), 4, 0.2, "integral", 5, **kw)


def _assert_instances(got, winst, wps, wisc, n=None):
    n = len(winst) if n is None else n
    assert int(got["n_valid"][0]) == n
    gi = got["instance_peaks"][0]
    assert_array_equal(np.isnan(gi), np.isnan(winst[:n]))
    assert_allclose(gi, winst[:n], atol=4 * TOL, rtol=0, equal_nan=True)
    assert_array_equal(np.nan_to_num(got["instance_peak_vals"][0], nan=-1), np.nan_to_num(wps[:n], nan=-1))
    assert_allclose(got["instance_scores"][0], wisc[:n], atol=TOL, rtol=0)


def test_bottomup_crowded_node_at_capacity():
    """120 peaks of one node at max_node_peaks 128: k_score_match with more than 48 KB of shared memory, k_group over
    128-peak node lists."""
    cms, pafs = _crowded_maps()
    (winst, wps, wisc, wei, wepi, wls), (p, v, ci) = _oracle_bottomup(cms, pafs, {})
    assert np.bincount(ci).tolist() == [120, 60, 40]
    got = _device_bottomup(cms, pafs, {}, max_peaks_per_sample=512, max_node_peaks=128, max_instances=256)
    assert int(got["flags"][0]) == 0
    assert_array_equal(got["peak_channel_inds"][0], ci)
    assert_array_equal(got["peak_vals"][0], v)
    assert_array_equal(got["edge_inds"][0], wei[0])
    assert_array_equal(got["edge_peak_inds"][0], wepi[0])
    assert_allclose(got["line_scores"][0], wls[0], atol=TOL, rtol=0, equal_nan=True)
    assert 40 <= len(winst[0]) <= 140
    _assert_instances(got, winst[0], wps[0], wisc[0])


def test_bottomup_node_peak_truncation():
    """max_node_peaks 32: the flag is set and only the first 32 peaks of each node, in tf.where order, are grouped."""
    cms, pafs = _crowded_maps()
    (winst, wps, wisc, *_), _ = _oracle_bottomup(cms, pafs, {}, keep_node_peaks=32)
    got = _device_bottomup(cms, pafs, {}, max_peaks_per_sample=512, max_node_peaks=32, max_instances=256)
    assert int(got["flags"][0]) & FLAG_NODE_PEAKS_TRUNCATED
    assert not int(got["flags"][0]) & FLAG_INSTANCES_TRUNCATED
    _assert_instances(got, winst[0], wps[0], wisc[0])


@pytest.mark.parametrize("max_instances", [1, 7])
def test_bottomup_instance_truncation(max_instances):
    """max_instances below the instance count: the flag is set and the first max_instances instances are returned."""
    cms, pafs = _crowded_maps()
    (winst, wps, wisc, *_), _ = _oracle_bottomup(cms, pafs, {})
    got = _device_bottomup(cms, pafs, {}, max_peaks_per_sample=512, max_node_peaks=128, max_instances=max_instances)
    assert int(got["flags"][0]) == FLAG_INSTANCES_TRUNCATED
    _assert_instances(got, winst[0], wps[0], wisc[0], n=max_instances)


@pytest.mark.parametrize("kw", [dict(min_instance_peaks=3, min_line_scores=0.5), dict(min_instance_peaks=1.0),
                                dict(min_line_scores=0.8)])
def test_bottomup_instance_filters(kw):
    """min_instance_peaks (an int, or a float share of the nodes) and a min_line_scores that drops some matches."""
    cms, pafs = _crowded_maps(1)
    (winst, wps, wisc, *_), _ = _oracle_bottomup(cms, pafs, kw)
    (winst0, _, wisc0, *_), _ = _oracle_bottomup(cms, pafs, {})
    assert len(winst[0]) > 0 and wisc[0].sum() < wisc0[0].sum()      # the filters remove something, not everything
    got = _device_bottomup(cms, pafs, kw, max_peaks_per_sample=512, max_node_peaks=128, max_instances=256)
    assert int(got["flags"][0]) == 0
    _assert_instances(got, winst[0], wps[0], wisc[0])


# ---------------------------------------------------------------------------------------------------------------------
# the fused top-down pipeline
def _mk(spec, seed, input_scale=1.0):
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    cm = A.compile_model(spec, 1, input_scale)
    w = A.make_synthetic_weights(cm, seed)
    rng = np.random.default_rng(seed + 1)
    for L in cm.layers:
        if L["kind"] in ("conv", "tconv"):
            w[L["name"]]["bias"] = rng.normal(0, 0.1, size=L["cout"]).astype(np.float32)
    return DeviceModel(spec, w, input_channels=1, input_scale=input_scale, precision=1), w


@pytest.mark.parametrize("dtype", ["uint8", "float32"])
def test_topdown_chunks_and_empty_frame(dtype):
    """More crops than max_crops_per_call (the instance network runs over several chunks), a frame without centroids
    between two populated ones, uint8 and float frames: fused == stage by stage, and both match the oracle chain on the
    device's centroid maps."""
    from sleap_b200.nn.inference import TopDownPredictor
    ccfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=2, middle_block=True, up_interpolate=True)
    cspec = dict(backbone="unet", backbone_cfg=ccfg, head_type="centroid", part_names=None, edges=None,
                 heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
    icfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=4, middle_block=True, up_interpolate=False)
    ispec = dict(backbone="unet", backbone_cfg=icfg, head_type="centered_instance", part_names=list("abcd"), edges=None,
                 heads=[dict(name="CenteredInstanceConfmapsHead", channels=4, output_stride=4)])
    cmodel, _ = _mk(cspec, 51)
    imodel, iw = _mk(ispec, 53)
    rng = np.random.default_rng(8)
    imgs = rng.integers(0, 256, size=(3, 192, 224, 1), dtype=np.uint8)
    imgs[1] = 0                                              # flat frame: its centroid map has no peak above the others'
    if dtype == "float32":
        imgs = (imgs.astype(np.float32) / np.float32(255.0)).astype(np.float32)
    ccms = cmodel.forward(imgs)[0]
    thr = float(max(ccms[1].max(), np.sort(ccms[[0, 2]].reshape(-1))[-60]))
    max_inst = 6
    pred = TopDownPredictor(cmodel, imodel, crop_size=64, peak_threshold=thr, integral_refinement=True, batch_size=3,
                            max_instances=max_inst)
    im = pred.inference_model
    im.instance_peaks.peak_threshold = -1e9
    im.instance_peaks.max_crops_per_call = 4
    # oracle chain on the device's centroid maps
    cp, cv, csi, _ = opf.find_local_peaks(ccms, thr, "integral", 5)
    cp = (cp * np.float32(2)).astype(np.float32)
    keep = []
    for s in range(3):
        idx = np.nonzero(csi == s)[0]
        if len(idx) > max_inst:
            idx = idx[np.argsort(-cv[idx], kind="stable")[:max_inst]]
        keep.append(idx)
    keep = np.concatenate(keep)
    cp, cv, csi = cp[keep], cv[keep], csi[keep]
    counts = [int((csi == s).sum()) for s in range(3)]
    assert counts[1] == 0 and counts[0] > 0 and counts[2] > 0 and sum(counts) > 4, counts
    bb = tf_ops.make_centered_bboxes(cp, 64, 64)
    crops = tf_ops.crop_bboxes(imgs, bb, csi)
    icms = convnet.model_forward(opre.preprocess(crops, True, 1.0, 16), ispec, iw)[0]
    dcms = imodel.forward(crops)[0]
    assert_allclose(dcms, icms, atol=1e-4 * max(1, np.abs(icms).max()), rtol=1e-4)
    wp, _ = opf.find_global_peaks(dcms, -1e9, "integral", 5)
    wp = wp * np.float32(4) + (cp - np.float32(32))[:, None, :]
    assert im._can_fuse()
    outs = []
    for fused in (True, False):
        im.fused = fused
        outs.append(im.predict_on_batch(imgs))
    a, b = outs
    assert_array_equal(a["n_valid"], b["n_valid"])
    for k in ("centroids", "centroid_vals", "instance_peaks", "instance_peak_vals"):
        assert_array_equal(np.nan_to_num(a[k], nan=-7.0), np.nan_to_num(b[k], nan=-7.0))
    for s in range(3):
        n = int(a["n_valid"][s])
        assert n == counts[s]
        assert_allclose(a["centroids"][s, :n], cp[csi == s], atol=TOL * 2)
        assert_allclose(a["centroid_vals"][s, :n], cv[csi == s], atol=0)
        assert_allclose(a["instance_peaks"][s, :n], wp[csi == s], atol=5e-4, equal_nan=True)


def _pass_through_centroid_model():
    """A centroid UNet whose weights make its confidence map the preprocessed frame itself: the first block and the
    stride-1 refine convs carry channel 0 through their centre taps (the refine conv takes it from either half of its
    concatenated input), every other weight and bias is zero, so the deeper levels contribute exact zeros.  With fp32
    convolutions the map is the frame to the last bit, which lets a test plant tied centroid values and place centroids
    anywhere, including at the frame edge."""
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    cfg = dict(filters=8, filters_rate=2, max_stride=4, output_stride=1, middle_block=False, up_interpolate=True)
    spec = dict(backbone="unet", backbone_cfg=cfg, head_type="centroid", part_names=None, edges=None,
                heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=1)])
    cm = A.compile_model(spec, 1)
    w = A.make_synthetic_weights(cm, 0)
    for L in cm.layers:
        w[L["name"]]["kernel"][...] = 0
        w[L["name"]]["bias"][...] = 0
    w["stack0_enc0_conv0"]["kernel"][1, 1, 0, 0] = 1
    w["stack0_enc0_conv1"]["kernel"][1, 1, 0, 0] = 1
    w["stack0_dec1_s2_to_s1_refine_conv0"]["kernel"][1, 1, [0, 16], 0] = 1
    w["stack0_dec1_s2_to_s1_refine_conv1"]["kernel"][1, 1, 0, 0] = 1
    w["CentroidConfmapsHead"]["kernel"][0, 0, 0, 0] = 1
    return DeviceModel(spec, w, input_channels=1, precision=1), spec, w


def _stamp(img, x, y, c):
    """A 3 x 3 blob with centre value c (a strict maximum) and fixed, asymmetric neighbours."""
    img[y - 1:y + 2, x - 1:x + 2, 0] = np.array([[60, 90, 70], [100, c, 80], [50, 110, 40]], np.uint8)
    img[y, x, 0] = c


@pytest.mark.parametrize("dtype", ["uint8", "float32"])
def test_topdown_tied_and_edge_centroids(dtype):
    """Frame 0 has 9 centroids for max_instances 4, and the cut falls inside a run of equal values: top-k keeps the
    higher values, then the tied ones in tf.where order (lower index first).  Frame 1 has none.  Frame 2 has centroids
    within half a crop (32 px) of every edge, so the crops reach past the frame.  Frame 3 brings the crop count to 11,
    three chunks of max_crops_per_call 4.  Fused == stage by stage == the oracle chain."""
    from sleap_b200.nn.inference import TopDownPredictor
    cmodel, cspec, cw = _pass_through_centroid_model()
    icfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=4, middle_block=True, up_interpolate=False)
    ispec = dict(backbone="unet", backbone_cfg=icfg, head_type="centered_instance", part_names=list("abcd"), edges=None,
                 heads=[dict(name="CenteredInstanceConfmapsHead", channels=4, output_stride=4)])
    imodel, iw = _mk(ispec, 57)
    H, W = 160, 192
    imgs = np.zeros((4, H, W, 1), np.uint8)
    for (x, y), c in zip([(20, 20), (60, 20), (150, 25), (30, 60), (90, 60), (170, 70), (40, 110), (100, 120), (160, 130)],
                         [200, 200, 230, 200, 200, 180, 230, 200, 200]):
        _stamp(imgs[0], x, y, c)
    for (x, y), c in zip([(100, 1), (1, 40), (W - 2, H - 3), (20, H - 2)], [170, 150, 160, 140]):
        _stamp(imgs[2], x, y, c)
    for (x, y), c in zip([(50, 50), (120, 80), (80, 130)], [190, 210, 170]):
        _stamp(imgs[3], x, y, c)
    if dtype == "float32":
        imgs = (imgs.astype(np.float32) / np.float32(255.0)).astype(np.float32)
    ccms = cmodel.forward(imgs)[0]
    want_map = convnet.model_forward(opre.preprocess(imgs, True, 1.0, 4), cspec, cw)[0]
    assert_allclose(ccms, want_map, rtol=1e-6, atol=0)       # the map is the preprocessed frame
    thr = float(0.5 * ccms.max())
    max_inst = 4
    pred = TopDownPredictor(cmodel, imodel, crop_size=64, peak_threshold=thr, integral_refinement=True, batch_size=4,
                            max_instances=max_inst)
    im = pred.inference_model
    im.instance_peaks.peak_threshold = -1e9
    im.instance_peaks.max_crops_per_call = 4
    # oracle chain on the device's centroid maps
    cp, cv, csi, _ = opf.find_local_peaks(ccms, thr, "integral", 5)
    assert [int((csi == s).sum()) for s in range(4)] == [9, 0, 4, 3]
    v0 = np.sort(cv[csi == 0])[::-1]
    assert v0[0] > v0[max_inst - 1] == v0[max_inst]          # higher values first, then a tie across the cut
    keep = []
    for s in range(4):
        idx = np.nonzero(csi == s)[0]
        if len(idx) > max_inst:
            idx = idx[np.argsort(-cv[idx], kind="stable")[:max_inst]]
        keep.append(idx)
    keep = np.concatenate(keep)
    cp, cv, csi = cp[keep], cv[keep], csi[keep]
    edge = cp[csi == 2]
    assert np.all(np.minimum.reduce([edge[:, 0], edge[:, 1], W - 1 - edge[:, 0], H - 1 - edge[:, 1]]) < 32)
    bb = tf_ops.make_centered_bboxes(cp, 64, 64)
    crops = tf_ops.crop_bboxes(imgs, bb, csi)
    dcms = imodel.forward(crops)[0]
    wp, _ = opf.find_global_peaks(dcms, -1e9, "integral", 5)
    wp = wp * np.float32(4) + (cp - np.float32(32))[:, None, :]
    assert im._can_fuse()
    outs = []
    for fused in (True, False):
        im.fused = fused
        outs.append(im.predict_on_batch(imgs))
    a, b = outs
    assert_array_equal(a["n_valid"], [4, 0, 4, 3])
    assert_array_equal(a["n_valid"], b["n_valid"])
    for k in ("centroids", "centroid_vals", "instance_peaks", "instance_peak_vals"):
        assert_array_equal(np.nan_to_num(a[k], nan=-7.0), np.nan_to_num(b[k], nan=-7.0))
    for s in range(4):
        n = int(a["n_valid"][s])
        assert_allclose(a["centroids"][s, :n], cp[csi == s], atol=TOL)
        assert_array_equal(a["centroid_vals"][s, :n], cv[csi == s])
        assert_allclose(a["instance_peaks"][s, :n], wp[csi == s], atol=5e-4, equal_nan=True)
