"""The identity kernels past one pass of their 128-thread loops and at their caps: k_class_group with more than 128 and
256 (peak, class) pairs per node, 128 classes and max_node_peaks up to the largest that fits in shared memory;
k_class_vectors over 129 to 4096 tap channels, a 9,600-input Flatten, 129 to 4096 units and 128 classes; k_td_class_assign
with more crops than classes at 128 classes.  The references are the ones the step tests use: the host chain on the same
maps (bit for bit), the float64 restatement of the head (pooled features bit for bit, probabilities within 1e-6) and
identity.classify_peaks_from_vectors on the device's own probabilities (bit for bit).

Also the caps themselves: 129 classes, 4097 units and a 4097-channel global pool are refused, a Flatten of more than
4096 inputs is not, and a max_node_peaks whose grouping kernels would not fit in the device's shared memory is refused
at configure time, with nothing queued and the previous chain kept."""
import numpy as np
import pytest
from numpy.testing import assert_allclose

import layer_audit as la
from test_gpu_multiclass_step import assert_bit_equal, host_chain
from test_gpu_topdown_multiclass_step import NODES, _staged_peaks, dense_weights, head_restated, synth_crops

pytestmark = pytest.mark.gpu

F32 = np.float32
THREADS = 128                       # the CTA width of k_class_group, k_class_vectors and k_td_class_assign


# ------------------------------------------------------------------------------------------------ shared memory
# Python restatements of the kernels' dynamic shared memory (sb_post.cu); the tests below pin them to the configure check
# by running the largest K that fits and refusing the next one.
def _lsap_bytes(L):
    return L * (3 * 8 + 4 * 4 + 2) + 16


def _ceil16(x):
    return (x + 15) & ~15


def class_group_smem(K, NC):
    L, M = max(K, NC), min(K, NC)
    return _ceil16(_lsap_bytes(L)) + (K * NC + 2 * K) * 4 + (K + 2 * M) * 4


def score_match_smem(K):
    return _ceil16(4 * K * K) + _lsap_bytes(K)


def smem_optin():
    import torch
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def largest_k(smem):
    K, limit = 1, smem_optin()
    while smem(K + 1) <= limit:
        K += 1
    return K


def _launches():
    from sleap_b200 import _lib
    return _lib.default_handle().gpu_launches()


# ------------------------------------------------------------------------------------------------ bottom-up: k_class_group
def crowd_maps(seed, n_animals, n_classes, B=2, n_nodes=2, cm_stride=2, cs=2, tie=None, spacing=10):
    """Confidence maps (B,H,W,n_nodes) with n_animals animals on a jittered grid (every node a distinct peak) and class-map
    logits (B,Hc,Wc,n_classes): noise around -3, and animal a's class rising around each of its nodes; the animals take
    the classes in a random order.  tie: "all" gives every class the same logits, "pairs" classes 2i and 2i+1."""
    from oracle import synth
    rng = np.random.default_rng(seed)
    cols = int(np.ceil(np.sqrt(n_animals * 1.3)))
    rows = -(-n_animals // cols)
    H, W = rows * spacing + 8, cols * spacing + 8
    Himg, Wimg = H * cm_stride, W * cm_stride
    Hc, Wc = Himg // cs, Wimg // cs
    xv, yv = synth.make_grid_vectors(Himg, Wimg, cm_stride)
    xc, yc = synth.make_grid_vectors(Himg, Wimg, cs)
    cms = np.zeros((B, H, W, n_nodes), F32)
    logits = rng.normal(-3.0, 0.5, (B, Hc, Wc, n_classes)).astype(F32)
    for b in range(B):
        gy, gx = np.divmod(rng.permutation(rows * cols)[:n_animals], cols)
        centre = np.stack([4 + (gx + 0.5) * spacing, 4 + (gy + 0.5) * spacing], -1) * cm_stride
        inst = (centre[:, None, :] + rng.uniform(-2, 2, (n_animals, n_nodes, 2)) * cm_stride).astype(F32)
        cms[b] = synth.make_multi_confmaps(inst, xv, yv, sigma=1.5 * cm_stride)
        cls = rng.permutation(n_animals) % n_classes
        for a in range(n_animals):
            for p in inst[a]:
                g = np.exp(-((xc[None] - p[0]) ** 2 + (yc[:, None] - p[1]) ** 2) / F32(2 * (1.5 * cs) ** 2))
                logits[b, :, :, cls[a]] += F32(7.0) * g.astype(F32)
    if tie == "all":
        logits[...] = logits[..., :1]
    elif tie == "pairs":
        logits[..., 1::2] = logits[..., 0:n_classes - n_classes % 2:2]
    return cms, logits


def _max_node_peaks(cms, thr=0.2):
    from sleap_b200.nn import peak_finding
    _, _, si, ci = peak_finding.find_local_peaks(cms, threshold=thr, refinement="integral", integral_patch_size=5)
    return int(np.bincount(np.asarray(si) * cms.shape[3] + np.asarray(ci)).max())


BU_CASES = {                        # reach: n * NC above it on some (frame, node)
    "animals12_classes20": dict(n_animals=12, n_classes=20, reach=THREADS),
    "animals30_classes64": dict(n_animals=30, n_classes=64, reach=2 * THREADS),
    "animals10_classes128": dict(n_animals=10, n_classes=128, reach=2 * THREADS),
    "more_peaks_than_classes": dict(n_animals=40, n_classes=16, reach=2 * THREADS),
    "more_peaks_than_threads": dict(n_animals=150, n_classes=8, mnp=160, reach=2 * THREADS),
    "k128_classes128": dict(n_animals=40, n_classes=128, mnp=128, reach=2 * THREADS),
    "kmax_classes128": dict(n_animals=40, n_classes=128, mnp="max", reach=2 * THREADS),
    "all_classes_tied_128": dict(n_animals=20, n_classes=128, tie="all", reach=2 * THREADS),
    "class_pairs_tied_128": dict(n_animals=20, n_classes=128, tie="pairs", reach=2 * THREADS),
}


@pytest.mark.parametrize("case", list(BU_CASES))
def test_class_group_matches_host_chain(case):
    from sleap_b200.nn.inference import bottomup_multiclass_from_maps
    cfg = BU_CASES[case]
    NC = cfg["n_classes"]
    mnp = cfg.get("mnp", 64)
    if mnp == "max":
        mnp = largest_k(lambda K: class_group_smem(K, NC))
        assert 128 < mnp < 512, mnp
    cms, logits = crowd_maps(sum(map(ord, case)), cfg["n_animals"], NC, tie=cfg.get("tie"))
    n = _max_node_peaks(cms)
    assert n == cfg["n_animals"] and n * NC > cfg["reach"], (n, NC)
    out = bottomup_multiclass_from_maps(cms, logits, 2, 2, 0.2, "integral", 5, max_node_peaks=mnp)
    want = host_chain(cms, logits, 2, 2, 0.2, "integral", 5, max_node_peaks=mnp)
    assert_bit_equal(out["instance_peaks"], want[0], f"{case}: points")
    assert_bit_equal(out["instance_peak_vals"], want[1], f"{case}: point values")
    assert_bit_equal(out["instance_scores"], want[2], f"{case}: class probabilities")
    assert not out["flags"].any(), out["flags"]
    assigned = np.isfinite(out["instance_scores"]).sum(1)            # (B, n_nodes): classes holding a peak
    assert (assigned <= min(n, NC)).all() and assigned.min() > 0, assigned
    if cfg.get("tie") == "all":                                       # every peak's probabilities tie: every match is kept
        assert (assigned == min(n, NC)).all(), assigned


# ------------------------------------------------------------------------------------------------ top-down: k_class_vectors, k_td_class_assign
TD_CASES = {
    "pool_c129": dict(counts=[3, 2], Cf=129, units=16, n_classes=5),
    "pool_c384_units256_classes20": dict(counts=[4, 3, 5], Cf=384, units=256, n_classes=20),
    "pool_c4096": dict(counts=[2, 3], Hf=2, Wf=2, Cf=4096, units=64, n_classes=6),
    "flatten_5x5x384": dict(counts=[3, 2], global_pool=False, Hf=5, Wf=5, Cf=384, units=129, n_classes=7),
    "units129_two_fc": dict(counts=[3, 4], Cf=64, units=129, n_fc=2, n_classes=9),
    "units1000": dict(counts=[3, 4], Cf=200, units=1000, n_classes=10),
    "units4096": dict(counts=[2, 2], Cf=130, units=4096, n_classes=12),
    "no_fc_c384": dict(counts=[3, 3], Cf=384, n_fc=0, n_classes=30),
    "one_fc_c384_units300": dict(counts=[3, 3], Cf=384, n_fc=1, units=300, n_classes=30),
    "three_fc_units300": dict(counts=[3, 3], Cf=384, n_fc=3, units=300, n_classes=30),
    "crops150_classes128": dict(counts=[150, 7], Cf=256, units=256, n_classes=128),
    "crops3_classes128": dict(counts=[3], Cf=160, units=200, n_classes=128),
    "empty_frame_between_full_ones": dict(counts=[40, 0, 40], Cf=160, units=160, n_classes=30),
    "nan_in_one_channel": dict(counts=[3, 2], Cf=200, units=150, n_classes=8),
    "negative_preactivations": dict(counts=[4, 3], Cf=300, units=200, n_fc=2, n_classes=8),
}


def _td_case(name):
    cfg = {k: v for k, v in TD_CASES[name].items()}
    case = synth_crops(sum(map(ord, name)), **cfg)
    if name == "nan_in_one_channel":            # crop 1: NaN past the first pixel; crop 3: NaN at the first pixel
        case["feats"][1, 2, 3, 17] = np.nan
        case["feats"][3, 0, 0, 150] = np.nan
    if name == "negative_preactivations":       # bias each first-layer unit to its median pre-activation over the crops
        p = case["weights"]["pre_classification0_fc"]
        z = case["feats"].max(axis=(1, 2)).astype(np.float64) @ p["kernel"].astype(np.float64)
        p["bias"] = (-np.median(z, axis=0) + np.random.default_rng(3).normal(0, 0.05, z.shape[1])).astype(F32)
    return case


def _td_run(case, thr=0.3):
    from sleap_b200.nn.inference import topdown_multiclass_from_features
    return topdown_multiclass_from_features(case["cms"], case["feats"], case["sinds"], case["B"], case["head"], case["weights"],
                                            case["stride"], peak_threshold=thr, refinement="local", offsets=case["offsets"],
                                            crop_offsets=case["crop_offsets"])


@pytest.mark.parametrize("name", list(TD_CASES))
def test_class_vectors_and_assignment(name):
    from sleap_b200.nn import identity
    case = _td_case(name)
    head = case["head"]
    out = _td_run(case)
    pooled, probs = head_restated(case["feats"], head, case["weights"])
    assert_bit_equal(out["features"], pooled, f"{name}: pooled features")
    got = out["class_vectors"]
    assert np.array_equal(np.isnan(got), np.isnan(probs)), f"{name}: NaN pattern of the probabilities"
    assert_allclose(got, probs, rtol=1e-6, atol=0)
    fin = np.isfinite(probs)
    exact = float(np.mean(got[fin].view(np.uint32) == probs[fin].view(np.uint32)))
    print(f"{name}: {exact:.4f} of the probabilities bit-equal to the restatement")
    if name == "nan_in_one_channel":            # np.max propagates the NaN into the crop's channel, and on into its head
        assert np.isnan(out["features"][1, 17]) and np.isnan(out["features"][3, 150])
        assert np.isnan(out["features"]).sum() == 2
        assert np.isnan(got[[1, 3]]).all() and np.isfinite(np.delete(got, [1, 3], 0)).all()
        return                                  # SciPy refuses NaN costs: no host assignment to compare with
    if name == "negative_preactivations":
        x = pooled
        p = case["weights"]["pre_classification0_fc"]
        z = (x.astype(np.float64) @ p["kernel"].astype(np.float64) + p["bias"]).astype(F32)
        assert 0.2 < float(np.mean(z < 0)) < 0.8
    pts, pv = _staged_peaks(case, "local", 0.3)
    want = identity.classify_peaks_from_vectors(pts, pv, got, case["sinds"], case["B"])
    assert_bit_equal(out["instance_peaks"], want[0], f"{name}: points")
    assert_bit_equal(out["instance_peak_vals"], want[1], f"{name}: point values")
    assert_bit_equal(out["instance_scores"], want[2], f"{name}: class probabilities")
    counts = np.bincount(case["sinds"], minlength=case["B"])
    assigned = np.isfinite(out["instance_scores"]).sum(1)
    assert np.all(assigned <= np.minimum(counts, head["channels"])) and np.all((assigned > 0) == (counts > 0)), assigned
    if name == "empty_frame_between_full_ones":
        assert np.isnan(out["instance_scores"][1]).all() and np.isnan(out["instance_peaks"][1]).all()


# ------------------------------------------------------------------------------------------------ the fused step at a wide head
def _wide_models(precision, filters=16, n_fc=1, units=256, n_classes=20):
    """The top-down multi-class test's centroid model and a centered-instance UNet of `filters` filters whose
    ClassVectorsHead taps stride 16 (16 filters: 256 channels)."""
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    ccfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=2, middle_block=True, up_interpolate=True)
    cspec = dict(backbone="unet", backbone_cfg=ccfg, head_type="centroid", part_names=None, edges=None,
                 heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
    icfg = dict(filters=filters, filters_rate=2, max_stride=16, output_stride=4, middle_block=True, up_interpolate=False)
    ispec = dict(backbone="unet", backbone_cfg=icfg, head_type="multi_class_topdown", part_names=NODES, edges=None,
                 classes=[f"c{i}" for i in range(n_classes)],
                 heads=[dict(name="CenteredInstanceConfmapsHead", channels=len(NODES), output_stride=4),
                        dict(name="ClassVectorsHead", channels=n_classes, output_stride=16, vector=True, num_fc_layers=n_fc,
                             num_fc_units=units, global_pool=True)])
    cw = A.make_synthetic_weights(A.compile_model(cspec, 1), 61)
    icm = A.compile_model(ispec, 1)
    iw = la.synthetic_weights(icm, 63)
    iw.update(dense_weights(icm.vector_taps["ClassVectorsHead"]["C"], n_fc, units, n_classes, 65, logit_scale=8.0))
    return DeviceModel(cspec, cw, input_channels=1, precision=precision), DeviceModel(ispec, iw, input_channels=1, precision=precision)


@pytest.fixture(scope="module")
def frames():
    imgs = np.random.default_rng(9).integers(0, 256, size=(4, 192, 224, 1), dtype=np.uint8)
    imgs[1] = 0                                      # no centroid in this frame
    return imgs


def _wide_predictor(precision, frames):
    from sleap_b200.nn.inference import TopDownMultiClassPredictor
    cmodel, imodel = _wide_models(precision)
    thr = max(float(np.quantile(cmodel.forward(frames)[0], 0.99)), 1e-3)
    pred = TopDownMultiClassPredictor(cmodel, imodel, crop_size=64, peak_threshold=thr, integral_refinement=True,
                                      batch_size=len(frames))
    pred.inference_model.instance_peaks.peak_threshold = 0.0
    pred.inference_model.instance_peaks.return_class_vectors = True
    return pred


@pytest.mark.parametrize("precision", [0, 1, 2])
def test_fused_step_wide_head(precision, frames):
    im = _wide_predictor(precision, frames).inference_model
    fp = im.instance_peaks
    mi = fp.keras_model
    tap = mi.cm.vector_taps["ClassVectorsHead"]
    assert tap["C"] >= 256 and fp.class_head["num_fc_units"] == 256 and fp.class_head["channels"] == 20
    if precision == 2:                               # the [lo | hi | hi] planes: channel pitch 3C
        assert tap["planes"] == 3 and tap["buf_C"] == 3 * tap["C"], tap
    assert im._can_fuse()
    fused = im.predict_on_batch(frames)
    taps, host_head = [], mi._class_vectors          # the staged path's tap features, as the device computed them
    mi._class_vectors = lambda buf, name: (taps.append(buf.copy()), host_head(buf, name))[1]
    try:
        im.fused = False
        staged = im.predict_on_batch(frames)
    finally:
        im.fused = True
        del mi._class_vectors
    for k in ("centroids", "centroid_vals", "instance_peaks", "instance_peak_vals"):
        assert_bit_equal(fused[k], staged[k], f"precision {precision}: {k}")
    assert np.array_equal(np.isnan(fused["instance_scores"]), np.isnan(staged["instance_scores"])), "class assignments differ"
    assert_allclose(fused["instance_scores"], staged["instance_scores"], atol=1e-5, rtol=0)
    n_crops = int(np.isfinite(fused["centroid_vals"]).sum())
    assert n_crops > len(frames) and np.isfinite(fused["instance_scores"]).any(), n_crops
    buf = np.concatenate(taps)
    c0, C = tap["coff"], tap["C"]
    feat = buf[..., c0:c0 + C] + buf[..., c0 + C:c0 + 2 * C] if tap["planes"] == 3 else buf[..., c0:c0 + C]
    assert len(feat) == n_crops == len(fused["class_vectors"])
    _, probs = head_restated(feat, fp.class_head, mi.dense_weights)
    got = fused["class_vectors"]
    assert_allclose(got, probs, rtol=1e-6, atol=0)
    exact = float(np.mean(got.view(np.uint32) == probs.view(np.uint32)))
    print(f"precision {precision}: {n_crops} crops, {exact:.4f} of the probabilities bit-equal to the restatement")


# ------------------------------------------------------------------------------------------------ refusals at the caps
def test_head_caps_refused_keep_the_pipeline(frames):
    from ctypes import byref
    from sleap_b200._lib import MAX_CLASSES, MAX_DENSE_WIDTH, SleapB200Error
    from sleap_b200.nn.inference import _topdown_params, topdown_multiclass_params
    from sleap_b200.nn.model import pack_dense_weights
    pred = _wide_predictor(0, frames)
    im = pred.inference_model
    cc, fp = im.centroid_crop, im.instance_peaks
    mc, mi = cc.keras_model, fp.keras_model
    first = im.predict_on_batch(frames)
    td, _ = _topdown_params(cc, fp)
    tap = mi.cm.vector_taps["ClassVectorsHead"]
    for what, head, msg in (("129 classes", dict(fp.class_head, channels=MAX_CLASSES + 1), "129 classes"),
                            ("4097 units", dict(fp.class_head, num_fc_units=MAX_DENSE_WIDTH + 1), "dense width above 4096")):
        dense = pack_dense_weights(head, dense_weights(tap["C"], head["num_fc_layers"], head["num_fc_units"], head["channels"], 5))
        p = topdown_multiclass_params(td, tap, head, dense)
        n0 = _launches()
        with pytest.raises(SleapB200Error, match=msg):
            mc.handle.call("sb_topdown_multiclass_configure", byref(p), *frames.shape)
        assert _launches() == n0, f"{what}: the refused configure queued work"
        again = im.predict_on_batch(frames)
        for k in first:
            assert first[k].tobytes() == again[k].tobytes(), (what, k)


def test_global_pool_cap_refused_flatten_uncapped():
    from sleap_b200._lib import MAX_DENSE_WIDTH, SleapB200Error
    case = synth_crops(17, [2, 1], Hf=1, Wf=1, Cf=MAX_DENSE_WIDTH + 1, n_classes=3)
    n0 = _launches()
    with pytest.raises(SleapB200Error, match="dense width above 4096"):
        _td_run(case)
    assert _launches() == n0
    # the same 4097 inputs through a Flatten: read from global memory, no cap
    case = synth_crops(17, [2, 1], global_pool=False, Hf=1, Wf=1, Cf=MAX_DENSE_WIDTH + 1, n_classes=3)
    out = _td_run(case)
    pooled, probs = head_restated(case["feats"], case["head"], case["weights"])
    assert_bit_equal(out["features"], pooled, "flatten of 4097 inputs")
    assert_allclose(out["class_vectors"], probs, rtol=1e-6, atol=0)


# ------------------------------------------------------------------------------------------------ shared-memory capacity
def _chains(frames_shape=(2, 64, 96, 1)):
    from test_gpu_chain import Chains
    return Chains(np.random.default_rng(5).integers(0, 256, size=frames_shape, dtype=np.uint8))


def _same(got, want, what):
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and g.tobytes() == w.tobytes(), f"{what}: output {i} differs"


def test_paf_chain_node_peaks_capacity():
    """The PAF chain: the largest max_node_peaks whose k_score_match fits runs and matches the oracle on 120-peak nodes;
    the next one and 512 are refused at configure, by sb_bottomup_configure and sb_bottomup_from_maps alike, with nothing
    queued and the previous chain kept."""
    from sleap_b200._lib import SleapB200Error
    from test_gpu_post_edges import _assert_instances, _crowded_maps, _device_bottomup, _oracle_bottomup
    kmax = largest_k(score_match_smem)
    assert 128 < kmax < 256, kmax
    cms, pafs = _crowded_maps()
    (winst, wps, wisc, *_), (_, _, ci) = _oracle_bottomup(cms, pafs, {})
    assert np.bincount(ci).max() == 120
    got = _device_bottomup(cms, pafs, {}, max_peaks_per_sample=512, max_node_peaks=kmax, max_instances=256)
    assert int(got["flags"][0]) == 0
    _assert_instances(got, winst[0], wps[0], wisc[0])
    for K in (kmax + 1, 512):
        n0 = _launches()
        with pytest.raises(SleapB200Error, match=rf"failed \(-3\): max_node_peaks {K}: .*shared memory"):
            _device_bottomup(cms, pafs, {}, max_peaks_per_sample=512, max_node_peaks=K, max_instances=256)
        assert _launches() == n0, K
    c = _chains()
    c.paf.max_node_peaks = kmax
    c.configure("paf")
    want = c.run("paf")
    n0 = c.m.handle.gpu_launches()
    for K in (kmax + 1, 512):
        c.paf.max_node_peaks = K
        with pytest.raises(SleapB200Error, match=r"failed \(-3\).*shared memory"):
            c.configure("paf")
    assert c.m.handle.gpu_launches() == n0
    _same(c.run("paf"), want, "PAF chain after refused capacities")


def test_class_chain_node_peaks_capacity():
    """The multi-class chain: with 128 classes the largest max_node_peaks whose k_class_group fits runs (the
    kmax_classes128 case above) and the next one and 512 are refused by sb_multiclass_from_maps; on a configured
    2-class model the same rule holds at its own largest K, and a refusal keeps the chain."""
    from sleap_b200._lib import SleapB200Error
    from sleap_b200.nn.inference import bottomup_multiclass_from_maps
    kmax = largest_k(lambda K: class_group_smem(K, 128))
    cms, logits = crowd_maps(1, 4, 128)
    for K in (kmax + 1, 512):
        n0 = _launches()
        with pytest.raises(SleapB200Error, match=rf"failed \(-3\): max_node_peaks {K} with 128 classes: .*shared memory"):
            bottomup_multiclass_from_maps(cms, logits, 2, 2, 0.2, "integral", 5, max_node_peaks=K)
        assert _launches() == n0, K
    c = _chains()
    k2 = largest_k(lambda K: class_group_smem(K, 2))
    assert k2 > 1024, k2
    c.cls.max_node_peaks = k2
    c.configure("class")
    want = c.run("class")
    n0 = c.m.handle.gpu_launches()
    c.cls.max_node_peaks = k2 + 1
    with pytest.raises(SleapB200Error, match=r"failed \(-3\).*shared memory"):
        c.configure("class")
    assert c.m.handle.gpu_launches() == n0
    _same(c.run("class"), want, "2-class chain after a refused capacity")
