"""One post-processing chain per device model: every configure call drops the previous chain (with its tracker), calls
for another chain than the model's are refused before any launch, a refused configure keeps the previous chain, and the
fused top-down pipeline runs only while both its models still have the chains it was configured with."""
import itertools
from ctypes import byref, c_int32

import numpy as np
import pytest

import layer_audit as la

pytestmark = pytest.mark.gpu

B, H, W = 2, 64, 96
NODES, EDGES = ["a", "b", "c"], [("a", "b"), ("b", "c")]
CHAINS = ("paf", "class", "global", "centroid")


@pytest.fixture(scope="module", autouse=True)
def pinned_input_stage():
    """Models configured apart take the same input stage (a timed choice), so that their heads are the same bits."""
    with pytest.MonkeyPatch.context() as mp:
        mp.setenv("SB_FORCE_CONV01", "0")
        mp.setenv("SB_FORCE_FIRST_VIEW", "0")
        yield


def _model(seed=3):
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    cfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=2, middle_block=True, up_interpolate=True)
    spec = dict(backbone="unet", backbone_cfg=cfg, head_type="multi_instance", part_names=NODES, edges=EDGES,
                heads=[dict(name="MultiInstanceConfmapsHead", channels=3, output_stride=2),
                       dict(name="PartAffinityFieldsHead", channels=4, output_stride=2),
                       dict(name="ClassMapsHead", channels=2, output_stride=2)])
    m = DeviceModel(spec, A.make_synthetic_weights(A.compile_model(spec, 1), seed), input_channels=1, precision=0)
    return m.configure(B, H, W, 1)


class Chains:
    """The four per-model chains on one synthetic model, configured and run through the C-ABI."""

    def __init__(self, frames):
        from sleap_b200.nn import paf_grouping as pg
        from sleap_b200.nn.inference import class_params, paf_params
        self.m = _model()
        self.frames = np.ascontiguousarray(frames)
        cms = self.m.forward(self.frames)[0]
        self.thr = float(np.quantile(cms, 0.9))
        heads = self.m.cm.head_buffers
        cb = heads["MultiInstanceConfmapsHead"]
        self.paf, self.keep = paf_params(pg.PAFScorer(NODES, EDGES, 2), (cb, heads["PartAffinityFieldsHead"], -1), 2, 2, self.thr,
                                         "integral", 5, 1.0, 256, 16, 8)
        self.cls = class_params((cb, heads["ClassMapsHead"], -1), 2, 2, self.thr, "integral", 5, 3, 2, 1.0, 256, 16)
        from sleap_b200._lib import CentroidParams, GlobalParams
        self.glb = GlobalParams(cb, -1, 2, self.thr, 1, 5, 1.0)
        self.cen = CentroidParams(cb, -1, 2, self.thr, 1, 5, 1.0, 64)

    def call(self, name, *args):
        self.m.handle.call(name, self.m.model_id, *args)

    def configure(self, chain):
        fn, p = {"paf": ("sb_bottomup_configure", self.paf), "class": ("sb_multiclass_configure", self.cls),
                 "global": ("sb_global_configure", self.glb), "centroid": ("sb_centroid_configure", self.cen)}[chain]
        self.call(fn, byref(p))

    def run(self, chain):
        from sleap_b200._lib import ptr
        f = self.frames
        if chain == "paf":
            I, N = self.paf.max_instances, len(NODES)
            out = [np.zeros((B, I, N, 2), np.float32), np.zeros((B, I, N), np.float32), np.zeros((B, I), np.float32),
                   np.zeros(B, np.int32), np.zeros(B, np.int32)]
            self.call("sb_infer_bottomup", ptr(f), B, *map(ptr, out))
        elif chain == "class":
            out = [np.zeros((B, 2, 3, 2), np.float32), np.zeros((B, 2, 3), np.float32), np.zeros((B, 2, 3), np.float32),
                   np.zeros(B, np.int32)]
            self.call("sb_infer_multiclass", ptr(f), 1, B, *map(ptr, out))
        elif chain == "global":
            out = [np.zeros((B, 3, 2), np.float32), np.zeros((B, 3), np.float32)]
            self.call("sb_infer_global", ptr(f), 1, B, None, *map(ptr, out))
        else:
            cap = B * self.cen.max_peaks_per_sample
            out = [np.zeros((cap, 2), np.float32), np.zeros(cap, np.float32), np.zeros(cap, np.int32)]
            n, fl = c_int32(0), np.zeros(B, np.int32)
            self.call("sb_infer_centroids", ptr(f), 1, B, *map(ptr, out), byref(n), ptr(fl))
            out = [a[:n.value] for a in out] + [fl]
        return out


def _assert_same(got, want, what):
    for i, (g, w) in enumerate(zip(got, want)):
        assert g.shape == w.shape and g.tobytes() == w.tobytes(), f"{what}: output {i} differs"


@pytest.fixture(scope="module")
def frames():
    return np.random.default_rng(5).integers(0, 256, size=(B, H, W, 1), dtype=np.uint8)


@pytest.fixture(scope="module")
def fresh(frames):
    """Each chain's results on a model that never ran another chain."""
    out = {}
    for chain in CHAINS:
        c = Chains(frames)
        c.configure(chain)
        out[chain] = c.run(chain)
    return out


def test_one_chain_at_a_time(frames, fresh):
    from sleap_b200._lib import SleapB200Error
    c = Chains(frames)
    for first, second in itertools.permutations(CHAINS, 2):
        c.configure(first)
        _assert_same(c.run(first), fresh[first], f"{first}")
        c.configure(second)
        with pytest.raises(SleapB200Error, match="not configured"):
            c.run(first)
        _assert_same(c.run(second), fresh[second], f"{second} after {first}")


def test_refused_configure_keeps_the_chain(frames, fresh):
    from sleap_b200._lib import SleapB200Error
    c = Chains(frames)
    c.configure("paf")
    c.paf.n_nodes += 1                                   # the confidence-map head has 3 channels
    with pytest.raises(SleapB200Error):
        c.configure("paf")
    c.paf.n_nodes -= 1
    _assert_same(c.run("paf"), fresh["paf"], "PAF chain after a refused configure")
    c.configure("global")
    c.glb.cms_buffer = c.m.cm.n_buffers
    with pytest.raises(SleapB200Error):
        c.configure("global")
    _assert_same(c.run("global"), fresh["global"], "global chain after a refused configure")


def test_configure_detaches_the_tracker(frames):
    from sleap_b200._lib import SleapB200Error
    from sleap_b200.nn import paf_grouping as pg, tracking as T
    from sleap_b200.nn.inference import BottomUpInferenceLayer
    m = _model()
    layer = BottomUpInferenceLayer(m, pg.PAFScorer(NODES, EDGES, 2), peak_threshold=0.5, max_instances=8, max_node_peaks=16)
    layer.tracker = T.Tracker.make_tracker_by_name(tracker="simple", similarity="instance", match="greedy", track_window=5,
                                                   track_device=0)
    for drop in (lambda: m.handle.call("sb_bottomup_configure", m.model_id, byref(layer.params())),
                 lambda: m.configure(B + 1, H, W, 1)):
        out = layer.call(frames)
        assert out["track_n"].shape == (B,)
        drop()
        with pytest.raises(SleapB200Error, match="no tracker attached"):
            layer.track_fields(0, B)
        m.chain = None
    layer.tracker = None


def _topdown():
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.inference import TopDownPredictor
    from sleap_b200.nn.model import DeviceModel
    ccfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=2, middle_block=True, up_interpolate=True)
    cspec = dict(backbone="unet", backbone_cfg=ccfg, head_type="centroid", part_names=None, edges=None,
                 heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
    icfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=4, middle_block=True, up_interpolate=False)
    ispec = dict(backbone="unet", backbone_cfg=icfg, head_type="centered_instance", part_names=list("abcd"), edges=None,
                 heads=[dict(name="CenteredInstanceConfmapsHead", channels=4, output_stride=4)])
    cmodel, imodel = (DeviceModel(s, la.synthetic_weights(A.compile_model(s, 1), seed), input_channels=1, precision=0)
                      for s, seed in ((cspec, 51), (ispec, 53)))
    imgs = np.random.default_rng(8).integers(0, 256, size=(3, 192, 224, 1), dtype=np.uint8)
    thr = float(np.quantile(cmodel.forward(imgs)[0], 0.9))
    pred = TopDownPredictor(cmodel, imodel, crop_size=64, peak_threshold=thr, integral_refinement=True, batch_size=3,
                            max_instances=6)
    return pred.inference_model, imgs, thr


def test_topdown_follows_its_models():
    from sleap_b200._lib import SleapB200Error
    im, imgs, _ = _topdown()
    assert im._can_fuse()
    first = im.predict_on_batch(imgs)
    staged = im.instance_peaks.call(im.centroid_crop.call(dict(image=imgs)))        # the instance model's own chain
    assert len(staged["instance_peaks"]) == len(imgs)
    again = im.predict_on_batch(imgs)
    for k in first:
        assert first[k].tobytes() == again[k].tobytes(), k
    mi = im.instance_peaks.keras_model
    mi.handle.call("sb_global_configure", mi.model_id, byref(im.instance_peaks.params()))   # behind the Python record
    with pytest.raises(SleapB200Error, match="a model was reconfigured; call sb_topdown_configure again"):
        im.predict_on_batch(imgs)


def test_centroid_cap_change_reconfigures():
    from sleap_b200.nn.inference import CentroidCrop
    from sleap_b200.nn.model import DeviceModel
    im, imgs, thr = _topdown()
    cm = im.centroid_crop.keras_model
    cc = CentroidCrop(cm, crop_size=64, peak_threshold=thr, max_peaks_per_sample=64, return_crops=False)
    wide = cc.call(dict(image=imgs))
    cc.max_peaks_per_sample = 4
    narrow = cc.call(dict(image=imgs))
    twin = DeviceModel(cm.spec, la.synthetic_weights(cm.cm, 51), input_channels=1, precision=0)
    want = CentroidCrop(twin, crop_size=64, peak_threshold=thr, max_peaks_per_sample=4, return_crops=False).call(dict(image=imgs))
    assert max(len(c) for c in wide["centroids"]) > 4
    for k in ("centroids", "centroid_vals"):
        for s in range(len(imgs)):
            assert len(narrow[k][s]) <= 4
            assert narrow[k][s].tobytes() == want[k][s].tobytes(), (k, s)

