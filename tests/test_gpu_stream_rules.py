"""The rules every streamed (submit / collect) step follows (include/sleap_b200.h, "Streamed steps"), form by form on small
models: single-instance, bottom-up, bottom-up identity, top-down, top-down identity and ground-truth top-down (plain and
identity).

Each refusal is SB_ERR_INVALID with its message and queues nothing: a bad slot or B, a submit into a slot that holds a
batch, a collect of an empty slot, with another B or out of submit order, a second collect of a slot, and (bottom-up and
top-down with a device tracker) a tracks read of a slot before its collect or with another B.  After the refusals the
in-order collects still equal predict_on_batch bit for bit, and a configure call between a submit and its collect makes
the collect fail cleanly while the next stream runs.

The synchronous call of a form (predict_on_batch: sb_infer_global, sb_infer_bottomup, sb_infer_multiclass,
sb_infer_topdown, sb_infer_topdown_multiclass) is a submit into slot 0 and its collect: it is refused while a batch is
submitted and not collected, and its track records are then slot 0's (slot -1 is refused)."""
import numpy as np
import pytest

import reference_models as rm
from sleap_b200 import _lib
from sleap_b200.nn import tracking as T

pytestmark = pytest.mark.gpu

B = 2
NODES = list("abcd")
SIMPLE = dict(tracker="simple", similarity="instance", match="greedy", track_window=5)
FORMS = ["single_instance", "bottomup", "bottomup_identity", "topdown", "topdown_identity", "ground_truth",
         "ground_truth_identity"]


def _unet(output_stride, up_interpolate=True):
    return dict(filters=8, filters_rate=2, max_stride=16, output_stride=output_stride, middle_block=True, up_interpolate=up_interpolate)


def _variants(img, n):
    """n distinct frames from one: flips and rolls."""
    return np.ascontiguousarray(np.stack([np.roll(img[::-1] if k % 2 else img, 7 * (k // 2), axis=1) for k in range(n)]))


def _synthetic(spec, seed, **kw):
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    return DeviceModel(spec, A.make_synthetic_weights(A.compile_model(spec, 1), seed), input_channels=1, precision=0, **kw)


def _instance_spec():
    return dict(backbone="unet", backbone_cfg=_unet(4, False), head_type="centered_instance", part_names=NODES, edges=None,
                heads=[dict(name="CenteredInstanceConfmapsHead", channels=len(NODES), output_stride=4)])


def _class_model():
    """The centered-instance UNet with a 3-class ClassVectorsHead of tools/sanitize_stream.py."""
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    classes = ["c0", "c1", "c2"]
    ispec = _instance_spec()
    mspec = dict(ispec, head_type="multi_class_topdown", classes=classes,
                 heads=ispec["heads"] + [dict(name="ClassVectorsHead", channels=len(classes), output_stride=16, vector=True,
                                              num_fc_layers=1, num_fc_units=16, global_pool=True)])
    icm = A.compile_model(mspec, 1)
    iw = A.make_synthetic_weights(icm, 65)
    rng = np.random.default_rng(67)
    dims = [icm.vector_taps["ClassVectorsHead"]["C"], 16, len(classes)]
    for i, name in enumerate(["pre_classification0_fc", "ClassVectorsHead"]):
        iw[name] = dict(kernel=(rng.normal(0, 1, dims[i:i + 2]) * np.sqrt(2.0 / dims[i])).astype(np.float32),
                        bias=rng.normal(0, 0.1, dims[i + 1]).astype(np.float32))
    return DeviceModel(mspec, iw, input_channels=1, precision=0)


def _centroid_model(frames):
    spec = dict(backbone="unet", backbone_cfg=_unet(2), head_type="centroid", part_names=None, edges=None,
                heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
    m = _synthetic(spec, 61)
    return m, max(float(np.quantile(m.forward(frames[:B])[0], 0.99)), 1e-3)


class Form:
    """One streamed form: its inference model, two batches of B frames (examples, for ground truth), the per-batch
    results, and the tracks call when it runs a device tracker."""

    def __init__(self, name):
        from sleap_b200.nn.inference import (Predictor, SingleInstancePredictor, TopDownMultiClassPredictor,
                                             TopDownPredictor)
        self.name, self.tracks, self.layer = name, None, None
        self.gt = name.startswith("ground_truth")
        rng = np.random.default_rng(9)
        synth = rng.integers(0, 256, size=(2 * B, 192, 224, 1), dtype=np.uint8)
        if name == "single_instance":
            spec = dict(backbone="unet", backbone_cfg=_unet(2), head_type="single_instance", part_names=NODES, edges=None,
                        heads=[dict(name="SingleInstanceConfmapsHead", channels=len(NODES), output_stride=2)])
            self.im, frames = SingleInstancePredictor(_synthetic(spec, 59), batch_size=B).inference_model, synth
        elif name == "bottomup":
            self.im = Predictor.from_model_paths([rm.model_dir("minimal_instance.bottomup")], precision=1, batch_size=B).inference_model
            frames = _variants(rm.frames("minimal_instance")[0][0], 2 * B)
            self.layer, self.tracks = self.im.bottomup_layer, "sb_bottomup_tracks"
        elif name == "bottomup_identity":
            paths = [rm.model_dir("min_tracks_2node.bottomup_multiclass")]
            self.im = Predictor.from_model_paths(paths, precision=1, batch_size=B).inference_model
            frames = _variants(rm.frames("tracks_2node")[0][0][:512, :512], 2 * B)
        elif name in ("topdown", "topdown_identity"):
            cm, thr = _centroid_model(synth)
            if name == "topdown":
                pred = TopDownPredictor(cm, _synthetic(_instance_spec(), 63), crop_size=64, peak_threshold=thr, batch_size=B,
                                        max_instances=4)
                self.tracks = "sb_topdown_tracks"
            else:
                pred = TopDownMultiClassPredictor(cm, _class_model(), crop_size=64, peak_threshold=thr, batch_size=B, max_instances=4)
            self.im = pred.inference_model
            self.layer = self.im if self.tracks else None
            self.im.instance_peaks.peak_threshold = 0.0
            self.im.instance_peaks.max_crops_per_call = 3
            frames = synth
        else:
            if name == "ground_truth":
                pred = TopDownPredictor(None, _synthetic(_instance_spec(), 63), crop_size=64, peak_threshold=0.05, batch_size=B)
            else:
                pred = TopDownMultiClassPredictor(None, _class_model(), crop_size=64, integral_refinement=True, batch_size=B)
            self.im = pred.inference_model
            self.im.instance_peaks.peak_threshold = 0.0
            assert self.im.ground_truth and self.im._can_fuse()
            cents = [rng.uniform(0, [224, 192], (n, 2)).astype(np.float32) for n in (2, 0, 3, 1)]
            frames = [dict(image=synth[i:i + B], centroids=cents[i:i + B]) for i in range(0, 2 * B, B)]
        if not self.gt:
            frames = [np.ascontiguousarray(frames[i:i + B]) for i in range(0, 2 * B, B)]
        self.batches = frames
        self.want = [self.im.predict_on_batch(b) for b in frames]

    def images(self, batch):
        from sleap_b200.nn.inference import InferenceLayer
        return InferenceLayer._prep(batch["image"] if self.gt else batch)

    def stream(self, tracker=False):
        """(device model, submit call, collect(slot, B), the submit arrays of a batch), set up for the batches."""
        from sleap_b200.nn.inference import _centroid_table
        if tracker:
            self.layer.tracker = T.Tracker.make_tracker_by_name(track_device=0, **SIMPLE)
        first = self.images(self.batches[0])
        if not self.gt:
            m, fn, collect = self.im._stream(first, B)
            return m, fn, collect, lambda b: (self.images(b),)
        maxc = max(len(c) for b in self.batches for c in b["centroids"])
        (m, fn, collect), K = self.im._stream_ground_truth(first, B, maxc)
        return m, fn, collect, lambda b: (self.images(b),) + _centroid_table(b["centroids"], K)

    def untrack(self):
        if self.layer is not None and self.layer.tracker is not None:
            self.layer.detach_tracker()
            self.layer.tracker = None


@pytest.fixture(scope="module", params=FORMS)
def form(request):
    return Form(request.param)


def _same(got, want, what):
    """Every field of the per-batch result, bit for bit (a stream with a tracker adds its track fields)."""
    for k in want:
        a, b = np.asarray(got[k]), np.asarray(want[k])
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), (what, k)


def test_refusals_keep_the_stream(form):
    m, fn, collect, args = form.stream(tracker=form.tracks is not None)
    keep = [args(b) for b in form.batches]          # the host arrays stay alive until their batch is collected

    def submit(k, slot, n=B):
        m.handle.call(fn, m.model_id, *[_lib.ptr(a) for a in keep[k]], n, slot)

    def fails(msg, call, *a):
        with pytest.raises(_lib.SleapB200Error, match=msg):
            call(*a)

    def tracks(slot, n):
        rec = np.zeros((B, 2 + 3 * form.layer.tracker._device.max_instances))
        m.handle.call(form.tracks, m.model_id, slot, n, _lib.ptr(rec))

    try:
        fails("slot 1 holds no submitted batch", collect, 1, B)
        fails("bad slot / batch", submit, 0, 2)
        fails("bad slot / batch", submit, 0, 0, B + 1)
        submit(0, 0)
        fails("slot 0 holds a batch that was not collected", submit, 1, 0)
        fails(f"slot 0 holds a batch of {B} frames, not {B - 1}", collect, 0, B - 1)
        if form.tracks:
            fails(f"slot 0 holds no collected batch of {B} frames", tracks, 0, B)
        submit(1, 1)
        fails("slot 0 was submitted first; collect batches in submit order", collect, 1, B)
        _same(collect(0, B), form.want[0], "batch 0")
        if form.tracks:
            tracks(0, B)
            fails(f"slot 0 holds no collected batch of {B - 1} frames", tracks, 0, B - 1)
        fails("slot 0 holds no submitted batch", collect, 0, B)
        _same(collect(1, B), form.want[1], "batch 1")
    finally:
        form.untrack()


def test_reconfigure_between_submit_and_collect(form):
    m, fn, collect, args = form.stream()
    keep = args(form.batches[0])
    m.handle.call(fn, m.model_id, *[_lib.ptr(a) for a in keep], B, 0)
    m.handle.call("sb_model_configure", m.model_id, *m.configured_for)
    m.configured_for = m.chain = None
    _, _, collect, _ = form.stream()                 # the step configured again: the submitted batch is gone
    with pytest.raises(_lib.SleapB200Error):
        collect(0, B)
    m, fn, collect, args = form.stream()
    got = []
    for k, b in enumerate(form.batches):
        keep = args(b)
        m.handle.call(fn, m.model_id, *[_lib.ptr(a) for a in keep], B, k % 2)
        got.append(collect(k % 2, B))
    for k, (g, w) in enumerate(zip(got, form.want)):
        _same(g, w, f"batch {k}")


def test_sync_call_is_a_slot_0_step(form):
    if form.gt:
        pytest.skip("the ground-truth forms have no synchronous call")
    m, fn, collect, args = form.stream()
    keep = args(form.batches[0])
    m.handle.call(fn, m.model_id, *[_lib.ptr(a) for a in keep], B, 0)
    with pytest.raises(_lib.SleapB200Error, match="a batch was submitted and not collected; collect it first"):
        form.im.predict_on_batch(form.batches[1])
    _same(collect(0, B), form.want[0], "batch 0")
    if not form.tracks:
        return
    form.layer.tracker = T.Tracker.make_tracker_by_name(track_device=0, **SIMPLE)
    try:
        out = form.im.predict_on_batch(form.batches[1])
        _same(out, form.want[1], "batch 1 with a tracker")
        rec = np.full((B, 2 + 3 * form.layer.tracker._device.max_instances), -1.0)
        m.handle.call(form.tracks, m.model_id, 0, B, _lib.ptr(rec))
        assert (rec[:, 0] >= 0).all() and np.array_equal(rec[:, 0].astype(np.int64), out["track_n"])
        with pytest.raises(_lib.SleapB200Error, match="bad slot / batch"):
            m.handle.call(form.tracks, m.model_id, -1, B, _lib.ptr(rec))
    finally:
        form.untrack()
