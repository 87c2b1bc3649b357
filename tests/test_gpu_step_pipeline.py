"""Every step of the pipelined bottom-up loop that bench.py times, against per-batch runs and the oracle.

bench.py calls sb_infer_bottomup_dev back to back on resident frames.  The post-processing of step k (peaks, PAF
scoring, LSAP, grouping) runs on the handle's second stream while step k+1's network runs on the first; only the wait
run_program queues before the model's guard op (the first op that writes a head buffer) keeps step k+1 from
overwriting the maps step k is still reading, and programmatic dependent launch lets step k+1's first launch start
while step k's last head launch drains.

The recorder below is that loop: a non-default stream set on the handle, K batches of distinct frames resident, no host
synchronisation between steps, forward timing on, and after each step a copy of the device records into slot k of a
device history, queued on the post-processing stream behind the step's grouping kernel (where bench.py's NCCL fallback
queues its gather).  Every step is then compared with
  * the same batch run alone through the synchronous entry (sb_infer_bottomup, under predict_on_batch), bit for bit,
    NaNs included.  A frame's outputs do not depend on its batch (test_gpu_batch_audit.py), so a difference is a hazard
    between steps;
  * the oracle's post-processing of the device's own maps of that batch (instance count, missing nodes and peak values
    exact, coordinates within 1e-4 of a map cell, instance scores within 1e-4).
Cases: C4 as bench.py builds it (default, SB_DISABLE_POST_OVERLAP=1, SB_DISABLE_PDL=1), C4 at precision 2, a network
that reaches its heads in microseconds fed crowded maps, submit/collect, an attached device tracker, two models on one
handle, and a heads fetch and a per-op profile between steps.  In C4 the heads are written at the end of a forward of
milliseconds, so a missing guard wait would rarely show there; the crowded-maps network is the case that can see it,
and it measures with CUDA events that one step's post-processing outlasts the next forward up to its heads."""
import os
import re
import subprocess
import sys
import tempfile
from ctypes import byref, c_int, c_int32, c_void_p

import numpy as np
import pytest
from numpy.testing import assert_array_equal

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.dirname(os.path.abspath(__file__))
K = 6                                   # steps of every recorded loop
B = 8                                   # frames per step, as bench.py
CAPS = dict(max_peaks_per_sample=1024, max_node_peaks=32, max_instances_per_frame=32)     # bench.py's predictor


# ------------------------------------------------------------------------------------------------ records
def _n_fields(I, C):
    """Floats of a record that carry a value: peaks | peak values | instance scores | n_valid | flags (then padding)."""
    return I * C * 3 + I + 2


def _field_name(i, I, C):
    if i < I * C * 2:
        j, r = divmod(i, C * 2)
        return f"instance_peaks[instance {j}, node {r // 2}, {'xy'[r % 2]}]"
    i -= I * C * 2
    if i < I * C:
        return f"instance_peak_vals[instance {i // C}, node {i % C}]"
    i -= I * C
    return f"instance_scores[instance {i}]" if i < I else ("n_valid" if i == I else "flags")


def assert_records_equal(got, want, I, C, what, ref):
    """got, want: (steps, B, record width) float32; bit for bit over the fields that carry a value."""
    n = _n_fields(I, C)
    g = np.ascontiguousarray(got[..., :n]).view(np.uint32)
    w = np.ascontiguousarray(want[..., :n]).view(np.uint32)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = np.argwhere(g != w)
    if bad.size:
        k, b, i = (int(x) for x in bad[0])
        frames = len({(int(x), int(y)) for x, y, _ in bad})
        raise AssertionError(f"{what}: step {k} frame {b}: {_field_name(i, I, C)} is {got[k, b, i]!r} where {ref} has "
                             f"{want[k, b, i]!r} ({len(bad)} fields differ, in {frames} frames)")


def _unpack(rec, I, C):
    Bn = rec.shape[0]
    peaks = rec[:, :I * C * 2].reshape(Bn, I, C, 2)
    vals = rec[:, I * C * 2:I * C * 3].reshape(Bn, I, C)
    scores = rec[:, I * C * 3:I * C * 3 + I]
    return peaks, vals, scores, rec[:, I * C * 3 + I].astype(np.int64), rec[:, I * C * 3 + I + 1].astype(np.int64)


def sync_records(handle, model_id, frames, I, C):
    """One batch through the synchronous entry (sb_infer_bottomup, what predict_on_batch calls; here with every instance
    slot kept), packed as the grouping kernel packs a device record."""
    from sleap_b200 import parallel
    from sleap_b200._lib import ptr
    frames = np.ascontiguousarray(frames)
    n = len(frames)
    ip = np.zeros((n, I, C, 2), np.float32); iv = np.zeros((n, I, C), np.float32); isc = np.zeros((n, I), np.float32)
    nv = np.zeros((n,), np.int32); fl = np.zeros((n,), np.int32)
    handle.call("sb_infer_bottomup", model_id, ptr(frames), n, ptr(ip), ptr(iv), ptr(isc), ptr(nv), ptr(fl))
    rec = np.zeros((n, parallel.record_width(I, C)), np.float32)
    o = I * C * 3 + I
    rec[:, :o] = np.concatenate([ip.reshape(n, -1), iv.reshape(n, -1), isc], axis=1)
    rec[:, o], rec[:, o + 1] = nv, fl
    return rec


def records_view(handle, model_id, rows, I, C):
    """torch view of the model's device records (written by the grouping kernel's epilogue)."""
    import torch
    from sleap_b200 import parallel
    p = c_void_p()
    handle.call("sb_bottomup_device_records", model_id, byref(p))

    class _V:
        pass
    v = _V()
    v.__cuda_array_interface__ = {"shape": (rows, parallel.record_width(I, C)), "typestr": "<f4", "data": (p.value, False),
                                  "version": 2}
    return torch.as_tensor(v, device="cuda")


def record_steps(handle, stream, plan, between=None):
    """bench.py's timed loop over plan = [(model id, frames on the device (n, H, W, 1) uint8, records view)]: one
    sb_infer_bottomup_dev per step on `stream` with no host synchronisation, each step's records copied into slot k of
    a device history on the post-processing stream, forward timing on; `between(k)` runs after step k.  Returns the
    history, one (n, width) array per step."""
    import torch
    post = c_void_p()
    handle.call("sb_get_post_stream", byref(post))
    post_stream = torch.cuda.ExternalStream(post.value)
    hist = [torch.full((f.shape[0], r.shape[1]), float("nan"), dtype=torch.float32, device="cuda") for _, f, r in plan]
    ids = sorted({mid for mid, _, _ in plan})
    for mid in ids:
        handle.call("sb_model_forward_times", mid, 1, 0, None, None)
    torch.cuda.synchronize()
    for k, (mid, frames, rec) in enumerate(plan):
        with torch.cuda.stream(stream):
            handle.call("sb_infer_bottomup_dev", mid, c_void_p(frames.data_ptr()), frames.shape[0])
        with torch.cuda.stream(post_stream):
            hist[k].copy_(rec[:frames.shape[0]])
        if between is not None:
            between(k)
    stream.wait_stream(post_stream)
    torch.cuda.synchronize()
    for mid in ids:
        n_fwd, ms = c_int32(0), np.zeros(4 * len(plan), np.float32)
        handle.call("sb_model_forward_times", mid, 0, len(ms), ms.ctypes.data_as(c_void_p), byref(n_fwd))
        assert n_fwd.value >= sum(m == mid for m, _, _ in plan) and np.all(ms[:n_fwd.value] > 0)
    return [h.cpu().numpy() for h in hist]


# ------------------------------------------------------------------------------------------------ C4 as bench.py builds it
def _configure_reporting_input_stage(layer, hw):
    """Configures (and autotunes) the predictor's model with SB_DEBUG=1 and returns the input stage the autotune picked,
    as the environment that forces the same picks in another process.  The two timed input-stage choices (the frame
    view or k_conv_first, k_conv01 or the separate launches) differ in arithmetic (test_gpu_batch_audit.py), so two
    processes compare bit for bit only at the same picks."""
    saved = os.environ.get("SB_DEBUG")
    os.environ["SB_DEBUG"] = "1"
    sys.stderr.flush()
    fd = os.dup(2)
    with tempfile.TemporaryFile(mode="w+") as log:
        os.dup2(log.fileno(), 2)
        try:
            layer._configure(B, *hw, 1)
        finally:
            os.dup2(fd, 2)
            os.close(fd)
            if saved is None:
                del os.environ["SB_DEBUG"]
            else:
                os.environ["SB_DEBUG"] = saved
        log.seek(0)
        text = log.read()
    picks = {}
    m = re.search(r"first layer: .* -> (view|direct)", text)
    if m:
        picks["SB_FORCE_FIRST_VIEW"] = "1" if m.group(1) == "view" else "0"
    m = re.search(r"first block \(B = \d+\): .* -> (fused|separate)", text)
    if m:
        picks["SB_FORCE_CONV01"] = "1" if m.group(1) == "fused" else "0"
    return picks


class C4:
    """bench.py's model and predictor (8 x 1024^2, calibrated bench weights, capacities 1024 / 32 / 32, autotuned) on a
    handle of its own whose stream is a non-default torch stream, and K batches of distinct frames."""

    def __init__(self, weights, frames, precision=0):
        import torch
        import bench
        from sleap_b200 import _lib
        from sleap_b200.nn.inference import BottomUpPredictor
        from sleap_b200.nn.model import DeviceModel
        self.handle = _lib.Handle(0)
        self.stream = torch.cuda.Stream()
        self.handle.set_stream(self.stream.cuda_stream)
        self.model = DeviceModel(bench.c4_spec(), weights, input_channels=1, precision=precision, handle=self.handle)
        self.pred = BottomUpPredictor(self.model, bench.NODES, bench.EDGES, peak_threshold=0.2, batch_size=B,
                                      integral_refinement=True, **CAPS)
        self.layer = self.pred.inference_model.bottomup_layer
        self.frames = np.ascontiguousarray(frames)
        self.hw = frames.shape[1:3]
        self.input_stage = _configure_reporting_input_stage(self.layer, self.hw)
        self.I, self.C = self.layer.max_instances, len(bench.NODES)
        self.dev = [torch.from_numpy(self.batch(k)).cuda() for k in range(len(frames) // B)]
        torch.cuda.synchronize()

    def batch(self, k):
        return np.ascontiguousarray(self.frames[k * B:(k + 1) * B])

    def reconfigure(self):
        """sb_bottomup_configure again (it reads SB_DISABLE_POST_OVERLAP); the network keeps its configuration."""
        self.model.chain = None
        self.layer._configure(B, *self.hw, 1)

    def refs(self):
        return np.stack([sync_records(self.handle, self.model.model_id, self.batch(k), self.I, self.C) for k in range(len(self.dev))])

    def record(self, between=None, steps=None):
        rec = records_view(self.handle, self.model.model_id, B, self.I, self.C)
        plan = [(self.model.model_id, self.dev[k], rec) for k in (steps if steps is not None else range(len(self.dev)))]
        return np.stack(record_steps(self.handle, self.stream, plan, between))

    def close(self):
        import torch
        torch.cuda.synchronize()
        self.handle.close()


def _c4_frames():
    import bench
    return bench.make_frames(K * B, 7000)


def c4_child(d):
    """SB_DISABLE_PDL=1 is read once per process: the child interpreter's half of test_c4_loop_without_pdl."""
    from sleap_b200.nn.model import load_weights_npz
    c4 = C4(load_weights_npz(os.path.join(d, "weights.npz")), np.load(os.path.join(d, "frames.npy")))
    np.save(os.path.join(d, "history.npy"), c4.record())
    np.save(os.path.join(d, "refs.npy"), c4.refs())
    c4.close()


@pytest.fixture(scope="module")
def c4():
    from test_gpu_batch_audit import _bench_weights
    c = C4(_bench_weights(), _c4_frames())
    c.ref = c.refs()
    n_inst = _unpack(c.ref.reshape(-1, c.ref.shape[-1]), c.I, c.C)[3]
    assert n_inst.sum() > 2 * K * B, n_inst                 # the calibrated heads give instances to group
    yield c
    c.close()


@pytest.fixture(scope="module")
def c4_history(c4):
    return c4.record()


def test_c4_loop_matches_per_batch(c4, c4_history):
    assert_records_equal(c4_history, c4.ref, c4.I, c4.C, "C4 loop", "the batch run alone (sb_infer_bottomup)")


def test_c4_loop_matches_oracle(c4, c4_history):
    """Steps 1 and K - 1: the oracle's peak finding and PAF grouping on the device's own maps of that batch."""
    import bench
    from oracle import paf_grouping as opg, peak_finding as opf
    stride = 4
    for k in (1, K - 1):
        cms, pafs = c4.model.forward(c4.batch(k))
        p, v, si, ci = opf.find_local_peaks(cms, 0.2, "integral", 5)
        p = (p * np.float32(stride)).astype(np.float32)
        winst, wps, wisc, *_ = opg.PAFScorer(bench.NODES, bench.EDGES, 8).predict(
            pafs, [p[si == b] for b in range(B)], [v[si == b] for b in range(B)], [ci[si == b] for b in range(B)])
        peaks, vals, scores, n_valid, flags = _unpack(c4_history[k], c4.I, c4.C)
        for b in range(B):
            what = f"C4 loop step {k} frame {b} vs the oracle post-processing of the device maps"
            n = int(n_valid[b])
            assert flags[b] == 0 and n == len(winst[b]), (what, int(flags[b]), n, len(winst[b]))
            if n == 0:
                continue
            assert_array_equal(np.isnan(peaks[b, :n]), np.isnan(winst[b]), err_msg=what + ": missing nodes")
            assert_array_equal(np.nan_to_num(vals[b, :n], nan=-1), np.nan_to_num(wps[b], nan=-1), err_msg=what + ": peak values")
            d_xy = np.nanmax(np.abs(peaks[b, :n] - winst[b])) / stride
            d_sc = np.abs(scores[b, :n] - wisc[b]).max()
            assert d_xy <= 1e-4 and d_sc <= 1e-4, (what, float(d_xy), float(d_sc))


def test_c4_loop_without_post_overlap(c4, c4_history, monkeypatch):
    """SB_DISABLE_POST_OVERLAP=1: the post-processing does not overlap the next network; the same records, and the
    records are still ready for a consumer queued on the post-processing stream."""
    monkeypatch.setenv("SB_DISABLE_POST_OVERLAP", "1")
    c4.reconfigure()
    try:
        hist = c4.record()
    finally:
        monkeypatch.delenv("SB_DISABLE_POST_OVERLAP")
        c4.reconfigure()
    assert_records_equal(hist, c4_history, c4.I, c4.C, "C4 loop, SB_DISABLE_POST_OVERLAP=1", "the default loop")
    assert_records_equal(hist, c4.ref, c4.I, c4.C, "C4 loop, SB_DISABLE_POST_OVERLAP=1", "the batch run alone")


CHILD = """
import sys
sys.path[:0] = [sys.argv[2], sys.argv[3]]
import test_gpu_step_pipeline as t
t.c4_child(sys.argv[1])
"""


def test_c4_loop_without_pdl(c4, c4_history, tmp_path):
    """SB_DISABLE_PDL=1 in a child interpreter (the switch is read once per process).  The child's loop equals its own
    per-batch runs (a hazard between steps without PDL), and, at the input stage this process's autotune picked, the
    default loop's records."""
    from sleap_b200.nn.model import save_weights_npz
    from test_gpu_batch_audit import _bench_weights
    assert "SB_FORCE_CONV01" in c4.input_stage, c4.input_stage          # C4's first block has both forms to pick from
    save_weights_npz(str(tmp_path / "weights.npz"), _bench_weights())
    np.save(tmp_path / "frames.npy", c4.frames)
    env = dict(os.environ, SB_DISABLE_PDL="1", PYTHONPATH=ROOT, **c4.input_stage)
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", CHILD, str(tmp_path), ROOT, TESTS], cwd=ROOT, env=env,
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    hist = np.load(tmp_path / "history.npy")
    assert_records_equal(hist, np.load(tmp_path / "refs.npy"), c4.I, c4.C, "C4 loop, SB_DISABLE_PDL=1",
                         "the batch run alone in the same process")
    assert_records_equal(hist, c4_history, c4.I, c4.C, f"C4 loop, SB_DISABLE_PDL=1, input stage {c4.input_stage}",
                         "the default loop")


def test_c4_precision2_loop_matches_per_batch(c4):
    """Precision 2 at 512 x 512 (the strict block of bench.py), the same frames cropped."""
    from test_gpu_batch_audit import _bench_weights
    c = C4(_bench_weights(), c4.frames[:, 256:768, 256:768], precision=2)
    try:
        ref = c.refs()
        assert_records_equal(c.record(), ref, c.I, c.C, "C4 precision 2 loop at 512^2", "the batch run alone")
    finally:
        c.close()


def test_c4_submit_collect_matches_per_batch(c4):
    """BottomUpPredictor.predict (sb_bottomup_submit / collect, double-buffered) on 5 batches of 8 and a ragged 3."""
    frames = np.ascontiguousarray(c4.frames[:43])
    got = c4.pred.predict(frames, make_labels=False)
    assert [len(g["n_valid"]) for g in got] == [8] * 5 + [3]
    for j, g in enumerate(got):
        want = c4.pred.inference_model.predict_on_batch(frames[8 * j:8 * j + 8])
        for key in ("instance_peaks", "instance_peak_vals", "instance_scores", "n_valid", "flags"):
            a, b = np.ascontiguousarray(g[key]), np.ascontiguousarray(want[key])
            same = a.shape == b.shape and np.array_equal(a.view(np.uint8), b.view(np.uint8))
            if not same:
                diff = np.argwhere(a != b) if a.shape == b.shape else None
                where = "shape" if diff is None else f"frame {int(diff[0][0])} at {tuple(int(x) for x in diff[0])}"
                raise AssertionError(f"submit/collect batch {j}: {key} differs from predict_on_batch of that batch ({where})")


def test_c4_loop_with_device_tracker(c4):
    """The simple tracker on the device (k_track after the grouping kernel), K steps without synchronisation: the last
    step's track records (which depend on every step before it) equal those of the same loop synchronised per step."""
    import torch
    from sleap_b200.nn import tracking as T
    kw = dict(tracker="simple", similarity="instance", match="greedy", track_window=5)
    layer = c4.layer

    def attach():
        layer.tracker = T.Tracker.make_tracker_by_name(track_device=0, **kw)
        layer.attach_tracker(c4.hw)
        return layer.tracker._device.max_instances

    try:
        Id = attach()
        synced = None
        for k in range(K):                                         # test_gpu_track_pipeline.py's per-step loop
            torch.cuda.synchronize()
            with torch.cuda.stream(c4.stream):
                c4.handle.call("sb_infer_bottomup_dev", c4.model.model_id, c_void_p(c4.dev[k].data_ptr()), B)
            synced = np.zeros((B, 2 + 3 * Id))
            c4.handle.call("sb_bottomup_device_tracks", c4.model.model_id, B, synced.ctypes.data_as(c_void_p))
        layer.detach_tracker()
        assert attach() == Id
        hist = c4.record()
        last = np.zeros((B, 2 + 3 * Id))
        c4.handle.call("sb_bottomup_device_tracks", c4.model.model_id, B, last.ctypes.data_as(c_void_p))
    finally:
        layer.detach_tracker()
        layer.tracker = None
    assert synced[:, 0].sum() > B and not synced[:, 1].any(), synced[:, :2]
    bad = np.argwhere(last.view(np.uint64) != synced.view(np.uint64))
    assert bad.size == 0, (f"device tracker, step {K - 1} frame {int(bad[0][0])}: track record field {int(bad[0][1])} is "
                           f"{last[tuple(bad[0])]!r} where the per-step synchronised loop has {synced[tuple(bad[0])]!r}")
    assert_records_equal(hist, c4.ref, c4.I, c4.C, "C4 loop with the device tracker", "the batch run alone")


def test_c4_loop_with_calls_between_steps(c4):
    """A heads fetch (sb_model_forward) of batch 5 after step 2 and a per-op profile (sb_model_profile_ops) of batch 1
    after step 3, both while that step's post-processing is pending and both on other frames than that step's, so that
    either call writing the heads too early changes the step's records.  The records are unchanged and the fetched heads
    equal batch 5's own."""
    from sleap_b200._lib import ptr
    want = c4.model.forward(c4.batch(5))
    got = {}

    def between(k):
        if k == 2:
            got["heads"] = c4.model.forward(c4.batch(5))
        if k == 3:
            n = len(c4.model.cm.ops_array())
            ms, kind, fl, n_ops = np.zeros(n, np.float32), np.zeros(n, np.int32), np.zeros(n, np.float64), c_int32(0)
            c4.handle.call("sb_model_profile_ops", c4.model.model_id, c_void_p(c4.dev[1].data_ptr()), B, n, ptr(ms),
                           ptr(kind), ptr(fl), byref(n_ops))
            got["n_ops"] = n_ops.value

    hist = c4.record(between)
    assert got["n_ops"] > 0
    for name, a, b in zip(("cms", "pafs"), got["heads"], want):
        bad = np.argwhere(a.view(np.uint32) != b.view(np.uint32))
        assert bad.size == 0, (f"heads of batch 5 fetched between steps 2 and 3: {name} frame {int(bad[0][0])} "
                               f"differs from the batch's own heads in {len(bad)} elements")
    assert_records_equal(hist, c4.ref, c4.I, c4.C, "C4 loop with a heads fetch and a per-op profile between steps",
                         "the batch run alone")


# ------------------------------------------------------------------------------------------------ hazard-exposing network
# PREPROCESS -> 3x3 conv 1 -> 16 (channel k < 9 is the frame shifted by tap k) -> two 1x1 heads: node c's map is the
# frame shifted by tap SHIFT[c], each PAF is a constant unit vector along its edge plus half the frame.  The frames hold
# 120 bright spots on a jittered grid, so every node has 120 peaks, every edge a 120 x 120 LSAP and every frame about 120
# instances.  test_hazard_loop_matches_per_batch measures that the post-processing of a step outlasts the next forward
# up to its heads, so that with the guard wait missing, later forwards would overwrite maps still being read.
HZ_HW = 256
HZ_NODES = 6
HZ_EDGES = [(c, c + 1) for c in range(HZ_NODES - 1)]
HZ_SHIFT = [0, 1, 2, 3, 4, 5]
HZ_SPOTS = 120
HZ_I = 128


def _hz_pos(c):
    """(x, y) of node c's peak relative to the spot: map c(y, x) = frame(y + ky - 1, x + kx - 1)."""
    ky, kx = divmod(HZ_SHIFT[c], 3)
    return np.array([1 - kx, 1 - ky], np.float64)


def hazard_frames(n, seed):
    rng = np.random.default_rng(seed)
    out = rng.integers(0, 31, size=(n, HZ_HW, HZ_HW, 1), dtype=np.uint8)         # background below the 0.2 threshold
    gy, gx = np.divmod(np.arange(HZ_SPOTS), 12)
    for f in range(n):
        ys = (12 + 24 * gy + rng.integers(-3, 4, HZ_SPOTS)).astype(int)
        xs = (12 + 20 * gx + rng.integers(-3, 4, HZ_SPOTS)).astype(int)
        for y, x in zip(ys, xs):
            v = int(rng.integers(150, 256))
            out[f, y - 1:y + 2, x - 1:x + 2, 0] = (v * rng.uniform(0.2, 0.6, (3, 3))).astype(np.uint8)
            out[f, y, x, 0] = v
    return out


def hazard_model(handle, batch):
    """Loads, configures (network and bottom-up) the hazard network on `handle`; returns its model id."""
    from sleap_b200._lib import BottomUpParams, ptr
    from sleap_b200.nn import oplist as ol
    from sleap_b200.nn import paf_grouping as pg
    M, C, E = 16, HZ_NODES, len(HZ_EDGES)
    recs = [ol.buffer_record(0, 1, 1, 0, 1), ol.buffer_record(1, 1, M, 0, 0), ol.buffer_record(2, 1, C, 1, 0),
            ol.buffer_record(3, 1, 2 * E, 1, 0), ol.preprocess_record(0, 1, 1.0, 1)]
    w0 = np.zeros((3, 3, 1, M), np.float32)
    for k in range(9):
        w0[k // 3, k % 3, 0, k] = 1.0
    recs.append(ol.conv_record(0, 0, 1, 1, 0, M, 3, 1, False, 0, w0.size))
    off = w0.size + M
    wc = np.zeros((M, C), np.float32)
    for c in range(C):
        wc[HZ_SHIFT[c], c] = 1.0
    recs.append(ol.conv_record(1, 0, M, 2, 0, C, 1, 1, False, off, off + wc.size))
    off += wc.size + C
    wp, bp = np.zeros((M, 2 * E), np.float32), np.zeros(2 * E, np.float32)
    for e, (s, d) in enumerate(HZ_EDGES):
        u = _hz_pos(d) - _hz_pos(s)
        bp[2 * e:2 * e + 2] = u / np.linalg.norm(u)
        wp[4, 2 * e:2 * e + 2] = 0.5
    recs.append(ol.conv_record(1, 0, M, 3, 0, 2 * E, 1, 1, False, off, off + wp.size))
    blob = np.concatenate([w0.reshape(-1), np.zeros(M, np.float32), wc.reshape(-1), np.zeros(C, np.float32),
                           wp.reshape(-1), bp]).astype(np.float32)
    ops = np.ascontiguousarray(np.stack(recs).astype(np.int32))
    mid = c_int(-1)
    handle.call("sb_load_model", ptr(ops), ops.shape[0], ptr(blob), int(blob.size), 0, byref(mid))
    handle.call("sb_model_configure", mid.value, batch, HZ_HW, HZ_HW, 1)
    names = [str(c) for c in range(C)]
    ps = pg.PAFScorer(names, [(names[s], names[d]) for s, d in HZ_EDGES], 1)
    edges = np.ascontiguousarray(np.asarray(ps.edge_inds, np.int32).reshape(-1, 2))
    sorted_e = np.ascontiguousarray(np.asarray(list(ps.sorted_edge_inds), np.int32))
    p = BottomUpParams(2, 3, -1, 1, 1, 0.2, 1, 5, C, E, edges.ctypes.data, sorted_e.ctypes.data, len(sorted_e), 10, 0.25,
                       1.0, 0.25, 0, 1.0, 1024, 128, HZ_I)
    handle.call("sb_bottomup_configure", mid.value, byref(p))
    return mid.value


def _hazard_refs(handle, mid, frames):
    ref = np.stack([sync_records(handle, mid, frames[k * B:(k + 1) * B], HZ_I, HZ_NODES) for k in range(len(frames) // B)])
    _, _, _, n_valid, flags = _unpack(ref.reshape(-1, ref.shape[-1]), HZ_I, HZ_NODES)
    assert not flags.any() and n_valid.min() >= 100, (n_valid, flags)        # crowded: ~120 instances per frame
    return ref


def hazard_times(handle, stream, mid, frames_dev):
    """(post-processing of one step, the forward up to its first head op), in ms by CUDA events: the first from the end
    of the step's network on the handle's stream to the end of its post-processing on the post-processing stream, the
    second the per-op times (sb_model_profile_ops) of the PREPROCESS and 3x3 conv ops."""
    import torch
    from sleap_b200._lib import ptr
    cap = 16
    ms, kind, fl, n_ops = np.zeros(cap, np.float32), np.zeros(cap, np.int32), np.zeros(cap, np.float64), c_int32(0)
    handle.call("sb_model_profile_ops", mid, c_void_p(frames_dev.data_ptr()), B, cap, ptr(ms), ptr(kind), ptr(fl),
                byref(n_ops))
    assert n_ops.value == 4
    post = c_void_p()
    handle.call("sb_get_post_stream", byref(post))
    post_stream = torch.cuda.ExternalStream(post.value)
    fwd_end, post_end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    with torch.cuda.stream(stream):
        handle.call("sb_infer_bottomup_dev", mid, c_void_p(frames_dev.data_ptr()), frames_dev.shape[0])
        fwd_end.record(stream)
    post_end.record(post_stream)
    torch.cuda.synchronize()
    return fwd_end.elapsed_time(post_end), float(ms[:2].sum())


def test_hazard_loop_matches_per_batch():
    """Distinct frames per step: if step k+1's heads were written before step k's post-processing finished, step k's
    records would be built (in part) from the wrong frame's maps."""
    import torch
    from sleap_b200 import _lib
    handle = _lib.Handle(0)
    stream = torch.cuda.Stream()
    handle.set_stream(stream.cuda_stream)
    try:
        mid = hazard_model(handle, B)
        frames = hazard_frames(K * B, 31)
        ref = _hazard_refs(handle, mid, frames)
        dev = [torch.from_numpy(np.ascontiguousarray(frames[k * B:(k + 1) * B])).cuda() for k in range(K)]
        rec = records_view(handle, mid, B, HZ_I, HZ_NODES)
        hist = np.stack(record_steps(handle, stream, [(mid, dev[k], rec) for k in range(K)]))
        assert_records_equal(hist, ref, HZ_I, HZ_NODES, "hazard network loop", "the batch run alone (sb_infer_bottomup)")
        post_ms, heads_ms = hazard_times(handle, stream, mid, dev[1])
        print(f"hazard network: post-processing of one step {post_ms:.3f} ms, forward up to the heads {heads_ms:.3f} ms")
        assert post_ms > 4 * heads_ms, (post_ms, heads_ms)
    finally:
        torch.cuda.synchronize()
        handle.close()


def test_two_models_on_one_handle(c4):
    """C4 and the hazard network interleaved on C4's handle (A, B, A, B, ...): they share the handle's post-processing
    event and pending flag but each has its own guard op.  Each model's steps equal its own per-batch runs."""
    import torch
    mid = hazard_model(c4.handle, B)
    frames = hazard_frames(K * B, 32)
    ref_b = _hazard_refs(c4.handle, mid, frames)
    dev_b = [torch.from_numpy(np.ascontiguousarray(frames[k * B:(k + 1) * B])).cuda() for k in range(K)]
    rec_a = records_view(c4.handle, c4.model.model_id, B, c4.I, c4.C)
    rec_b = records_view(c4.handle, mid, B, HZ_I, HZ_NODES)
    plan = []
    for k in range(K):
        plan += [(c4.model.model_id, c4.dev[k], rec_a), (mid, dev_b[k], rec_b)]
    hist = record_steps(c4.handle, c4.stream, plan)
    assert_records_equal(np.stack(hist[0::2]), c4.ref, c4.I, c4.C, "C4 interleaved with the hazard network",
                         "the C4 batch run alone")
    assert_records_equal(np.stack(hist[1::2]), ref_b, HZ_I, HZ_NODES, "hazard network interleaved with C4",
                         "the hazard batch run alone")
