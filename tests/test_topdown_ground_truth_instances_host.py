"""Host side of the ground-truth instances top-down step (a centroid model with FindInstancePeaksGroundTruth): the
instance table sb_topdown_gt_instances_submit takes, the growth of its capacity N, and the batch dict built from the
collect's arrays, whose centroid and instance arrays have two widths, as the host route's have."""
import numpy as np
import pytest
from numpy.testing import assert_array_equal

F = np.float32


def test_instance_table_packing():
    from sleap_b200.nn.inference import _instance_table
    a = np.arange(12, dtype=np.float64).reshape(2, 3, 2)
    a[1, 2] = np.nan
    insts = [a, np.zeros((0, 3, 2), F), np.full((1, 3, 2), np.nan, F)]
    table, counts = _instance_table(insts, 4, 3)
    assert table.dtype == F and table.shape == (3, 4, 3, 2) and table.flags.c_contiguous
    assert counts.dtype == np.int32 and counts.tolist() == [2, 0, 1]
    assert_array_equal(table[0, :2], a.astype(F))                    # NaN nodes kept in place
    assert np.isnan(table[2, 0]).all()
    for b, n in enumerate(counts):
        assert np.isnan(table[b, n:]).all()
    # more instances than N: the count is kept, so the submit refuses the batch instead of dropping instances
    table, counts = _instance_table([np.zeros((5, 3, 2), F)], 2, 3)
    assert table.shape == (1, 2, 3, 2) and counts.tolist() == [5]
    table, counts = _instance_table([], 1, 3)
    assert table.shape == (0, 1, 3, 2) and counts.shape == (0,)


@pytest.mark.parametrize("insts,want", [
    ([np.zeros((2, 3, 2)), np.zeros((0, 3, 2))], 3),
    ([np.zeros((0, 5, 2)), np.zeros((1, 3, 2))], None),              # the host dict is 5 nodes wide: rows of 3 do not fit
    ([np.zeros((0, 2, 2)), np.zeros((1, 4, 2))], 4),
    ([np.zeros((0, 0, 2)), np.zeros((0,))], None),                  # no nodes
    ([np.zeros((1, 3, 3))], None),
])
def test_instance_nodes(insts, want):
    from sleap_b200.nn.inference import _instance_nodes
    assert _instance_nodes(insts) == want


def _host_match(insts, cents):
    """FindInstancePeaksGroundTruth.call's rule as the device restates it, per frame: the picks of the kept centroids."""
    picks = []
    for inst, cent in zip(insts, cents):
        rows = []
        for cx, cy in cent:
            d = [np.nanmin(np.sqrt((inst[j, :, 0] - F(cx)) ** 2 + (inst[j, :, 1] - F(cy)) ** 2)) if not np.isnan(inst[j]).all()
                 else np.nan for j in range(len(inst))]
            if not len(d) or np.isnan(d).all():
                continue
            best = 0
            for j in range(1, len(d)):
                if d[j] < d[best]:
                    best = j
            rows.append(best)
        picks.append(rows)
    return picks


class _Handle:
    """Records the calls and answers sb_topdown_gt_instances_collect with the records of ``frames``."""

    def __init__(self, frames=None):
        self.calls, self.frames = [], frames

    def call(self, name, *args):
        self.calls.append((name, args))
        if name != "sb_topdown_gt_instances_collect":
            return
        ce, cv, nc, ip, iv, nr, fl = args[3:]
        K = ce.shape[1]
        for a in (ce, cv, ip, iv):
            a[:] = np.nan
        for b, (cent, inst, rows) in enumerate(self.frames):
            ce[b, :len(cent)], cv[b, :len(cent)], nc[b] = cent, 0.5, len(cent)
            ip[b, :len(rows)], iv[b, :len(rows)], nr[b] = inst[rows], 1.0, len(rows)
            fl[b] = 2 * b
        assert K >= max(len(c) for c, _, _ in self.frames)


def _model(handle, max_instances=None):
    from sleap_b200._lib import CentroidParams
    from sleap_b200.nn.inference import FindInstancePeaksGroundTruth, TopDownInferenceModel

    class Dev:
        model_id, chain, configured_for = 3, None, None

    class Crop:
        crop_size, precrop_resize, max_peaks_per_sample = 1, 1.0, 16

        def params(self):
            return CentroidParams(0, -1, 4, 0.2, 1, 5, 1.0, 16)

    cc = Crop()
    cc.max_instances, cc.keras_model = max_instances, Dev()
    cc.keras_model.handle = handle
    return TopDownInferenceModel(cc, FindInstancePeaksGroundTruth())


def test_capacity_grows_only_when_a_batch_exceeds_it():
    h = _Handle()
    im = _model(h, max_instances=3)
    mc = im.centroid_crop.keras_model
    assert im._configure_gt_instances(4, 0, 2, (32, 48, 1)) == (3, 1)          # N at least 1; K = max_instances
    assert im._configure_gt_instances(2, 1, 2, (32, 48, 1)) == (3, 1)
    assert len(h.calls) == 1
    assert im._configure_gt_instances(2, 5, 2, (32, 48, 1)) == (3, 5)          # N grows, B stays the larger
    assert h.calls[-1][1][1:] == (2, 5, 4, 32, 48, 1)
    assert mc.configured_for == (4, 32, 48, 1) and mc.chain[0] == "sb_topdown_gt_instances_configure"
    assert im._configure_gt_instances(4, 3, 2, (32, 48, 1)) == (3, 5) and len(h.calls) == 2
    mc.chain = ("sb_centroid_configure", b"")                                   # another chain dropped the pipeline
    assert im._configure_gt_instances(1, 1, 2, (32, 48, 1)) == (3, 1) and len(h.calls) == 3
    assert im._configure_gt_instances(1, 1, 3, (32, 48, 1)) == (3, 1) and len(h.calls) == 4   # other node count
    assert im._configure_gt_instances(1, 1, 3, (16, 48, 1)) == (3, 1) and len(h.calls) == 5   # other frames


def test_batch_dict_widths_equal_the_host_route(monkeypatch):
    """Centroids padded to the batch's most centroids, instances to its most rows: the host route's dict, key for key,
    dtype for dtype, NaN for NaN."""
    from sleap_b200.nn import inference as inf
    rng = np.random.default_rng(3)
    insts = [rng.uniform(0, 40, (3, 2, 2)).astype(F), np.zeros((0, 2, 2), F), rng.uniform(0, 40, (2, 2, 2)).astype(F),
             np.full((1, 2, 2), np.nan, F)]
    insts[0][0] = np.nan                                                         # all-NaN instance 0: kept as a pick
    insts[2][1, 0] = np.nan
    cents = [rng.uniform(0, 40, (4, 2)).astype(F), rng.uniform(0, 40, (3, 2)).astype(F), np.zeros((0, 2), F),
             rng.uniform(0, 40, (5, 2)).astype(F)]
    picks = _host_match(insts, cents)
    crop_out = dict(centroids=cents, centroid_vals=[np.full(len(c), 0.5, F) for c in cents],
                    flags=np.asarray([0, 2, 4, 6], np.int32))
    host = inf.FindInstancePeaksGroundTruth().call(dict(instances=insts), crop_out)
    assert [len(p) for p in host["instance_peaks"]] == [len(p) for p in picks] == [4, 0, 0, 0]
    ip, nv = inf._ragged_to_dense(host["instance_peaks"], (2, 2))
    iv, _ = inf._ragged_to_dense(host["instance_peak_vals"], (2,))
    want = {"centroids": inf._ragged_to_dense(cents, (2,))[0], "centroid_vals": inf._ragged_to_dense(crop_out["centroid_vals"], ())[0],
            "instance_peaks": ip, "instance_peak_vals": iv, "n_valid": nv, "flags": crop_out["flags"]}
    monkeypatch.setattr(inf, "ptr", lambda a: a)
    im = _model(_Handle([(c, i, p) for c, i, p in zip(cents, insts, picks)]))
    got = im._run_gt_instances(4, 16, 2, 0)
    assert list(got) == list(want)
    for k in want:
        assert got[k].dtype == want[k].dtype and got[k].shape == want[k].shape, k
        assert_array_equal(got[k], want[k], err_msg=k)
    assert got["centroids"].shape[1] == 5 and got["instance_peaks"].shape[1] == 4
