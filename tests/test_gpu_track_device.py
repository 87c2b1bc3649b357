"""The identity tracker on the GPU (make_tracker_by_name(track_device=0): k_track in sb_track.cu) against the host
tracker with stable greedy ties, on the tracking clip, on seeded synthetic sets and on the known-answer scenarios of
tests/test_tracking.py."""
import numpy as np
import pytest

from sleap_b200.nn import tracking as T
from sleap_b200.nn.inference import LabeledFrame, PredictedInstance
from flow_clip import clip_labeled_frames
from track_cases import assert_same_tracking, copy_frames, host_twin, synthetic_frames

pytestmark = pytest.mark.gpu


def _both(frames, images=None, **kw):
    host_tr, dev_tr = host_twin(**kw), T.Tracker.make_tracker_by_name(track_device=0, **kw)
    host = T.run_tracker(copy_frames(frames), host_tr, images=images)
    dev = T.run_tracker(copy_frames(frames), dev_tr, images=images, device_chunk=97)
    assert_same_tracking(host, dev, host_tr, dev_tr)
    return host, dev


SIMS = [dict(similarity="instance"), dict(similarity="normalized_instance"), dict(similarity="centroid"),
        dict(similarity="iou"), dict(similarity="object_keypoint"),
        dict(similarity="object_keypoint", oks_errors=[3.0, 5.0, 8.0], oks_score_weighting=True),
        dict(similarity="object_keypoint", oks_errors=np.linspace(2, 9, 20), oks_normalization="ref"),
        dict(similarity="object_keypoint", oks_errors=4.0, oks_score_weighting=True, oks_normalization="union")]


@pytest.fixture(scope="module")
def clip():
    return clip_labeled_frames(300)


@pytest.mark.parametrize("sim", range(len(SIMS)))
@pytest.mark.parametrize("match", ["greedy", "hungarian"])
@pytest.mark.parametrize("tracker", ["simple", "simplemaxtracks"])
def test_clip_parity(clip, tracker, match, sim):
    kw = dict(tracker=tracker, match=match, max_tracks=2, max_tracking=tracker == "simplemaxtracks", **SIMS[sim])
    imgs = {lf.frame_idx: np.zeros((1024, 1024, 1), np.uint8) for lf in clip} if sim == 1 else None
    _both(clip, images=imgs, **kw)
    if match == "greedy":                             # on this clip the stable twin is the default host greedy
        a = T.run_tracker(copy_frames(clip), T.Tracker.make_tracker_by_name(**kw), images=imgs)
        b = T.run_tracker(copy_frames(clip), host_twin(**kw), images=imgs)
        assert [[x.track.name for x in lf.instances] for lf in a] == [[x.track.name for x in lf.instances] for lf in b]


@pytest.mark.parametrize("robust,window", [(0.95, 5), (0.95, 1), (1.0, 1), (0.5, 3)])
@pytest.mark.parametrize("tracker", ["simple", "simplemaxtracks"])
def test_clip_parity_robust_window(clip, tracker, robust, window):
    _both(clip, tracker=tracker, similarity="instance", match="hungarian", robust=robust, track_window=window, max_tracks=2,
          max_tracking=tracker == "simplemaxtracks")


STRESS = [
    dict(tracker="simple", similarity="instance", match="greedy"),
    dict(tracker="simple", similarity="centroid", match="greedy", robust=0.95, track_window=4),
    dict(tracker="simple", similarity="iou", match="greedy", target_instance_count=6, pre_cull_to_target=True,
         pre_cull_iou_threshold=0.5),
    dict(tracker="simple", similarity="object_keypoint", match="greedy", oks_errors=[6.0], oks_score_weighting=True,
         target_instance_count=8, pre_cull_to_target=True, min_new_track_points=6, min_match_points=4),
    dict(tracker="simplemaxtracks", similarity="centroid", match="hungarian", max_tracks=10, max_tracking=True),
    dict(tracker="simplemaxtracks", similarity="instance", match="greedy", max_tracks=12, max_tracking=True, robust=0.8,
         min_match_points=5, target_instance_count=12, pre_cull_to_target=True, pre_cull_iou_threshold=0.3),
    dict(tracker="simplemaxtracks", similarity="object_keypoint", match="greedy", oks_normalization="ref"),
    dict(tracker="simplemaxtracks", similarity="centroid", match="hungarian", track_window=2, min_new_track_points=8),
]


@pytest.mark.parametrize("case", range(len(STRESS)))
def test_stress_parity(case):
    kw = STRESS[case]
    _both(synthetic_frames(seed=100 + case, n_frames=300, all_nan=0.0 if kw["match"] == "hungarian" else 0.03), **kw)


def test_infeasible_hungarian_raises_like_the_host():
    """A frame whose only instance has no visible node: its similarity row is NaN, its cost row +inf, and SciPy rejects
    the matrix."""
    pts = np.array([[10.0, 10.0], [12.0, 12.0]])
    mk = lambda p: PredictedInstance.from_numpy(p, [1, 1], 1.0)
    frames = [LabeledFrame(0, 0, [mk(pts)]), LabeledFrame(0, 1, [mk(np.full((2, 2), np.nan))])]
    for tr in (host_twin(match="hungarian"), T.Tracker.make_tracker_by_name(match="hungarian", track_device=0)):
        with pytest.raises(ValueError):
            T.run_tracker(copy_frames(frames), tr)


def test_capacity_overflow_raises():
    from sleap_b200._lib import SleapB200Error
    tr = T.Tracker.make_tracker_by_name(track_device=0)
    tr.device_max_instances = 4
    frames = [LabeledFrame(0, 0, [PredictedInstance.from_numpy(np.full((3, 2), float(i)), [1, 1, 1], 1.0) for i in range(5)])]
    with pytest.raises(SleapB200Error):
        T.run_tracker(frames, tr)
    tr = T.Tracker.make_tracker_by_name(tracker="simplemaxtracks", track_device=0)
    tr.device_track_table = 3
    with pytest.raises(SleapB200Error):                # four new tracks, a queue table of three
        T.run_tracker(frames[:1] + [LabeledFrame(0, 1, frames[0].instances[:4])], tr)


# ---- the known answers of tests/test_tracking.py, on the device ----------------------------------------------------
def _make_insts(trx):
    return [[PredictedInstance.from_numpy(np.array([[-0.1, -0.1], [0.0, 0.0], [0.1, 0.1]]) + np.array([[x, y]]), [1, 1, 1], 1)
             for x, y in frame] for frame in trx]


def _n_tracks(preds, **kw):
    tracker = T.Tracker.make_tracker_by_name(match="hungarian", track_window=2, track_device=0, **kw)
    tracked = [tracker.track(insts, img_hw=(1, 1)) for insts in preds]
    return len({id(inst.track) for frame in tracked for inst in frame}), tracked


CASES = {
    "large_gap_single_track": ([[(0, 0), (0, 1)], [(0.1, 0), (0.1, 1)], [(0.2, 0), (0.2, 1)], [(0.3, 0)], [(0.4, 0)], [(0.5, 0), (0.5, 1)],
                                [(0.6, 0), (0.6, 1)]], 3),
    "small_gap_on_both_tracks": ([[(0, 0), (0, 1)], [(0.1, 0), (0.1, 1)], [(0.2, 0), (0.2, 1)], [], [], [(0.5, 0), (0.5, 1)],
                                  [(0.6, 0), (0.6, 1)]], 4),
    "extra_detections": ([[(0, 0), (0, 1)], [(0.1, 0), (0.1, 1)], [(0.2, 0), (0.2, 1)], [(0.3, 0)], [(0.4, 0)], [(0.5, 0), (0.5, 1)],
                          [(0.6, 0), (0.6, 1), (0.6, 0.5)]], 4),
}


@pytest.mark.parametrize("name", list(CASES))
def test_max_tracking_on_device(name):
    trx, n_simple = CASES[name]
    assert _n_tracks(_make_insts(trx), tracker="simple")[0] == n_simple
    n, tracked = _n_tracks(_make_insts(trx), tracker="simplemaxtracks", max_tracks=2, max_tracking=True)
    assert n == 2
    by_track = {}
    for frame in tracked:
        for inst in frame:
            by_track.setdefault(id(inst.track), set()).add(round(float(inst.numpy()[1, 1])))
    assert all(len(v) == 1 or name == "extra_detections" for v in by_track.values())


@pytest.mark.parametrize("similarity", ["instance", "normalized_instance", "iou", "centroid", "object_keypoint"])
@pytest.mark.parametrize("match", ["greedy", "hungarian"])
@pytest.mark.parametrize("tracker", ["simple", "simplemaxtracks"])
def test_tracker_by_name_on_device(tracker, similarity, match):
    shape = np.array([[-5.0, -5.0], [0.0, 0.0], [5.0, 5.0]])
    frames = [LabeledFrame(0, t, [PredictedInstance.from_numpy(shape + np.array([[10.0 + t, 10.0]]), [1, 1, 1], 1),
                                  PredictedInstance.from_numpy(shape + np.array([[60.0 - t, 40.0]]), [1, 1, 1], 1)]) for t in range(6)]
    kw = dict(tracker=tracker, similarity=similarity, match=match, max_tracks=2, max_tracking=tracker == "simplemaxtracks")
    out = T.run_tracker(copy_frames(frames), T.Tracker.make_tracker_by_name(track_device=0, **kw))
    ids = [[id(i.track) for i in lf.instances] for lf in out]
    assert all(len(set(x)) == 2 for x in ids) and all(x == ids[0] for x in ids)
    _both(frames, **kw)


def test_jump_simple_half_on_device():
    """The simple tracker cannot bridge a 6 px step with the instance similarity: at least two identities appear."""
    shape = np.array([[-8.0, 0.0], [0.0, 0.0], [8.0, 0.0]])
    pos = lambda t: (shape + [30.0 + 6 * t, 30.0], shape + [100.0 - 6 * t, 70.0])
    frames = [LabeledFrame(0, t, [PredictedInstance.from_numpy(pos(t)[0], [1, 1, 1], 1.0), PredictedInstance.from_numpy(pos(t)[1], [1, 1, 1], 1.0)])
              for t in range(6)]
    out = T.run_tracker(copy_frames(frames), T.Tracker.make_tracker_by_name(tracker="simple", similarity="instance", match="hungarian",
                                                                            track_device=0))
    assert len({i.track.name for lf in out for i in lf.instances}) >= 2
    _both(frames, tracker="simple", similarity="instance", match="hungarian")


def test_per_frame_calls_equal_chunked_calls(clip):
    """Tracker.track frame by frame (as the predictors call it, t=None included) gives what run_tracker's chunks give."""
    kw = dict(tracker="simplemaxtracks", similarity="instance", match="greedy", max_tracks=2, max_tracking=True)
    a = T.run_tracker(copy_frames(clip[:120]), T.Tracker.make_tracker_by_name(track_device=0, **kw))
    tr = T.Tracker.make_tracker_by_name(track_device="cuda:0", **kw)
    b = [tr.track(list(lf.instances)) for lf in clip[:120]]
    assert [[x.track.name for x in lf.instances] for lf in a] == [[x.track.name for x in f] for f in b]
    assert [[x.tracking_score for x in lf.instances] for lf in a] == [[x.tracking_score for x in f] for f in b]
