"""The device tracker (k_track in sb_track.cu) at its caps -- 128 instances per frame, 64 nodes, a 64-frame window, the
queue table -- and just past them, against the host tracker with stable greedy ties.  At these sizes every lane loop
of k_track runs more than one pass: the queue-entry copy (2 * 64 and 64 values over 32 lanes), the candidates of one
track (more than 32 in a 64-frame window) with their quantile sort, the greedy row clear (128 rows), the pairwise
nansum over 64 nodes, the pre-cull of 128 instances and the Hungarian solver with 128 rows."""
import numpy as np
import pytest

from sleap_b200._lib import SleapB200Error
from sleap_b200.nn import tracking as T
from sleap_b200.nn.inference import PredictedInstance
from track_cases import assert_same_tracking, copy_frames, counted_frames, host_twin, stable_argsort

pytestmark = pytest.mark.gpu

# full frames, a drop to 20 and back: both more instances than tracks (the transposed Hungarian branch at 128 rows)
# and fewer.  13 frames of 128.
JUMPS = [20, 20, 128, 128, 128, 20, 128, 128, 20, 20, 20, 128, 128, 64, 128, 100, 128, 33, 128, 128, 128, 7, 128, 128]


def _both(frames, images=None, host_ctx=None, **kw):
    host_tr, dev_tr = host_twin(**kw), T.Tracker.make_tracker_by_name(track_device=0, **kw)
    with host_ctx or stable_argsort():
        host = T.run_tracker(copy_frames(frames), host_tr, images=images)
    dev = T.run_tracker(copy_frames(frames), dev_tr, images=images)
    assert_same_tracking(host, dev, host_tr, dev_tr)
    return host, dev


def _n_matched(frames):
    return sum(x.tracking_score != 0.0 for lf in frames for x in lf.instances)


@pytest.mark.parametrize("match", ["greedy", "hungarian"])
@pytest.mark.parametrize("tracker", ["simple", "simplemaxtracks"])
def test_full_frames_and_jumps(tracker, match):
    frames = counted_frames(1, JUMPS)
    host, _ = _both(frames, tracker=tracker, match=match, track_window=2)
    assert _n_matched(host) > 1000                    # the animals are followed, not respawned every frame


# 64 nodes at 128 instances, window 2
SIMS_64 = [dict(similarity="instance"), dict(similarity="normalized_instance"), dict(similarity="iou"),
           dict(similarity="centroid"), dict(similarity="object_keypoint", oks_errors=np.linspace(2.0, 9.0, 64)),
           dict(similarity="object_keypoint", oks_errors=np.linspace(3.0, 7.0, 20)),
           dict(similarity="object_keypoint", oks_errors=5.0, oks_normalization="ref"),
           dict(similarity="object_keypoint", oks_errors=np.linspace(2.0, 9.0, 64), oks_normalization="union",
                oks_score_weighting=True)]
NODES_64 = [128, 128, 20, 128, 128, 128, 50, 128]


@pytest.mark.parametrize("sim", range(len(SIMS_64)))
def test_64_nodes_at_128_instances(sim):
    # the host's centroid (two np.nanmedian per pair) is slow: three frames there
    frames = counted_frames(2 + sim, NODES_64[:3] if SIMS_64[sim]["similarity"] == "centroid" else NODES_64, n_nodes=64)
    imgs = {lf.frame_idx: np.zeros((1024, 960, 1), np.uint8) for lf in frames} if sim == 1 else None
    tracker, match = [("simple", "greedy"), ("simplemaxtracks", "hungarian")][sim % 2]
    host, _ = _both(frames, images=imgs, tracker=tracker, match=match, track_window=2, **SIMS_64[sim])
    assert _n_matched(host) > (100 if len(frames) == 3 else 500)


@pytest.mark.parametrize("robust", [0.5, 0.95])
@pytest.mark.parametrize("tracker", ["simple", "simplemaxtracks"])
def test_window_64_quantiles(tracker, robust):
    """3-5 animals over 150 frames with a 64-frame window: from frame 33 on, every track has more than 32 candidates."""
    shown = [[0, 1, 2, 3, 4][:3 + (t // 20) % 3] for t in range(150)]
    frames = counted_frames(7, shown)
    host, _ = _both(frames, tracker=tracker, match="hungarian", track_window=64, robust=robust)
    assert len({x.track.name for lf in host for x in lf.instances}) <= 6


@pytest.mark.parametrize("iou", [0.0, 0.2])
def test_pre_cull_128_to_100_with_tied_scores(iou):
    """cull_frame_instances from up to 128 instances to 100, with scores of 6 levels (ties everywhere): every animal
    has a second detection shifted 2-40 px, so that nms_fast suppresses some of them and hands some back, then the
    score cut."""
    frames = counted_frames(3, [64, 64, 55, 64, 64, 10, 64, 64], score_levels=6)
    rng = np.random.default_rng(3)
    for lf in frames:
        lf.instances += [PredictedInstance.from_numpy(x.points + rng.uniform(2, 40, 2), x.point_confidences,
                                                      rng.integers(6) / 6) for x in lf.instances]
    kw = dict(target_instance_count=100, pre_cull_to_target=True, pre_cull_iou_threshold=iou or None)
    host, _ = _both(frames, tracker="simple", match="greedy", track_window=2, **kw)
    n = [len(lf.instances) for lf in host]
    if iou:
        assert n[2] < 100, n                        # suppressed, and fewer handed back than the target
    else:
        assert n == [100] * 5 + [20] + [100] * 2, n


def test_caps_are_accepted():
    """128 instances of 64 nodes with a 64-frame window."""
    frames = counted_frames(4, [128, 128, 128], n_nodes=64)
    _both(frames, tracker="simplemaxtracks", match="greedy", track_window=64)
    tr = T.Tracker.make_tracker_by_name(track_device=0)
    assert tr.device_max_instances == 128


@pytest.mark.parametrize("case", ["window 65", "65 nodes", "129 instances", "table 65537"])
def test_past_the_caps_is_refused_at_create(case):
    kw = dict(tracker="simplemaxtracks", track_window=65 if case == "window 65" else 64)
    tr = T.Tracker.make_tracker_by_name(track_device=0, **kw)
    if case == "129 instances":
        tr.device_max_instances = 129
    if case == "table 65537":
        tr.device_track_table = 65537
    frames = counted_frames(5, [3, 3], n_nodes=65 if case == "65 nodes" else 5)
    with pytest.raises(SleapB200Error, match="sb_tracker_create"):
        T.run_tracker(frames, tr)
    assert all(x.track is None for lf in frames for x in lf.instances)


def _fails_at(frames, bad, attrs=None, **kw):
    """The device run raises SleapB200Error at frame ``bad``; the frames before it equal the host's."""
    dev_tr = T.Tracker.make_tracker_by_name(track_device=0, **kw)
    for k, v in (attrs or {}).items():
        setattr(dev_tr, k, v)
    dev = copy_frames(frames)
    with pytest.raises(SleapB200Error, match="sb_track_instances"):
        T.run_tracker(dev, dev_tr)
    host_tr = host_twin(**kw)
    with stable_argsort():
        host = T.run_tracker(copy_frames(frames[:bad]), host_tr)
    assert_same_tracking(host, dev[:bad], host_tr, dev_tr)
    assert all(x.track is None for lf in dev[bad:] for x in lf.instances)


def test_frame_of_129_instances_raises_at_that_frame():
    frames = counted_frames(6, [128, 60, 128, 129, 10])
    _fails_at(frames, 3, tracker="simple", match="greedy", track_window=2)


def test_uncapped_queue_table_raises_at_the_track_past_it():
    """A queue table of 200 rows.  Instances with one visible node spawn tracks but are no candidates
    (min_match_points 2), so tracks keep spawning: 128 in frame 0 (100 of them one-node), 72 in frame 1 (98 instances,
    all one-node, against the 26 candidate tracks), then the 201st in frame 2."""
    frames = counted_frames(8, [128, 98, 29, 5], n_nodes=4)
    for x in frames[0].instances[28:] + frames[1].instances:
        x.points[0] = np.nanmean(x.points, 0)
        x.points[1:] = np.nan
    kw = dict(tracker="simplemaxtracks", match="greedy", track_window=3, min_match_points=2)
    host_tr = host_twin(**kw)
    T.run_tracker(copy_frames(frames), host_tr)
    assert [host_tr.spawned_tracks[k].spawned_on for k in (199, 200)] == [1, 2]
    _fails_at(frames, 2, attrs=dict(device_track_table=200), **kw)
