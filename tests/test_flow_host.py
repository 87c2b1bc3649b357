"""Flow trackers on the host: collecting the shift requests of a frame before resolving them gives the candidates the
per-request makers gave, in the same order, and ``make_tracker_by_name(of_device=...)`` reaches the flow makers."""
import numpy as np
import pytest

from sleap_b200.nn import tracking as T
from flow_clip import PerRequestFlowCandidateMaker, PerRequestFlowMaxTracksCandidateMaker, clip_frames, clip_labeled_frames


def _candidate_log(maker_cls, tracker, save, frames, n):
    tr = T.Tracker.make_tracker_by_name(tracker=tracker, similarity="instance", match="greedy", track_window=5, max_tracks=2,
                                        max_tracking=tracker == "flowmaxtracks", save_shifted_instances=save)
    old = tr.candidate_maker
    maker = maker_cls(min_points=old.min_points, save_shifted_instances=save, track_window=5)
    if tracker == "flowmaxtracks":
        maker.max_tracks = 2
    tr.candidate_maker = maker
    log = []
    get = maker.get_candidates

    def logged(*a, **kw):
        out = get(*a, **kw)
        log.append([(x.track.name, x.numpy().copy(), x.shift_score, id(x.source)) for x in out])
        return out

    maker.get_candidates = logged
    frames_out = T.run_tracker(clip_labeled_frames(n), tr, images=lambda t: frames[t])
    return log, [[i.track.name for i in lf.instances] for lf in frames_out]


@pytest.mark.parametrize("tracker,save", [("flow", False), ("flow", True), ("flowmaxtracks", False), ("flowmaxtracks", True)])
def test_collected_requests_match_per_request_candidates(tracker, save):
    pytest.importorskip("cv2")
    n = 24
    frames = clip_frames(n)
    new_cls = T.FlowMaxTracksCandidateMaker if tracker == "flowmaxtracks" else T.FlowCandidateMaker
    old_cls = PerRequestFlowMaxTracksCandidateMaker if tracker == "flowmaxtracks" else PerRequestFlowCandidateMaker
    new_log, new_names = _candidate_log(new_cls, tracker, save, frames, n)
    old_log, old_names = _candidate_log(old_cls, tracker, save, frames, n)
    assert new_names == old_names
    assert len(new_log) == len(old_log) == n
    assert sum(len(c) for c in new_log) > 2 * n                  # the window holds several frames' candidates
    for a, b in zip(new_log, old_log):
        assert [(x[0], x[2]) for x in a] == [(x[0], x[2]) for x in b]
        for x, y in zip(a, b):
            np.testing.assert_array_equal(x[1], y[1])


def test_flowmaxtracks_shifts_a_frame_once_per_track():
    """flowmaxtracks asks for the same reference frame once per track, as the reference does."""
    frames = clip_frames(3)
    tr = T.Tracker.make_tracker_by_name(tracker="flowmaxtracks", track_window=5, max_tracks=2, max_tracking=True)
    seen = []
    resolve = tr.candidate_maker.resolve_requests
    tr.candidate_maker.resolve_requests = lambda reqs, img, t: seen.append([(r[0], r[1], len(r[3])) for r in reqs]) or resolve(reqs, img, t)
    T.run_tracker(clip_labeled_frames(3), tr, images=lambda t: frames[t])
    assert seen[0] == [] and seen[1] == [(0, 0, 2), (0, 0, 2)]
    assert seen[2] == [(0, 0, 2), (1, 1, 2), (0, 0, 2), (1, 1, 2)]


def test_make_tracker_by_name_of_device():
    for name in ("flow", "flowmaxtracks"):
        assert T.Tracker.make_tracker_by_name(tracker=name).candidate_maker.of_device is None
        tr = T.Tracker.make_tracker_by_name(tracker=name, of_device=0, save_shifted_instances=True, track_window=4,
                                            max_tracks=2, max_tracking=name == "flowmaxtracks")
        assert tr.candidate_maker.of_device == 0 and tr.candidate_maker._device_flow is None     # made on first use
        assert tr.candidate_maker.save_shifted_instances and tr.candidate_maker.track_window == 4
    assert T.Tracker.make_tracker_by_name(tracker="flow", max_tracks=2, max_tracking=True, of_device="cuda:0").candidate_maker.of_device == "cuda:0"
    assert isinstance(T.Tracker.make_tracker_by_name(tracker="flow", max_tracks=2, max_tracking=True, of_device=0).candidate_maker,
                      T.FlowMaxTracksCandidateMaker)
    T.Tracker.make_tracker_by_name(tracker="simple", of_device=0)                      # no flow, nothing to run on the GPU
    with pytest.raises(ValueError):
        T.Tracker.make_tracker_by_name(tracker="flow", max_tracks=2, kf_init_frame_count=10, kf_node_indices=[0], of_device=0)


def test_device_flow_without_gpu_raises():
    """A named GPU that is not there is an error, never a silent fall-back to cv2."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from sleap_b200 import _lib
    frames = clip_frames(2)
    tr = T.Tracker.make_tracker_by_name(tracker="flow", of_device=0)
    with pytest.raises(_lib.SleapB200Error):
        T.run_tracker(clip_labeled_frames(2), tr, images=lambda t: frames[t])
