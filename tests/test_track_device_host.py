"""Host side of the device tracker: which configurations may run on the GPU, the parameters handed to
sb_tracker_create, and the stable greedy matcher the device parity tests compare against."""
import numpy as np
import pytest

from sleap_b200.nn import tracking as T
from track_cases import greedy_matching_stable


def test_track_device_rejects_flow_and_kalman():
    for tracker in ("flow", "flowmaxtracks"):
        with pytest.raises(ValueError):
            T.Tracker.make_tracker_by_name(tracker=tracker, track_device=0)
    with pytest.raises(ValueError):
        T.Tracker.make_tracker_by_name(tracker="simple", max_tracks=2, kf_init_frame_count=10, kf_node_indices=[0],
                                       track_device=0)
    with pytest.raises(ValueError):                  # max_tracking turns "flow" into "flowmaxtracks"
        T.Tracker.make_tracker_by_name(tracker="flow", max_tracks=2, max_tracking=True, track_device="cuda:0")


def test_track_device_default_is_host():
    tr = T.Tracker.make_tracker_by_name(tracker="simple")
    assert tr.track_device is None and tr.device_params is None


def test_track_device_params():
    tr = T.Tracker.make_tracker_by_name(tracker="simple", similarity="object_keypoint", match="hungarian", track_window=3,
                                        robust=0.9, max_tracks=4, max_tracking=True, target_instance_count=3,
                                        pre_cull_to_target=True, pre_cull_iou_threshold=0.4, oks_errors=[2.0, 3.0],
                                        oks_score_weighting=True, oks_normalization="union", min_match_points=2,
                                        min_new_track_points=3, track_device="cuda:0")
    p = tr.device_params
    assert tr.track_device == "cuda:0" and tr.has_max_tracking
    assert (p["maker"], p["similarity"], p["match"], p["track_window"]) == (1, 2, 1, 3)
    assert (p["max_tracks"], p["max_tracking"], p["min_match_points"], p["min_new_track_points"]) == (4, 1, 2, 3)
    assert (p["robust"], p["cull_target"], p["cull_use_iou"], p["cull_iou_threshold"]) == (0.9, 3, 1, 0.4)
    assert p["oks_errors"].tolist() == [2.0, 3.0] and (p["oks_score_weighting"], p["oks_normalization"]) == (1, 2)
    p = T.Tracker.make_tracker_by_name(target_instance_count=3, pre_cull_iou_threshold=0.4, track_device=0).device_params
    assert p["cull_target"] == 0                       # pre-cull only with pre_cull_to_target


def test_stable_greedy_ties_and_infinities():
    cost = np.array([[1.0, 1.0, np.inf], [1.0, 0.5, np.inf], [np.inf, np.inf, np.inf]])
    assert greedy_matching_stable(cost) == [(1, 1), (0, 0), (2, 2)]
    assert greedy_matching_stable(np.array([[-0.0, 0.0]])) == [(0, 0)]
