"""The tracking clip fixture (tests/golden/tracks: 1024x1024, two flies) and the old per-request flow candidate
maker the collect-then-resolve makers are checked against."""
import os

import numpy as np

from sleap_b200.nn import tracking as T
from sleap_b200.nn.inference import LabeledFrame, PredictedInstance

CLIP_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tracks")


def clip_frames(n: int) -> np.ndarray:
    """The first ``n`` frames of clip.mp4 as decoded by cv2: (n, 1024, 1024, 3) uint8, three equal channels."""
    import cv2
    cap = cv2.VideoCapture(os.path.join(CLIP_DIR, "clip.mp4"))
    out = []
    for _ in range(n):
        ok, fr = cap.read()
        assert ok, "clip.mp4 could not be decoded"
        out.append(fr)
    cap.release()
    return np.stack(out)


def clip_points():
    """points (frame, instance, node, xy) float32 NaN padded, scores, instances per frame."""
    z = np.load(os.path.join(CLIP_DIR, "clip_predictions.npz"))
    return z["points"], z["scores"], z["n_instances"]


def clip_labeled_frames(n: int) -> list:
    pts, scores, counts = clip_points()
    return [LabeledFrame(0, t, [PredictedInstance.from_numpy(pts[t, j].copy(), np.ones(pts.shape[2], np.float32), float(scores[t, j]))
                                for j in range(counts[t])]) for t in range(n)]


def track_clip(tracker: str, save: bool, n: int, frames: np.ndarray, track_window: int = 5, **kw) -> list:
    tr = T.Tracker.make_tracker_by_name(tracker=tracker, similarity="instance", match="greedy", track_window=track_window, max_tracks=2,
                                        max_tracking=tracker == "flowmaxtracks", save_shifted_instances=save, **kw)
    return T.run_tracker(clip_labeled_frames(n), tr, images=lambda t: frames[t])


class PerRequestFlowCandidateMaker(T.FlowCandidateMaker):
    """The flow maker as it was before requests were collected: one flow_shift_instances call per queue item, saving each
    result as soon as it is made."""

    def get_shifted_instances(self, ref_instances, ref_img, ref_t, img, t):
        shifted = self.flow_shift_instances(ref_instances, ref_img, img, min_shifted_points=self.min_points, scale=self.img_scale,
                                            window_size=self.of_window_size, max_levels=self.of_max_levels)
        if self.save_shifted_instances:
            self.shifted_instances[(ref_t, t)] = (shifted, img, t)
        return shifted

    def get_candidates(self, track_matching_queue, t, img, **kw):
        out = []
        self.prune_shifted_instances(t)
        for item in track_matching_queue:
            ref_t, ref_instances, ref_img = item[0], item[1], item[2]
            if self.save_shifted_instances:
                _, ref_img, ref_instances = self.get_shifted_instances_from_earlier_time(ref_t, ref_img, ref_instances, t)
            if len(ref_instances) > 0:
                out.extend(self.get_shifted_instances(ref_instances, ref_img, ref_t, img, t))
        return out


class PerRequestFlowMaxTracksCandidateMaker(T.FlowMaxTracksCandidateMaker, PerRequestFlowCandidateMaker):
    def get_candidates(self, track_matching_queue_dict, max_tracking, t, img, **kw):
        out, tracks = [], []
        self.prune_shifted_instances(t)
        for track, hist in track_matching_queue_dict.items():
            if not max_tracking or len(tracks) < self.max_tracks:
                tracks.append(track)
                for item in hist:
                    ref_t, ref_img = item[0], item[2]
                    ref_instances = self.get_ref_instances(ref_t, ref_img, track_matching_queue_dict)
                    if self.save_shifted_instances:
                        _, ref_img, ref_instances = self.get_shifted_instances_from_earlier_time(ref_t, ref_img, ref_instances, t)
                    if len(ref_instances) > 0:
                        out.extend(self.get_shifted_instances(ref_instances, ref_img, ref_t, img, t))
        return out
