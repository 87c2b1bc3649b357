"""Identity tracking across frames: the step that follows the inference path (SURVEY 8f row 4).

Restates the default tracker of the reference -- candidates from the last ``track_window`` frames, one similarity
value per (instance, track), greedy or Hungarian assignment, new tracks for the unmatched, optional cap on the
number of tracks -- and the optical-flow variant that first shifts the candidates of earlier frames into the current frame
(Lucas-Kanade through OpenCV, exactly the library call the reference makes, or on a GPU named by ``of_device``:
sleap_b200/nn/flow.py); the Kalman variant is not built:
  sleap/nn/tracker/components.py:33-196   similarity functions (instance, normalized, object keypoint, centroid, IoU)
  sleap/nn/tracker/components.py:198-226  hungarian_matching / greedy_matching, :637-647 first_choice_matching
  sleap/nn/tracker/components.py:229-313  nms_instances / nms_fast, :316-422 cull_instances / cull_frame_instances
  sleap/nn/tracker/components.py:457-634  Match, FrameMatches
  sleap/nn/tracking.py:442-492            SimpleCandidateMaker, SimpleMaxTracksCandidateMaker
  sleap/nn/tracking.py:33-86, 108-360     ShiftedInstance, FlowCandidateMaker (flow_shift_instances, saved shifts, pruning)
  sleap/nn/tracking.py:363-440            FlowMaxTracksCandidateMaker
  sleap/nn/tracking.py:542-844            Tracker.track / spawn / queues, :844-995 make_tracker_by_name
Sequential host code by nature (frame t depends on t-1); instances are anything with ``numpy()`` (n_nodes, 2),
``score`` and a settable ``track`` (``sleap_b200.nn.inference.PredictedInstance``).
"""
import copy
import ctypes
from collections import deque
from typing import Callable, Dict, List, Optional, Sequence, Tuple

import numpy as np
from scipy.optimize import linear_sum_assignment


class Track:
    """sleap/instance.py Track: identity token; compared by identity."""

    def __init__(self, spawned_on: int = 0, name: str = ""):
        self.spawned_on, self.name = spawned_on, name

    def __repr__(self):
        return f"Track(spawned_on={self.spawned_on}, name={self.name!r})"


def _pts(inst) -> np.ndarray:
    return np.asarray(inst.numpy(), np.float64)


def n_visible_points(inst) -> int:
    return int(np.sum(~np.isnan(_pts(inst)).any(axis=1)))


def centroid(inst) -> np.ndarray:
    """Median of the visible points (instance.py:867-875)."""
    return np.nanmedian(_pts(inst), axis=0)


def bounding_box(inst) -> np.ndarray:
    """[y1, x1, y2, x2] over the visible points (instance.py:878-886)."""
    p = _pts(inst)
    if np.isnan(p).all():
        return np.full(4, np.nan)
    return np.concatenate([np.nanmin(p, axis=0)[::-1], np.nanmax(p, axis=0)[::-1]])


# ---- similarities (larger = more alike) -----------------------------------------------------------
def instance_similarity(ref, query) -> float:
    r, q = _pts(ref), _pts(query)
    n_ref = np.sum(~np.isnan(r).any(axis=1))
    d2 = np.sum((q - r) ** 2, axis=1)
    return float(np.nansum(np.exp(-d2)) / n_ref)


def normalized_instance_similarity(ref, query, img_hw: Tuple[int, int]) -> float:
    scale = np.asarray((img_hw[1], img_hw[0]), np.float64)
    r, q = _pts(ref) / scale, _pts(query) / scale
    n_ref = np.sum(~np.isnan(r).any(axis=1))
    return float(np.nansum(np.exp(-np.sum((q - r) ** 2, axis=1))) / n_ref)


def factory_object_keypoint_similarity(keypoint_errors=None, score_weighting: bool = False, normalization_keypoints: str = "all") -> Callable:
    errors = np.asarray(1 if keypoint_errors is None or (hasattr(keypoint_errors, "__len__") and len(keypoint_errors) == 0) else keypoint_errors,
                        np.float64)
    with np.errstate(divide="ignore"):
        precision = 1.0 / (2.0 * errors ** 2)

    def object_keypoint_similarity(ref, query) -> float:
        r, q = _pts(ref), _pts(query)
        ws = 1.0
        if score_weighting:
            ws = np.asarray(getattr(ref, "point_confidences", np.ones(len(r))), np.float64) * \
                np.asarray(getattr(query, "point_confidences", np.ones(len(q))), np.float64)
        vis_r = ~np.isnan(r).any(axis=1)
        if normalization_keypoints == "ref":
            denom = int(vis_r.sum())
        elif normalization_keypoints == "union":
            denom = int(np.logical_and(vis_r, ~np.isnan(q).any(axis=1)).sum())
        else:
            denom = len(r)
        if denom == 0:
            return 0.0
        prec = precision
        if prec.size > 1 and prec.size != len(r):               # fit the per-keypoint errors to the skeleton
            prec = prec[:len(r)] if prec.size > len(r) else np.pad(prec, (0, len(r) - prec.size), "edge")
        d = np.sum((q - r) ** 2, axis=1) * prec
        return float(np.nansum(ws * np.exp(-d)) / denom)

    return object_keypoint_similarity


def centroid_distance(ref, query) -> float:
    return float(-np.linalg.norm(centroid(ref) - centroid(query)))


def compute_iou(a: Sequence[float], b: Sequence[float]) -> float:
    """sleap/nn/utils.py:45-76: inclusive-pixel IoU of [y1, x1, y2, x2] boxes."""
    iy1, ix1, iy2, ix2 = max(a[0], b[0]), max(a[1], b[1]), min(a[2], b[2]), min(a[3], b[3])
    inter = max(ix2 - ix1 + 1, 0) * max(iy2 - iy1 + 1, 0)
    area = lambda t: (t[3] - t[1] + 1) * (t[2] - t[0] + 1)
    return float(inter / (area(a) + area(b) - inter))


def instance_iou(ref, query) -> float:
    return compute_iou(bounding_box(ref), bounding_box(query))


# ---- assignment -----------------------------------------------------------------------------------
def hungarian_matching(cost: np.ndarray) -> List[Tuple[int, int]]:
    rows, cols = linear_sum_assignment(cost)
    return list(zip(rows.tolist(), cols.tolist()))


def greedy_matching(cost: np.ndarray) -> List[Tuple[int, int]]:
    """Cheapest remaining (row, column) pair first; ties in ``argsort`` order of the flattened matrix."""
    order = np.argsort(cost, axis=None)
    used_r, used_c, out = set(), set(), []
    for flat in order.tolist():
        r, c = divmod(flat, cost.shape[1])
        if r in used_r or c in used_c:
            continue
        used_r.add(r); used_c.add(c)
        out.append((r, c))
    return out


def first_choice_matching(cost: np.ndarray) -> List[Tuple[int, int]]:
    return list(zip(range(len(cost)), cost.argmin(axis=1).tolist()))


# ---- suppression of duplicate detections ----------------------------------------------------------
def nms_fast(boxes: np.ndarray, scores: np.ndarray, iou_threshold: float, target_count: Optional[int] = None) -> List[int]:
    """Score-ordered box suppression (overlap measured against the *other* box's area, +1 pixel convention), then, when
    fewer than ``target_count`` survive, suppressed boxes are handed back best score first.  The hand-back count is
    ``min(n_suppressed, n_kept - target_count)`` used as a slice end, exactly as the reference computes it
    (components.py:306-309; negative ends drop from the tail, which its tests rely on)."""
    boxes = np.asarray(boxes)
    scores = np.asarray(scores, np.float64)
    if len(boxes) == 0:
        return []
    if target_count and len(boxes) < target_count:
        return list(range(len(boxes)))
    boxes = boxes.astype(np.float64)
    x1, y1, x2, y2 = boxes.T
    area = (x2 - x1 + 1) * (y2 - y1 + 1)
    alive = list(np.argsort(scores))
    kept, dropped = [], []
    while alive:
        top = alive.pop()                                   # best remaining score
        kept.append(int(top))
        rest = np.asarray(alive, np.int64)
        if len(rest) == 0:
            break
        w = np.maximum(0, np.minimum(x2[top], x2[rest]) - np.maximum(x1[top], x1[rest]) + 1)
        h = np.maximum(0, np.minimum(y2[top], y2[rest]) - np.maximum(y1[top], y1[rest]) + 1)
        over = (w * h) / area[rest] > iou_threshold
        dropped.extend(int(i) for i in rest[over])
        alive = [int(i) for i in rest[~over]]
    if target_count and dropped and len(kept) < target_count:
        dropped.sort(key=lambda i: -scores[i])
        kept.extend(dropped[:min(len(dropped), len(kept) - target_count)])
    return kept


def nms_instances(instances: list, iou_threshold: float, target_count: Optional[int] = None):
    boxes = np.asarray([bounding_box(i) for i in instances])
    scores = np.asarray([i.score for i in instances])
    picks = set(nms_fast(boxes, scores, iou_threshold, target_count))
    return [x for i, x in enumerate(instances) if i in picks], [x for i, x in enumerate(instances) if i not in picks]


def cull_frame_instances(instances: list, instance_count: int, iou_threshold: Optional[float] = None) -> list:
    """At most ``instance_count`` instances in this frame: overlapping duplicates go first (when a threshold is given),
    then the lowest scores.  Modifies and returns the list (components.py:365-422)."""
    if not instances or len(instances) <= instance_count:
        return instances
    keep = list(instances)
    if iou_threshold:
        keep, extra = nms_instances(keep, iou_threshold, target_count=instance_count)
        for x in extra:
            instances.remove(x)
    if len(keep) > instance_count:
        for x in sorted(keep, key=lambda i: i.score)[:-instance_count]:
            instances.remove(x)
    return instances


def cull_instances(frames: list, instance_count: int, iou_threshold: Optional[float] = None):
    for lf in sorted(frames, key=lambda f: f.frame_idx):
        cull_frame_instances(lf.instances, instance_count, iou_threshold)


def connect_single_track_breaks(frames: list, instance_count: int) -> list:
    """sleap/nn/tracker/components.py:417-466: whenever exactly one track disappears and exactly one new track appears
    between a frame and the last frame that had ``instance_count`` tracks, the new track is merged into the lost one
    (for the rest of the video).  Modifies the frames in place."""
    if not frames:
        return frames
    fix_track_map = {}
    last_good = {inst.track for inst in frames[0].instances}
    for lf in frames:
        frame_tracks = {inst.track for inst in lf.instances}
        if frame_tracks & set(fix_track_map):
            for inst in lf.instances:
                if inst.track in fix_track_map and fix_track_map[inst.track] not in frame_tracks:
                    inst.track = fix_track_map[inst.track]
                    frame_tracks = {i.track for i in lf.instances}
        extra, missing = frame_tracks - last_good, last_good - frame_tracks
        if len(extra) == 1 and len(missing) == 1:
            for inst in lf.instances:
                if inst.track in extra:
                    old, new = inst.track, missing.pop()
                    fix_track_map[old] = new
                    inst.track = new
                    break
        elif len(frame_tracks) == instance_count:
            last_good = frame_tracks
    return frames


class TrackCleaner:
    """tracking.py:1513-1539: cull each frame to ``instance_count`` instances, then join single track breaks."""

    def __init__(self, instance_count: int, iou_threshold: Optional[float] = None):
        self.instance_count, self.iou_threshold = instance_count, iou_threshold

    def run(self, frames: list):
        cull_instances(frames, self.instance_count, self.iou_threshold)
        connect_single_track_breaks(frames, self.instance_count)


# ---- matches of one frame ---------------------------------------------------------------------------
class Match:
    def __init__(self, track, instance, score=None, is_first_choice=False):
        self.track, self.instance, self.score, self.is_first_choice = track, instance, score, is_first_choice


class FrameMatches:
    """Matches of one frame + whether each instance got the track it would have picked alone (components.py:470-634)."""

    def __init__(self, matches: List[Match], cost_matrix: np.ndarray, unmatched_instances: list):
        self.matches, self.cost_matrix, self.unmatched_instances = matches, cost_matrix, unmatched_instances

    @property
    def has_only_first_choice_matches(self) -> bool:
        return all(m.is_first_choice for m in self.matches)

    @classmethod
    def from_cost_matrix(cls, cost_matrix: np.ndarray, instances: list, tracks: list, matching_function: Callable):
        matches, taken = [], set()
        if instances and tracks:
            first = cost_matrix.argmin(axis=1)
            for i, j in matching_function(cost_matrix):
                taken.add(i)
                matches.append(Match(tracks[j], instances[i], -cost_matrix[i, j], bool(first[i] == j)))
        return cls(matches, cost_matrix, [x for i, x in enumerate(instances) if i not in taken])

    @classmethod
    def from_candidate_instances(cls, untracked_instances: list, candidate_instances: list, similarity_function: Callable,
                                 matching_function: Callable, robust_best_instance: float = 1.0):
        cost, tracks = np.ndarray((0,)), []
        if candidate_instances:
            by_track: Dict[object, list] = {}
            for c in candidate_instances:                       # insertion order = order of first appearance
                by_track.setdefault(c.track, []).append(c)
            tracks = list(by_track)
            sim = np.full((len(untracked_instances), len(tracks)), np.nan)
            for i, u in enumerate(untracked_instances):
                for j, tr in enumerate(tracks):
                    s = [similarity_function(u, c) for c in by_track[tr]]
                    sim[i, j] = np.quantile(s, robust_best_instance) if 0 < robust_best_instance < 1 else np.max(s)
            cost = -sim
            cost[np.isnan(cost)] = np.inf
        return cls.from_cost_matrix(cost, untracked_instances, tracks, matching_function)


# ---- candidate pools --------------------------------------------------------------------------------
class SimpleCandidateMaker:
    """Every instance of the last ``track_window`` frames with enough visible points."""

    uses_image = False

    def __init__(self, min_points: int = 0):
        self.min_points = min_points

    def get_candidates(self, track_matching_queue, **kw) -> list:
        return [x for item in track_matching_queue for x in item[1] if n_visible_points(x) >= self.min_points]


class SimpleMaxTracksCandidateMaker(SimpleCandidateMaker):
    """Per-track history; with ``max_tracking`` only the first ``max_tracks`` tracks are matchable."""

    def __init__(self, min_points: int = 0, max_tracks: Optional[int] = None):
        super().__init__(min_points)
        self.max_tracks = max_tracks

    def get_candidates(self, track_matching_queue_dict, max_tracking: bool, **kw) -> list:
        out, n = [], 0
        for _, hist in track_matching_queue_dict.items():
            if not max_tracking or n < self.max_tracks:
                n += 1
                out.extend(item[1] for item in hist if n_visible_points(item[1]) >= self.min_points)
        return out


class ShiftedInstance:
    """A reference instance moved into the current frame by optical flow (tracking.py:33-86): same track, new points
    (NaN where the flow lost the point), ``shift_score`` = -mean tracking error."""

    def __init__(self, points_array: np.ndarray, track, shift_score: float = 0.0, source=None):
        self.points_array = np.asarray(points_array, np.float64)
        self.track, self.shift_score, self.source = track, shift_score, source
        self.score = getattr(source, "score", float("nan"))

    def numpy(self):
        return self.points_array

    @classmethod
    def from_instance(cls, ref_instance, new_points_array=None, shift_score: float = 0.0):
        pts = _pts(ref_instance) if new_points_array is None else new_points_array
        return cls(pts, getattr(ref_instance, "track", None), shift_score, ref_instance)


def _ensure_u8(img: np.ndarray) -> np.ndarray:
    """normalization.ensure_int (sleap/nn/data/normalization.py:52-66): float images in [0, 1] -> uint8."""
    img = np.asarray(img)
    if img.dtype == np.uint8:
        return img
    if np.issubdtype(img.dtype, np.floating) and img.size and float(np.nanmax(img)) <= 1.0:
        img = img * 255.0
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def shifted_instances_from_flow(ref_instances: list, shifted: np.ndarray, status: np.ndarray, errs: np.ndarray,
                                min_shifted_points: int = 0) -> list:
    """tracking.py:340-360: the flow result of the concatenated points of ``ref_instances`` -> one ShiftedInstance per
    instance that kept more than ``min_shifted_points`` points (lost points NaN, ``shift_score`` = -mean err of the
    found points)."""
    sections = np.cumsum([len(_pts(x)) for x in ref_instances])[:-1]
    out = []
    for ref, pts, found, err in zip(ref_instances, np.split(shifted, sections, axis=0), np.split(status, sections, axis=0),
                                    np.split(errs, sections, axis=0)):
        if found.sum() > min_shifted_points:
            found = found.reshape(-1).astype(bool)
            pts = pts.astype(np.float64)
            pts[~found] = np.nan
            out.append(ShiftedInstance.from_instance(ref, new_points_array=pts, shift_score=-float(np.mean(err.reshape(-1)[found]))))
    return out


class FlowCandidateMaker:
    """Candidates = the instances of the last ``track_window`` frames, each flow-shifted into the current frame
    (tracking.py:108-360).  ``save_shifted_instances`` chains the shifts frame to frame instead of always starting from
    the original frame (:139-160).

    ``of_device``: None shifts with ``cv2.calcOpticalFlowPyrLK``, one call per reference frame, as the reference does.
    A GPU index (or "cuda:N") shifts every reference frame's points with one ``DeviceFlow.shift`` call on that GPU
    (sleap_b200/nn/flow.py), building each frame's pyramid once."""

    uses_image = True

    def __init__(self, min_points: int = 0, img_scale: float = 1.0, of_window_size: int = 21, of_max_levels: int = 3,
                 save_shifted_instances: bool = False, track_window: int = 5, of_device=None):
        self.min_points, self.img_scale = min_points, img_scale
        self.of_window_size, self.of_max_levels = of_window_size, of_max_levels
        self.save_shifted_instances, self.track_window = save_shifted_instances, track_window
        self.of_device = of_device
        self._device_flow = None
        self.shifted_instances: Dict[Tuple[int, int], tuple] = {}        # (ref_t, t) -> (instances, img, t)

    def get_shifted_instances_from_earlier_time(self, ref_t: int, ref_img, ref_instances: list, t: int):
        """-> (frame index of the image, image, instances) to shift from."""
        for ti in reversed(range(ref_t, t)):
            if (ref_t, ti) in self.shifted_instances:
                insts, img, img_t = self.shifted_instances[(ref_t, ti)]
                if len(insts) > 0:
                    return img_t, img, insts
        return ref_t, ref_img, ref_instances

    def prune_shifted_instances(self, t: int):
        if not self.save_shifted_instances:
            return
        for k in list(self.shifted_instances):
            if t - k[0] > self.track_window:
                del self.shifted_instances[k]

    def add_request(self, requests: list, ref_t: int, ref_img, ref_instances: list, t: int):
        """Queue the shift of ``ref_instances`` (frame ``ref_t``) into frame ``t``, from the latest saved shift when
        ``save_shifted_instances`` is on.  Requests are (ref_t, frame index of the image, image, instances)."""
        img_t = ref_t
        if self.save_shifted_instances:
            img_t, ref_img, ref_instances = self.get_shifted_instances_from_earlier_time(ref_t, ref_img, ref_instances, t)
        if len(ref_instances) > 0:
            requests.append((ref_t, img_t, ref_img, ref_instances))

    def get_candidates(self, track_matching_queue, t: int, img, **kw) -> list:
        if img is None:
            raise ValueError("the flow tracker needs the frame image: Tracker.track(instances, img=frame, ...)")
        self.prune_shifted_instances(t)
        requests: list = []
        for item in track_matching_queue:
            self.add_request(requests, item[0], item[2], item[1], t)
        return self.resolve_requests(requests, img, t)

    def resolve_requests(self, requests: list, img, t: int) -> list:
        """Shift every request into frame ``t`` and return the candidates in request order."""
        if not requests:
            return []
        if self.of_device is None:
            shifted = [self.flow_shift_instances(insts, ref_img, img, min_shifted_points=self.min_points, scale=self.img_scale,
                                                 window_size=self.of_window_size, max_levels=self.of_max_levels)
                       for _, _, ref_img, insts in requests]
        else:
            shifted = self.device_shift(requests, img, t)
        out = []
        for (ref_t, _, _, _), insts in zip(requests, shifted):
            if self.save_shifted_instances:
                self.shifted_instances[(ref_t, t)] = (insts, img, t)
            out.extend(insts)
        return out

    def device_flow(self):
        """The DeviceFlow of ``of_device``, made on first use (``make_tracker_by_name`` sets the flow options after
        construction)."""
        if self._device_flow is None:
            from sleap_b200.nn.flow import DeviceFlow
            dev = int(str(self.of_device).split(":")[-1])
            self._device_flow = DeviceFlow(dev, self.of_window_size, self.of_max_levels, self.img_scale, self.track_window + 2)
        return self._device_flow

    def device_shift(self, requests: list, img, t: int) -> list:
        """All requests in one ``DeviceFlow.shift`` call; the frames they read are uploaded unless already held."""
        flow = self.device_flow()
        frames: Dict[int, object] = {}
        for _, img_t, ref_img, _ in requests:
            frames.setdefault(img_t, ref_img)
        flow.reserve(len(frames) + 1)
        flow.add_frame(t, _ensure_u8(img))          # gray conversion and resize run on the device
        for img_t, ref_img in frames.items():
            flow.add_frame(img_t, _ensure_u8(ref_img), replace=False)
        pts = [np.concatenate([_pts(x) for x in insts], axis=0).astype("float32") * self.img_scale for _, _, _, insts in requests]
        ref_t = np.concatenate([np.full(len(p), img_t, np.int64) for p, (_, img_t, _, _) in zip(pts, requests)])
        shifted, status, errs = flow.shift(t, ref_t, np.concatenate(pts, axis=0))
        shifted = shifted / self.img_scale
        sections = np.cumsum([len(p) for p in pts])[:-1]
        return [shifted_instances_from_flow(insts, s, st, e, self.min_points)
                for (_, _, _, insts), s, st, e in zip(requests, np.split(shifted, sections), np.split(status, sections),
                                                      np.split(errs, sections))]

    @staticmethod
    def flow_shift_instances(ref_instances: list, ref_img, new_img, min_shifted_points: int = 0, scale: float = 1.0,
                             window_size: int = 21, max_levels: int = 3) -> list:
        """tracking.py:262-360: pyramidal Lucas-Kanade (cv2.calcOpticalFlowPyrLK, 30 iterations / eps 0.01) of every
        reference point; instances keep the points the flow found (> min_shifted_points of them)."""
        import cv2
        ref_img, new_img = _ensure_u8(ref_img), _ensure_u8(new_img)
        if ref_img.ndim > 2 and ref_img.shape[-1] == 1:
            ref_img, new_img = ref_img[..., 0], new_img[..., 0]
        if ref_img.ndim > 2 and ref_img.shape[-1] == 3:
            ref_img, new_img = cv2.cvtColor(ref_img, cv2.COLOR_BGR2GRAY), cv2.cvtColor(new_img, cv2.COLOR_BGR2GRAY)
        if scale != 1:
            ref_img = cv2.resize(ref_img, None, None, scale, scale)
            new_img = cv2.resize(new_img, None, None, scale, scale)
        ref_pts = [_pts(x) for x in ref_instances]
        shifted, status, errs = cv2.calcOpticalFlowPyrLK(
            np.ascontiguousarray(ref_img), np.ascontiguousarray(new_img), (np.concatenate(ref_pts, axis=0)).astype("float32") * scale, None,
            winSize=(window_size, window_size), maxLevel=max_levels,
            criteria=(cv2.TERM_CRITERIA_EPS | cv2.TERM_CRITERIA_COUNT, 30, 0.01))
        return shifted_instances_from_flow(ref_instances, shifted / scale, status, errs, min_shifted_points)


class FlowMaxTracksCandidateMaker(FlowCandidateMaker):
    """Flow candidates from the per-track history, at most ``max_tracks`` tracks (tracking.py:363-440)."""

    def __init__(self, max_tracks: Optional[int] = None, **kw):
        super().__init__(**kw)
        self.max_tracks = max_tracks

    @staticmethod
    def get_ref_instances(ref_t: int, ref_img, track_matching_queue_dict) -> list:
        out = []
        for _, hist in track_matching_queue_dict.items():
            out += [item[1] for item in hist if item[0] == ref_t and np.all(item[2] == ref_img)]
        return out

    def get_candidates(self, track_matching_queue_dict, max_tracking: bool, t: int, img, **kw) -> list:
        if img is None:
            raise ValueError("the flow tracker needs the frame image: Tracker.track(instances, img=frame, ...)")
        requests: list = []
        tracks = []
        self.prune_shifted_instances(t)
        for track, hist in track_matching_queue_dict.items():
            if not max_tracking or len(tracks) < self.max_tracks:
                tracks.append(track)
                for item in hist:                               # one request per track and frame, duplicates included
                    ref_t, ref_img = item[0], item[2]
                    self.add_request(requests, ref_t, ref_img, self.get_ref_instances(ref_t, ref_img, track_matching_queue_dict), t)
        return self.resolve_requests(requests, img, t)


class DeviceTracker:
    """The queues and spawned-track counter of one tracker, resident on a GPU (sb_tracker_create), and its per-call
    step (sb_track_instances: k_track).  ``params``: the fields of sb_tracker_params.  It has a handle of its own, so
    that a predictor's consumer thread can track while the predictor's handle runs the next batch."""

    def __init__(self, device, params: dict, handle=None):
        from sleap_b200 import _lib
        self._lib = _lib
        self.handle = handle if handle is not None else _lib.Handle(int(str(device).split(":")[-1]))
        self.params = dict(params)
        errs = self.params.pop("oks_errors", None)
        self._errs = None if errs is None or len(errs) == 0 else np.ascontiguousarray(errs, np.float64)
        p = _lib.TrackerParams(**self.params, oks_errors=None if self._errs is None else _lib.ptr(self._errs),
                               n_oks_errors=0 if self._errs is None else len(self._errs))
        out = ctypes.c_int()
        self.handle.call("sb_tracker_create", ctypes.byref(p), ctypes.byref(out))
        self.id = out.value
        self.n_nodes, self.max_instances = int(params["n_nodes"]), int(params["max_instances"])

    def track(self, instance_lists: list, ts: Sequence[Optional[int]], img_hws: Sequence[Tuple[int, int]]) -> list:
        """-> (per frame done: (input indices, track ids, tracking scores, matched flags, frame index), error).  The
        error (None when every frame was tracked) is the one the host tracker raises at the first frame not tracked:
        ValueError for a matrix SciPy's Hungarian matcher rejects, SleapB200Error for a capacity overflow."""
        B, C = len(instance_lists), self.n_nodes
        I = max([1] + [len(x) for x in instance_lists])
        pts = np.full((B, I, C, 2), np.nan)
        conf = np.ones((B, I, C))
        scores = np.zeros((B, I))
        for b, lst in enumerate(instance_lists):
            for i, x in enumerate(lst):
                p = _pts(x)
                if p.shape != (C, 2):
                    raise ValueError(f"instance with {p.shape[0]} nodes given to a tracker of {C}")
                pts[b, i] = p
                conf[b, i] = np.asarray(getattr(x, "point_confidences", np.ones(C)), np.float64)
                scores[b, i] = x.score
        counts = np.asarray([len(x) for x in instance_lists], np.int32)
        hw = np.ascontiguousarray(np.asarray(img_hws, np.float64).reshape(B, 2))
        t = np.asarray([-1 if x is None else int(x) for x in ts], np.int64)
        o_idx, o_tid = np.zeros((B, I), np.int32), np.zeros((B, I), np.int32)
        o_score, o_m = np.zeros((B, I)), np.zeros((B, I), np.int32)
        o_n, o_t = np.zeros(B, np.int32), np.zeros(B, np.int64)
        n_done, flag = ctypes.c_int32(), ctypes.c_int32()
        P = self._lib.ptr
        rc = self._lib.lib().sb_track_instances(self.handle.h, self.id, B, I, P(pts), P(conf), P(scores), P(counts), P(hw),
                                                P(t), P(o_idx), P(o_tid), P(o_score), P(o_m), P(o_n), P(o_t),
                                                ctypes.byref(n_done), ctypes.byref(flag))
        err = None
        if rc != 0:
            err = self._lib.SleapB200Error(f"sb_track_instances failed ({rc}): {self._lib.lib().sb_last_error(self.handle.h).decode()}")
        elif flag.value != 0:
            err = ValueError("cost matrix is infeasible")
        return [(o_idx[b, :o_n[b]].tolist(), o_tid[b, :o_n[b]], o_score[b, :o_n[b]], o_m[b, :o_n[b]], o_t[b])
                for b in range(n_done.value)], err


DEVICE_MAKERS = dict(simple=0, simplemaxtracks=1)
DEVICE_SIMILARITIES = dict(instance=0, normalized_instance=1, object_keypoint=2, centroid=3, iou=4)
DEVICE_MATCHERS = dict(greedy=0, hungarian=1)
DEVICE_OKS_NORMALIZATIONS = dict(all=0, ref=1, union=2)

SIMILARITIES = dict(instance=instance_similarity, centroid=centroid_distance, iou=instance_iou,
                    normalized_instance=normalized_instance_similarity, object_keypoint=factory_object_keypoint_similarity)
MATCHERS = dict(hungarian=hungarian_matching, greedy=greedy_matching)
CANDIDATE_MAKERS = dict(simple=SimpleCandidateMaker, simplemaxtracks=SimpleMaxTracksCandidateMaker, flow=FlowCandidateMaker,
                        flowmaxtracks=FlowMaxTracksCandidateMaker)


class Tracker:
    """One ``track(instances)`` call per frame, in order (tracking.py:542-844)."""

    def __init__(self, track_window: int = 5, similarity_function: Optional[Callable] = instance_similarity,
                 matching_function: Callable = greedy_matching, candidate_maker=None, max_tracks: Optional[int] = None,
                 max_tracking: bool = False, min_new_track_points: int = 0, robust_best_instance: float = 1.0,
                 pre_cull_function: Optional[Callable] = None, target_instance_count: int = 0):
        self.track_window = track_window
        self.similarity_function, self.matching_function = similarity_function, matching_function
        self.candidate_maker = candidate_maker
        self.max_tracks, self.max_tracking = max_tracks, max_tracking
        self.min_new_track_points, self.robust_best_instance = min_new_track_points, robust_best_instance
        self.pre_cull_function, self.target_instance_count = pre_cull_function, target_instance_count
        self.track_matching_queue: deque = deque(maxlen=track_window)        # (t, [instances])
        self.track_matching_queue_dict: Dict[Track, deque] = {}               # track -> deque of (t, instance)
        self.spawned_tracks: List[Track] = []
        self.last_matches: Optional[FrameMatches] = None

    @property
    def is_valid(self):
        return self.similarity_function is not None

    @property
    def has_max_tracking(self) -> bool:
        return isinstance(self.candidate_maker, (SimpleMaxTracksCandidateMaker, FlowMaxTracksCandidateMaker))

    @property
    def uses_image(self) -> bool:
        return bool(getattr(self.candidate_maker, "uses_image", False))

    @property
    def unique_tracks_in_queue(self) -> List[Track]:
        if self.has_max_tracking:
            return list(self.track_matching_queue_dict)
        return list({x.track for item in self.track_matching_queue for x in item[1]})

    def reset_candidates(self):
        self.track_matching_queue = deque(maxlen=self.track_window)
        for tr in self.track_matching_queue_dict:
            self.track_matching_queue_dict[tr] = deque(maxlen=self.track_window)

    def _next_t(self) -> int:
        if self.has_max_tracking:
            if not self.track_matching_queue_dict:
                return 0
            longest = max(self.track_matching_queue_dict, key=lambda tr: len(self.track_matching_queue_dict[tr]))
            return self.track_matching_queue_dict[longest][-1][0] + 1
        return self.track_matching_queue[-1][0] + 1 if self.track_matching_queue else 0

    def track(self, untracked_instances: list, img_hw: Tuple[int, int] = (1, 1), img=None, t: Optional[int] = None) -> list:
        if self.candidate_maker is None:
            return untracked_instances
        if self.track_device is not None:
            out, err = self.track_frames([list(untracked_instances)], [t], [img_hw])
            if err is not None:
                raise err
            return out[0]
        sim = self.similarity_function
        if sim is normalized_instance_similarity:
            sim = lambda a, b: normalized_instance_similarity(a, b, img_hw=img_hw)
        if t is None:
            t = self._next_t()
        tracked: list = []
        if untracked_instances:
            if self.pre_cull_function:
                self.pre_cull_function(untracked_instances)
            if self.has_max_tracking:
                cands = self.candidate_maker.get_candidates(track_matching_queue_dict=self.track_matching_queue_dict,
                                                            max_tracking=self.max_tracking, t=t, img=img)
            else:
                cands = self.candidate_maker.get_candidates(track_matching_queue=self.track_matching_queue, t=t, img=img)
            fm = FrameMatches.from_candidate_instances(untracked_instances, cands, sim, self.matching_function, self.robust_best_instance)
            self.last_matches = fm
            for m in fm.matches:                                # matched: inherit the track
                x = copy.copy(m.instance)
                x.track, x.tracking_score = m.track, m.score
                tracked.append(x)
            for inst in fm.unmatched_instances:                 # unmatched: new tracks, unless the cap is reached
                if n_visible_points(inst) < self.min_new_track_points:
                    continue
                if self.has_max_tracking and self.max_tracking and len(self.track_matching_queue_dict) >= self.max_tracks:
                    break
                tr = Track(spawned_on=t, name=f"track_{len(self.spawned_tracks)}")
                self.spawned_tracks.append(tr)
                x = copy.copy(inst)
                x.track = tr
                tracked.append(x)
        keep_img = img if self.uses_image else None              # only the flow makers look at earlier frames (:780-800)
        if self.has_max_tracking:
            for x in tracked:
                if x.track in self.track_matching_queue_dict:
                    self.track_matching_queue_dict[x.track].append((t, x, keep_img))
                elif not self.max_tracking or len(self.track_matching_queue_dict) < self.max_tracks:
                    self.track_matching_queue_dict[x.track] = deque([(t, x, keep_img)], maxlen=self.track_window)
        else:
            self.track_matching_queue.append((t, tracked, keep_img))
        return tracked

    cleaner: Optional["TrackCleaner"] = None          # deprecated --clean_instance_count path (:924-927)
    post_connect_single_breaks: bool = False
    # GPU (index or "cuda:N") whose k_track kernel runs the whole per-frame step (make_tracker_by_name(track_device=...))
    track_device = None
    device_params: Optional[dict] = None               # the sb_tracker_params of that tracker, set with track_device
    device_max_instances = 128                         # per-frame capacity of the device tracker (at most 128)
    device_track_table = 4096                          # max-tracks queue table without a max_tracks cap

    def _device_tracker(self, n_nodes: int, handle=None, max_instances: Optional[int] = None) -> "DeviceTracker":
        """The device state of this tracker, made on first use: on its own handle of ``track_device``, or on ``handle``
        (a predictor's, so that the tracker can run inside its bottom-up step)."""
        dev = getattr(self, "_device", None)
        if dev is None:
            table = self.device_track_table
            if self.has_max_tracking and self.max_tracking:
                table = int(self.max_tracks)
            dev = self._device = DeviceTracker(self.track_device, dict(
                self.device_params, n_nodes=n_nodes, max_instances=max(self.device_max_instances, max_instances or 0),
                track_table=table), handle=handle)
            pending, self._pending = getattr(self, "_pending", []), []
            if pending:                                # empty frames seen before the node count was known
                dev.track([[] for _ in pending], [t for t, _ in pending], [hw for _, hw in pending])
        elif handle is not None and dev.handle is not handle:
            raise ValueError("this tracker's device state lives on another handle than the predictor's; make a new tracker")
        return dev

    def apply_device_tracks(self, instances: list, frame_idx: int, order, track_ids, scores, matched=None) -> list:
        """The tracked list of one frame from the device's output: copies of ``instances[order[k]]`` with the ``Track``
        of ``track_ids[k]`` (made in spawn order, ``spawned_on`` = the frame that spawned it) and, when matched, the
        tracking score."""
        tracked = []
        for k in range(len(order)):
            tid = int(track_ids[k])
            while tid >= len(self.spawned_tracks):
                self.spawned_tracks.append(Track(spawned_on=int(frame_idx), name=f"track_{len(self.spawned_tracks)}"))
            x = copy.copy(instances[int(order[k])])
            x.track = self.spawned_tracks[tid]
            if matched is None or matched[k]:
                x.tracking_score = float(scores[k])
            tracked.append(x)
        return tracked

    def track_frames(self, instance_lists: list, ts: Sequence[Optional[int]], img_hws: Sequence[Tuple[int, int]]):
        """``track`` of several frames in one ``sb_track_instances`` call on ``track_device`` -> (the tracked list of
        every frame tracked, in ``track``'s order, error).  As on the host, the frames before an error are tracked
        and the error (None if there is none) is for the caller to raise."""
        n_nodes = next((len(_pts(x)) for lst in instance_lists for x in lst), None)
        if getattr(self, "_device", None) is None and n_nodes is None:
            self._pending = getattr(self, "_pending", []) + [(t, hw) for t, hw in zip(ts, img_hws)]
            return [[] for _ in instance_lists], None
        res, err = self._device_tracker(n_nodes).track(instance_lists, ts, img_hws)
        return [self.apply_device_tracks(lst, t, idx, tids, scores, matched)
                for lst, (idx, tids, scores, matched, t) in zip(instance_lists, res)], err

    def final_pass(self, frames: list):
        """:816-835: post-processing after the last frame -- the (deprecated) cleaner, or the single-break joining."""
        if self.cleaner is not None:
            self.cleaner.run(frames)
        elif (self.target_instance_count or self.max_tracks) and self.post_connect_single_breaks:
            if not self.target_instance_count:
                self.target_instance_count = self.max_tracks
            connect_single_track_breaks(frames, self.target_instance_count)

    def get_name(self) -> str:
        return f"{type(self.candidate_maker).__name__}.{getattr(self.similarity_function, '__name__', 'none')}." \
               f"{getattr(self.matching_function, '__name__', 'none')}"

    @classmethod
    def make_tracker_by_name(cls, tracker: str = "simple", similarity: str = "instance", match: str = "greedy", track_window: int = 5,
                             robust: float = 1.0, min_new_track_points: int = 0, min_match_points: int = 0,
                             target_instance_count: int = 0, pre_cull_to_target: bool = False,
                             pre_cull_iou_threshold: Optional[float] = None, max_tracks: Optional[int] = None,
                             max_tracking: bool = False, oks_errors=None, oks_score_weighting: bool = False,
                             oks_normalization: str = "all", img_scale: float = 1.0, of_window_size: int = 21,
                             of_max_levels: int = 3, save_shifted_instances: bool = False, kf_init_frame_count: int = 0,
                             kf_node_indices: Optional[list] = None, post_connect_single_breaks: bool = False,
                             clean_instance_count: int = 0, clean_iou_threshold: Optional[float] = None, of_device=None,
                             track_device=None, **kwargs) -> "Tracker":
        """``of_device``: GPU (index or "cuda:N") that runs the flow shift of the flow trackers; None (default) runs
        it with cv2 on the CPU, as the reference does.

        ``track_device``: GPU (index or "cuda:N") that runs the whole per-frame step of the simple and
        simple-max-tracks trackers (pre-cull, candidates, similarities, matching, new tracks, queues) in one kernel,
        the queues staying on the GPU; ``final_pass`` stays on the host.  Ties between equal greedy costs go to the
        lower flat index (``np.argsort(kind="stable")``), and the pre-cull orders equal scores by ascending instance
        index (its suppression keeps the higher index of two equal scores first, its score cut drops the lower index
        first), where the host's default sorts leave these orders implementation-defined.  None (default): the host tracker."""
        max_tracking = max_tracking if max_tracks else False
        if max_tracking and tracker in ("simple", "flow"):          # :882-884
            tracker += "maxtracks"
        if track_device is not None:
            if tracker in ("flow", "flowmaxtracks"):
                raise ValueError("track_device runs the simple and simplemaxtracks trackers; the flow trackers take of_device")
            if kf_init_frame_count:
                raise ValueError("track_device does not run the Kalman tracker")
        if tracker.lower() == "none":
            return cls(track_window=track_window, similarity_function=None, matching_function=None, candidate_maker=None)
        if tracker not in CANDIDATE_MAKERS:
            raise ValueError(f"{tracker} is not a valid tracker.")
        if similarity not in SIMILARITIES:
            raise ValueError(f"{similarity} is not a valid tracker similarity function.")
        if match not in MATCHERS:
            raise ValueError(f"{match} is not a valid tracker matching function.")
        maker = CANDIDATE_MAKERS[tracker](min_points=min_match_points)
        if tracker in ("flow", "flowmaxtracks"):                   # :913-918
            maker.img_scale, maker.of_window_size, maker.of_max_levels = img_scale, of_window_size, of_max_levels
            maker.save_shifted_instances, maker.track_window = save_shifted_instances, track_window
            maker.of_device = of_device
        if tracker in ("simplemaxtracks", "flowmaxtracks"):
            maker.max_tracks = max_tracks
        sim = SIMILARITIES[similarity]
        if similarity == "object_keypoint":
            sim = factory_object_keypoint_similarity(oks_errors, oks_score_weighting, oks_normalization)
        pre_cull = None
        if target_instance_count and pre_cull_to_target:
            pre_cull = lambda insts: cull_frame_instances(insts, target_instance_count, pre_cull_iou_threshold)
        tracker_obj = cls(track_window=track_window, similarity_function=sim, matching_function=MATCHERS[match], candidate_maker=maker,
                          max_tracks=max_tracks, max_tracking=max_tracking, min_new_track_points=min_new_track_points,
                          robust_best_instance=robust, pre_cull_function=pre_cull, target_instance_count=target_instance_count)
        tracker_obj.post_connect_single_breaks = bool(post_connect_single_breaks)
        if track_device is not None:
            tracker_obj.track_device = track_device
            tracker_obj.device_params = dict(
                maker=DEVICE_MAKERS[tracker], similarity=DEVICE_SIMILARITIES[similarity], match=DEVICE_MATCHERS[match],
                track_window=int(track_window), max_tracks=int(max_tracks or 0), max_tracking=int(bool(max_tracking)),
                min_match_points=int(min_match_points), min_new_track_points=int(min_new_track_points), robust=float(robust),
                cull_target=int(target_instance_count) if (target_instance_count and pre_cull_to_target) else 0,
                cull_use_iou=int(bool(pre_cull_iou_threshold)), cull_iou_threshold=float(pre_cull_iou_threshold or 0.0),
                oks_errors=None if oks_errors is None else np.asarray(oks_errors, np.float64).reshape(-1),
                oks_score_weighting=int(bool(oks_score_weighting)), oks_normalization=DEVICE_OKS_NORMALIZATIONS[oks_normalization])
        if clean_instance_count:
            tracker_obj.cleaner = TrackCleaner(instance_count=int(clean_instance_count), iou_threshold=clean_iou_threshold)
        # Kalman filters on top of the regular tracker (:955-991; sleap_b200/nn/kalman.py)
        if (max_tracks or target_instance_count) and kf_init_frame_count:
            if not kf_node_indices:
                raise ValueError("Kalman filter requires node indices for instance tracking.")
            if tracker in ("flow", "flowmaxtracks"):
                raise ValueError("Kalman filter requires simple tracker for initial tracking.")
            if similarity == "normalized_instance":
                raise ValueError("Kalman filter does not support normalized_instance_similarity.")
            from sleap_b200.nn.kalman import KalmanTracker
            return KalmanTracker.make_tracker(init_tracker=tracker_obj, init_frame_count=int(kf_init_frame_count),
                                              node_indices=[int(i) for i in kf_node_indices],
                                              instance_count=int(target_instance_count or max_tracks),
                                              instance_iou_threshold=pre_cull_iou_threshold)
        if kf_init_frame_count and not (max_tracks or target_instance_count):
            raise ValueError("Kalman filter requires max tracks or target instance count.")
        return tracker_obj


def run_tracker(frames: list, tracker: Tracker, images=None, device_chunk: int = 256) -> list:
    """Track the predicted instances of ``frames`` (sorted by frame index) in place (tracking.py:1542-1580).
    ``images``: ``frame_idx -> image`` (mapping or callable), needed by the flow trackers.  A tracker with
    ``track_device`` tracks ``device_chunk`` frames per kernel call."""
    frames = sorted(frames, key=lambda lf: lf.frame_idx)
    if tracker.track_device is not None and tracker.candidate_maker is not None:
        for s in range(0, len(frames), device_chunk):
            chunk = frames[s:s + device_chunk]
            hws = []
            for lf in chunk:
                img = None
                if images is not None:
                    img = images(lf.frame_idx) if callable(images) else images[lf.frame_idx]
                hws.append(tuple(np.asarray(img).shape[:2]) if img is not None else (1, 1))
            out, err = tracker.track_frames([list(lf.instances) for lf in chunk], [lf.frame_idx for lf in chunk], hws)
            for lf, tracked in zip(chunk, out):
                lf.instances = tracked
            if err is not None:
                raise err
        tracker.final_pass(frames)
        return frames
    for lf in frames:
        img = None
        if images is not None:
            img = images(lf.frame_idx) if callable(images) else images[lf.frame_idx]
        hw = tuple(np.asarray(img).shape[:2]) if img is not None else (1, 1)
        lf.instances = tracker.track(list(lf.instances), img_hw=hw, img=img, t=lf.frame_idx)
    tracker.final_pass(frames)
    return frames
