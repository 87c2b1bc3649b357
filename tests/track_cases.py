"""Shared by the device-tracker tests: the host tracker with its greedy ties made stable, seeded synthetic frames and
the comparison of a host and a device tracking run."""
import contextlib
import math

import numpy as np

from sleap_b200.nn import tracking as T
from sleap_b200.nn.inference import LabeledFrame, PredictedInstance


def greedy_matching_stable(cost: np.ndarray):
    """greedy_matching with ties broken by ascending flat index (np.argsort(kind="stable")), the device's rule."""
    order = np.argsort(cost, axis=None, kind="stable")
    used_r, used_c, out = set(), set(), []
    for flat in order.tolist():
        r, c = divmod(flat, cost.shape[1])
        if r in used_r or c in used_c:
            continue
        used_r.add(r); used_c.add(c)
        out.append((r, c))
    return out


def host_twin(**kw) -> T.Tracker:
    """The host tracker of ``make_tracker_by_name(**kw)`` with the stable greedy matcher."""
    tr = T.Tracker.make_tracker_by_name(**kw)
    if tr.matching_function is T.greedy_matching:
        tr.matching_function = greedy_matching_stable
    return tr


def copy_frames(frames: list) -> list:
    """New LabeledFrames holding the same instance objects (tracking replaces the lists, not the instances)."""
    return [LabeledFrame(lf.video, lf.frame_idx, list(lf.instances)) for lf in frames]


def synthetic_frames(seed: int, n_frames: int = 300, max_instances: int = 32, n_nodes: int = 13, hw=(256, 256),
                     all_nan: float = 0.03) -> list:
    """Animals that appear, disappear and sometimes jump far; NaN nodes, all-NaN instances (a share ``all_nan``: their
    NaN similarity rows make SciPy's Hungarian matcher raise), distinct scores."""
    rng = np.random.default_rng(seed)
    n_animals = max_instances + 8
    pos = rng.uniform(20, min(hw) - 20, (n_animals, 2))
    shape = rng.normal(0, 6, (n_animals, n_nodes, 2))
    alive = rng.random(n_animals) < 0.5
    frames = []
    for t in range(n_frames):
        pos += rng.normal(0, 1.5, pos.shape)
        jump = rng.random(n_animals) < 0.02
        pos[jump] = rng.uniform(20, min(hw) - 20, (int(jump.sum()), 2))
        flip = rng.random(n_animals) < 0.05
        alive ^= flip
        ids = np.flatnonzero(alive)[:rng.integers(0, max_instances + 1)]
        rng.shuffle(ids)
        insts = []
        for a in ids:
            p = pos[a] + shape[a] + rng.normal(0, 0.7, (n_nodes, 2))
            p[rng.random(n_nodes) < 0.15] = np.nan
            if rng.random() < all_nan:
                p[:] = np.nan
            conf = rng.uniform(0.2, 1.0, n_nodes)
            insts.append(PredictedInstance.from_numpy(p, conf, float(rng.uniform(0.1, 5.0))))
        frames.append(LabeledFrame(0, t, insts))
    return frames


def counted_frames(seed: int, shown: list, n_nodes: int = 13, hw=(1024, 1024), score_levels: int = 0) -> list:
    """One frame per entry of ``shown``: an int k shows animals 0..k-1, a list shows those animal ids; each frame's
    order is shuffled.  Animals persist: each keeps its skeleton and walks 1.5 px per frame, so one that leaves and
    comes back can be matched again.  About 15 % of the nodes are NaN, never all of an instance's (no all-NaN
    similarity rows, which SciPy's Hungarian matcher rejects).  Scores are distinct, or with ``score_levels`` > 0
    drawn from that many values, so that most scores are tied."""
    rng = np.random.default_rng(seed)
    ids = [np.arange(s) if np.isscalar(s) else np.asarray(s) for s in shown]
    n_animals = 1 + max(int(i.max()) for i in ids if len(i))
    side = int(np.ceil(np.sqrt(n_animals)))                  # a jittered grid: neighbours 60+ px apart at 1024^2
    cell = np.array([hw[1], hw[0]], np.float64) / side
    pos = (np.stack([np.arange(n_animals) % side, np.arange(n_animals) // side], -1) + 0.5) * cell
    pos += rng.uniform(-0.15, 0.15, pos.shape) * cell
    shape = rng.normal(0, 0.12 * cell.min(), (n_animals, n_nodes, 2))
    frames = []
    for t, a_ids in enumerate(ids):
        pos += rng.normal(0, 1.5, pos.shape)
        insts = []
        for a in rng.permutation(a_ids):
            p = pos[a] + shape[a] + rng.normal(0, 0.7, (n_nodes, 2))
            lost = rng.random(n_nodes) < 0.15
            lost[rng.integers(n_nodes)] = False
            p[lost] = np.nan
            score = rng.integers(score_levels) / score_levels if score_levels else rng.uniform(0.1, 5.0)
            insts.append(PredictedInstance.from_numpy(p, rng.uniform(0.2, 1.0, n_nodes), float(score)))
        frames.append(LabeledFrame(0, t, insts))
    return frames


@contextlib.contextmanager
def stable_argsort():
    """Every np.argsort stable while the block runs: the host's nms_fast then orders equal scores as the device's
    pre-cull does (the default sort leaves that order to the implementation)."""
    argsort = np.argsort
    np.argsort = lambda a, axis=-1, kind=None, order=None: argsort(a, axis=axis, kind="stable", order=order)
    try:
        yield
    finally:
        np.argsort = argsort


def _close(a: float, b: float) -> bool:
    if math.isnan(a) or math.isnan(b):
        return math.isnan(a) and math.isnan(b)
    if math.isinf(a) or math.isinf(b):
        return a == b
    return abs(a - b) <= 1e-12 * max(abs(a), abs(b), 1e-300)


def assert_same_tracking(host: list, dev: list, host_tracker: T.Tracker, dev_tracker: T.Tracker):
    """Same instances per frame in the same order, same tracks, same spawned tracks, tracking scores within 1e-12."""
    assert len(host) == len(dev)
    for lh, ld in zip(host, dev):
        assert lh.frame_idx == ld.frame_idx
        assert [id(x.points) for x in lh.instances] == [id(x.points) for x in ld.instances], lh.frame_idx
        assert [x.track.name for x in lh.instances] == [x.track.name for x in ld.instances], lh.frame_idx
        for xh, xd in zip(lh.instances, ld.instances):
            assert _close(xh.tracking_score, xd.tracking_score), (lh.frame_idx, xh.tracking_score, xd.tracking_score)
    assert [(t.name, t.spawned_on) for t in host_tracker.spawned_tracks] == \
        [(t.name, t.spawned_on) for t in dev_tracker.spawned_tracks]
