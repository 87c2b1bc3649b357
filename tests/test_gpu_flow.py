"""Device flow shift (sleap_b200/csrc/sb_flow.cu) against OpenCV: gray conversion, resize, pyramid, derivatives and
level count bit-exact; Lucas-Kanade against cv2.calcOpticalFlowPyrLK; the flow trackers on the clip with and without
the device."""
import numpy as np
import pytest

cv2 = pytest.importorskip("cv2")

from sleap_b200.nn import tracking as T
from sleap_b200.nn.flow import DeviceFlow
from flow_clip import clip_frames, clip_points, track_clip

pytestmark = pytest.mark.gpu

CRIT = (cv2.TERM_CRITERIA_EPS | cv2.TERM_CRITERIA_COUNT, 30, 0.01)


@pytest.fixture(scope="module")
def clip():
    return clip_frames(200)


def _gray(img):
    img = img[..., 0] if img.ndim == 3 and img.shape[-1] == 1 else img
    return cv2.cvtColor(img, cv2.COLOR_BGR2GRAY) if img.ndim == 3 else img


def _frames(clip):
    rng = np.random.default_rng(11)
    smooth = lambda a: cv2.GaussianBlur(a, (0, 0), 2.0)
    return {"clip0": clip[0], "clip1_gray": clip[1][..., :1],
            "odd_97x131x3": smooth(rng.integers(0, 256, (97, 131, 3), dtype=np.uint8)),
            "odd_97x131x1": smooth(rng.integers(0, 256, (97, 131), dtype=np.uint8))[..., None],
            "odd_131x97": smooth(rng.integers(0, 256, (131, 97), dtype=np.uint8)),
            "small_45x60x3": rng.integers(0, 256, (45, 60, 3), dtype=np.uint8)}


@pytest.mark.parametrize("win,max_levels", [(21, 3), (5, 8), (9, 0), (41, 3), (4, 2), (3, 1)])
@pytest.mark.parametrize("scale", [1.0, 0.5])
def test_pyramid_bit_exact(clip, scale, win, max_levels):
    flow = DeviceFlow(0, win, max_levels, scale, ring=4)
    for t, (name, img) in enumerate(_frames(clip).items()):
        g = _gray(img)
        if scale != 1:
            g = cv2.resize(g, None, None, scale, scale)
        n, pyr = cv2.buildOpticalFlowPyramid(g, (win, win), max_levels, withDerivatives=True)
        flow.add_frame(t, img)
        for level in range(n + 1):
            im, der, n_levels = flow.fetch_level(t, level)
            assert n_levels == n + 1, (name, n_levels, n)
            np.testing.assert_array_equal(im, pyr[2 * level], err_msg=f"{name} level {level} image")
            np.testing.assert_array_equal(der, pyr[2 * level + 1], err_msg=f"{name} level {level} derivatives")
    flow.close()


def _lk_points(pts_ref, hw, seed):
    """Instance points + a seeded grid over the frame (flat background included) + points near and beyond every
    border + NaN points."""
    h, w = hw
    rng = np.random.default_rng(seed)
    grid = np.stack(np.meshgrid(np.linspace(3, w - 4, 14), np.linspace(3, h - 4, 14)), -1).reshape(-1, 2)
    grid = grid + rng.uniform(-2, 2, grid.shape)
    edge = np.concatenate([np.stack([rng.uniform(-3, 12, 12), rng.uniform(0, h, 12)], -1),
                           np.stack([rng.uniform(w - 12, w + 3, 12), rng.uniform(0, h, 12)], -1),
                           np.stack([rng.uniform(0, w, 12), rng.uniform(-3, 12, 12)], -1),
                           np.stack([rng.uniform(0, w, 12), rng.uniform(h - 12, h + 3, 12)], -1)])
    outside = np.array([[-40.0, 10.0], [w + 30.0, 50.0], [20.0, -60.0], [100.0, h + 45.0], [-500.0, -500.0]])
    nan = np.array([[np.nan, np.nan], [np.nan, 5.0], [7.0, np.nan]])
    return np.concatenate([pts_ref[np.isfinite(pts_ref).all(1)], grid, edge, outside, nan]).astype(np.float32)


def _assert_lk_matches(got, st_got, err_got, want, st_want, err_want, what, err_slack=0.0):
    """Status identical, found points within 0.01 px, err within 1e-3 (+ err_slack); returns the found points'
    differences."""
    st_want = st_want.reshape(-1)
    assert np.array_equal(st_got, st_want), (what, np.flatnonzero(st_got != st_want))
    found = st_want == 1
    d = np.abs(got[found] - want[found]).max(1)
    assert d.max() <= 0.01, (what, np.sort(d)[-5:])
    e = np.abs(err_got[found] - err_want.reshape(-1)[found])
    assert (e <= 1e-3 + err_slack).all(), (what, e.max(), d[np.argmax(e)])
    return d


def _lk_against_cv2(clip, scale, win, max_levels):
    """cv2.calcOpticalFlowPyrLK and the device on four frame pairs of the clip, _lk_points of each first frame."""
    pts_all, _, counts = clip_points()
    flow = DeviceFlow(0, win, max_levels, scale, ring=8)
    diffs, n_found, n_total = [], 0, 0
    for t0, gap in ((0, 1), (0, 5), (40, 1), (120, 5)):
        t1 = t0 + gap
        g0, g1 = _gray(clip[t0]), _gray(clip[t1])
        if scale != 1:
            g0, g1 = cv2.resize(g0, None, None, scale, scale), cv2.resize(g1, None, None, scale, scale)
        pts = _lk_points(pts_all[t0, :counts[t0]].reshape(-1, 2), clip[t0].shape[:2], t0) * np.float32(scale)
        want, st_want, err_want = cv2.calcOpticalFlowPyrLK(g0, g1, pts.copy(), None, winSize=(win, win), maxLevel=max_levels,
                                                           criteria=CRIT)
        flow.add_frame(t0, clip[t0], replace=False)
        flow.add_frame(t1, clip[t1], replace=False)
        got, st_got, err_got = flow.shift(t1, np.full(len(pts), t0), pts)
        d = _assert_lk_matches(got, st_got, err_got, want, st_want, err_want, (t0, gap))
        assert not st_got[-8:].any()                         # outside the frame and NaN
        diffs.append(d)
        n_found += len(d); n_total += len(pts)
    d = np.concatenate(diffs)
    print(f"\nLK vs cv2 (window {win}, {max_levels} levels, scale {scale}): {n_found}/{n_total} found, point difference "
          f"median {np.median(d):.2e} px, max {d.max():.2e} px")
    flow.close()


@pytest.mark.parametrize("scale", [1.0, 0.5])
def test_lk_matches_opencv(clip, scale):
    _lk_against_cv2(clip, scale, 21, 3)


# even windows (the window centre falls between pixels), the smallest and the largest window, no pyramid and 5 levels
@pytest.mark.parametrize("win,max_levels", [(3, 0), (4, 1), (8, 2), (13, 5), (31, 3), (41, 0), (41, 2)])
@pytest.mark.parametrize("scale", [1.0, 0.5])
def test_lk_windows_match_opencv(clip, scale, win, max_levels):
    _lk_against_cv2(clip, scale, win, max_levels)


def test_lk_checkerboard_at_window_41():
    """A binary checkerboard shifted by (3, 2) px: the largest derivatives and image differences a uint8 frame has,
    over the largest window (the per-lane int sums of k_flow_lk at their bound)."""
    yy, xx = np.mgrid[0:240, 0:320]
    board = lambda dx, dy: ((((xx - dx) // 12) + ((yy - dy) // 12)) % 2 * 255).astype(np.uint8)
    g0, g1 = board(0, 0), board(3, 2)
    pts = _lk_points(np.zeros((0, 2)), g0.shape, 5)
    want, st_want, err_want = cv2.calcOpticalFlowPyrLK(g0, g1, pts.copy(), None, winSize=(41, 41), maxLevel=2, criteria=CRIT)
    flow = DeviceFlow(0, 41, 2, 1.0, ring=2)
    flow.add_frame(0, g0)
    flow.add_frame(1, g1)
    got, st_got, err_got = flow.shift(1, np.zeros(len(pts), np.int64), pts)
    # err is read at the found point, and the found points differ by the rounding of OpenCV's float window sums (the
    # device sums exactly): on a 0/255 board a window sample moves by up to 255 per px of motion, so err may differ by
    # that much times the point difference on top of the usual 1e-3
    found = st_want.reshape(-1) == 1
    slack = 255 * np.abs(got[found] - want[found]).sum(1)
    d = _assert_lk_matches(got, st_got, err_got, want, st_want, err_want, "checkerboard", err_slack=slack)
    assert len(d) > 100
    flow.close()


def test_shift_many_reference_frames_in_one_call(clip):
    """One call shifts points of several reference frames; it equals one call per reference frame, and a frame that is
    not held is an error."""
    from sleap_b200 import _lib
    flow = DeviceFlow(0, 21, 3, 1.0, ring=6)
    for t in range(6):
        flow.add_frame(t, clip[t])
    pts_all, _, counts = clip_points()
    reqs = [(t, pts_all[t, :counts[t]].reshape(-1, 2)) for t in range(5)]
    pts = np.concatenate([p for _, p in reqs]).astype(np.float32)
    ref = np.concatenate([np.full(len(p), t) for t, p in reqs])
    got, st, err = flow.shift(5, ref, pts)
    for t, p in reqs:
        g1, s1, e1 = flow.shift(5, np.full(len(p), t), p)
        np.testing.assert_array_equal(got[ref == t], g1)
        np.testing.assert_array_equal(st[ref == t], s1)
    with pytest.raises(_lib.SleapB200Error):
        flow.shift(5, [99], pts[:1])
    with pytest.raises(_lib.SleapB200Error):
        flow.shift(98, [0], pts[:1])
    flow.add_frame(6, clip[6])                               # the ring is full: the least recently used frame (0) goes
    with pytest.raises(_lib.SleapB200Error):
        flow.shift(6, [0], pts[:1])
    flow.shift(6, [1], pts[:1])
    flow.add_frame(0, clip[0][:512, :512])                   # another frame size empties the ring
    with pytest.raises(_lib.SleapB200Error):
        flow.shift(0, [1], pts[:1])
    flow.close()


def test_ring_past_64_slots(clip):
    """A ring of 100 frames: points of the frames held in slots 64-98 shift into frame 99 as cv2 shifts them, and
    reserve grows a ring past 64 slots."""
    frames = clip[:100, :384, :384]
    flow = DeviceFlow(0, 21, 3, 1.0, ring=100)
    for t in range(100):
        flow.add_frame(t, frames[t])
    g1 = _gray(frames[99])
    for t in range(64, 99, 3):
        pts = _lk_points(np.zeros((0, 2)), (384, 384), t)
        want, st_want, err_want = cv2.calcOpticalFlowPyrLK(_gray(frames[t]), g1, pts.copy(), None, winSize=(21, 21), maxLevel=3,
                                                           criteria=CRIT)
        got, st_got, err_got = flow.shift(99, np.full(len(pts), t), pts)
        _assert_lk_matches(got, st_got, err_got, want, st_want, err_want, t)
    flow.shift(99, np.arange(100), np.full((100, 2), 50.0, np.float32))        # every frame is still held
    flow.close()
    flow = DeviceFlow(0, 9, 1, 0.5, ring=2)
    flow.reserve(80)
    assert flow.ring == 80
    for t in range(80):
        flow.add_frame(t, frames[t])
    flow.shift(79, np.arange(80), np.full((80, 2), 50.0, np.float32))
    flow.close()


def _same_tracking(cpu, dev, what):
    """The bars of the flow trackers: same track names, tracking scores within 1e-2."""
    names_cpu = [[i.track.name for i in lf.instances] for lf in cpu]
    names_dev = [[i.track.name for i in lf.instances] for lf in dev]
    assert names_dev == names_cpu
    sc_cpu = np.array([i.tracking_score for lf in cpu for i in lf.instances])
    sc_dev = np.array([i.tracking_score for lf in dev for i in lf.instances])
    diff = float(np.abs(sc_cpu - sc_dev).max())
    print(f"\n{what}: {len(sc_cpu)} instances, tracking score max difference {diff:.2e}")
    assert diff <= 1e-2


@pytest.mark.parametrize("tracker,save", [("flow", False), ("flow", True), ("flowmaxtracks", False)])
def test_tracking_device_matches_cv2(clip, tracker, save):
    n = 200
    _same_tracking(track_clip(tracker, save, n, clip), track_clip(tracker, save, n, clip, of_device=0), f"{tracker} save={save}")


@pytest.mark.parametrize("window", [63, 64])
def test_flow_tracker_window_past_the_old_ring_cap(clip, window):
    """track_window 63 and 64: the device flow keeps track_window + 2 = 65 and 66 frames."""
    n = 70
    _same_tracking(track_clip("flow", False, n, clip, track_window=window),
                   track_clip("flow", False, n, clip, track_window=window, of_device=0), f"flow window {window}")


def test_flow_tracker_small_window_one_level(clip):
    kw = dict(of_window_size=9, of_max_levels=1)
    n = 60
    _same_tracking(track_clip("flow", False, n, clip, **kw), track_clip("flow", False, n, clip, of_device=0, **kw),
                   "flow window 9, 1 level")


def _staggered_loss(n_frames=90):
    """16 three-node blob animals on a 140 x 170 frame; animal a is seen in frames [0, 6 + 5 a).  flowmaxtracks keeps
    the last 5 frames of every lost track, so from frame 65 on one shift reads more than 64 frames."""
    from sleap_b200.nn.inference import LabeledFrame, PredictedInstance
    from test_tracking import _blob_frame
    shape = np.array([[-6.0, 0.0], [0.0, 0.0], [6.0, 0.0]])
    pos = lambda a, t: shape + [20.0 + 40 * (a % 4) + 0.1 * t * (-1) ** a, 20.0 + 33 * (a // 4)]
    frames, imgs = [], {}
    for t in range(n_frames):
        seen = [a for a in range(16) if t < 6 + 5 * a]
        frames.append(LabeledFrame(0, t, [PredictedInstance.from_numpy(pos(a, t), [1, 1, 1], 1.0) for a in seen]))
        imgs[t] = _blob_frame([c for a in seen for c in pos(a, t)], hw=(140, 170))
    return frames, imgs


def test_flowmaxtracks_shift_reads_more_than_64_frames():
    from track_cases import copy_frames
    frames, imgs = _staggered_loss()
    # Hungarian: its matches come in instance order, where greedy lists them by cost, and the 16 near-perfect matches
    # have costs within the flow's rounding of each other
    kw = dict(tracker="flowmaxtracks", similarity="instance", match="hungarian", track_window=5, max_tracks=16, max_tracking=True)
    cpu = T.run_tracker(copy_frames(frames), T.Tracker.make_tracker_by_name(**kw), images=imgs)
    tr = T.Tracker.make_tracker_by_name(of_device=0, **kw)
    dev = T.run_tracker(copy_frames(frames), tr, images=imgs)
    _same_tracking(cpu, dev, "flowmaxtracks, staggered losses")
    assert tr.candidate_maker._device_flow.ring > 64


@pytest.mark.parametrize("tracker,save", [("flow", False), ("flow", True), ("flowmaxtracks", False)])
def test_device_flow_tracker_keeps_identities_across_a_jump(tracker, save):
    """test_tracking.py's jump scenario on the device: the shifted candidates bridge a 6 px step."""
    from sleap_b200.nn.inference import LabeledFrame, PredictedInstance
    from test_tracking import _blob_frame
    shape = np.array([[-8.0, 0.0], [0.0, 0.0], [8.0, 0.0]])
    pos = lambda t: (shape + [30.0 + 6 * t, 30.0], shape + [100.0 - 6 * t, 70.0])
    frames = [LabeledFrame(0, t, [PredictedInstance.from_numpy(pos(t)[0], [1, 1, 1], 1.0), PredictedInstance.from_numpy(pos(t)[1], [1, 1, 1], 1.0)])
              for t in range(6)]
    imgs = {t: _blob_frame(np.concatenate(pos(t))) for t in range(6)}
    tr = T.Tracker.make_tracker_by_name(tracker=tracker, similarity="instance", match="hungarian", track_window=3, max_tracks=2,
                                        max_tracking=tracker == "flowmaxtracks", save_shifted_instances=save, of_device=0)
    out = T.run_tracker(frames, tr, images=imgs)
    names = [[i.track.name for i in lf.instances] for lf in out]
    assert all(n == names[0] for n in names) and len(set(names[0])) == 2, names
    assert tr.candidate_maker._device_flow is not None
