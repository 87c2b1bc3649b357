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


@pytest.mark.parametrize("win,max_levels", [(21, 3), (5, 8), (9, 0)])
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


@pytest.mark.parametrize("scale", [1.0, 0.5])
def test_lk_matches_opencv(clip, scale):
    pts_all, _, counts = clip_points()
    flow = DeviceFlow(0, 21, 3, scale, ring=8)
    diffs, n_found, n_total = [], 0, 0
    for t0, gap in ((0, 1), (0, 5), (40, 1), (120, 5)):
        t1 = t0 + gap
        g0, g1 = _gray(clip[t0]), _gray(clip[t1])
        if scale != 1:
            g0, g1 = cv2.resize(g0, None, None, scale, scale), cv2.resize(g1, None, None, scale, scale)
        pts = _lk_points(pts_all[t0, :counts[t0]].reshape(-1, 2), clip[t0].shape[:2], t0) * np.float32(scale)
        want, st_want, err_want = cv2.calcOpticalFlowPyrLK(g0, g1, pts.copy(), None, winSize=(21, 21), maxLevel=3, criteria=CRIT)
        flow.add_frame(t0, clip[t0], replace=False)
        flow.add_frame(t1, clip[t1], replace=False)
        got, st_got, err_got = flow.shift(t1, np.full(len(pts), t0), pts)
        st_want = st_want.reshape(-1)
        assert np.array_equal(st_got, st_want), (t0, gap, np.flatnonzero(st_got != st_want))
        found = st_want == 1
        d = np.abs(got[found] - want[found]).max(1)
        assert d.max() <= 0.01, (t0, gap, np.sort(d)[-5:])
        assert np.abs(err_got[found] - err_want.reshape(-1)[found]).max() <= 1e-3
        assert not st_got[-8:].any()                         # outside the frame and NaN
        diffs.append(d)
        n_found += int(found.sum()); n_total += len(pts)
    d = np.concatenate(diffs)
    print(f"\nLK vs cv2 (scale {scale}): {n_found}/{n_total} found, point difference median {np.median(d):.2e} px, "
          f"max {d.max():.2e} px")
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


@pytest.mark.parametrize("tracker,save", [("flow", False), ("flow", True), ("flowmaxtracks", False)])
def test_tracking_device_matches_cv2(clip, tracker, save):
    n = 200
    cpu = track_clip(tracker, save, n, clip)
    dev = track_clip(tracker, save, n, clip, of_device=0)
    names_cpu = [[i.track.name for i in lf.instances] for lf in cpu]
    names_dev = [[i.track.name for i in lf.instances] for lf in dev]
    assert names_dev == names_cpu
    sc_cpu = np.array([i.tracking_score for lf in cpu for i in lf.instances])
    sc_dev = np.array([i.tracking_score for lf in dev for i in lf.instances])
    diff = float(np.abs(sc_cpu - sc_dev).max())
    print(f"\n{tracker} save={save}: {len(sc_cpu)} instances, tracking score max difference {diff:.2e}")
    assert diff <= 1e-2


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
