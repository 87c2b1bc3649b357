"""Runs below the configured batch, and each frame's outputs against its batch.

Production mostly runs a model below the batch it was configured (and autotuned) at: the top-down instance network on
the few crops of a call, the ragged last batch of a video.  There the persistent forms size their grid and walk their
items over the run's batch, and every buffer slot past the run's last frame still holds an earlier call's data, so a
kernel that reads a neighbouring frame (the next frame's first row for the bottom SAME-pad row) or indexes by the wrong
batch count reads stale data.

  * Partial-batch audit: the float64 per-element layer audit of test_gpu_layer_audit.py (``_audit`` with ``max_batch``):
    configure at B_cfg, one poison forward of B_cfg other frames with every buffer fetched, then the production and
    all-buffers audits of B_run < B_cfg frames, gated as there.  Every tensor-core form, each input stage (k_conv01, the
    frame view, k_conv_first, the stem and buffer views, k_preprocess's resize), uint8 and float frames, precisions 0-2.
  * Batch composition: each frame's fp32 head outputs are bit-identical whatever the configured batch, the run's batch,
    the frame's position and its neighbours, with programmatic dependent launch on or off (C4 at the benchmark's size),
    and a frame's fused top-down record is the same alone or between two others."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

import layer_audit as la
from conv_forms import PICKED, same_bits
from test_gpu_layer_audit import _audit, _c4, _frames, _resnet
from test_gpu_layer_audit_configs import BILINEAR_RGB, C3_INSTANCE, HOURGLASS

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FORMS = ["streaming", "resident", "halo", "wide", "tconv-fused"]                  # SB_FORCE_VARIANT = 0 .. 4
STAGES = {"conv01": ({"SB_FORCE_CONV01": "1"}, "-> fused"),
          "frame_view": ({"SB_FORCE_CONV01": "0", "SB_FORCE_FIRST_VIEW": "1"}, "-> view"),
          "conv_first": ({"SB_FORCE_CONV01": "0", "SB_DISABLE_FIRST_VIEW": "1"}, None)}
# first conv (op 1) on the tensor cores through a view, or k_conv_first on the CUDA cores; k_conv01 is checked by its line
STAGE_ENGINE = {"frame_view": "tc", "conv_first": "cuda"}


def _first_engine(rows):
    return next(r["engine"] for r in rows if r["op"] == 1)


# ------------------------------------------------------------------------------------------------ partial-batch audit
C4_CASES = {"autotuned_6to1": ({}, None, 6, 1), "autotuned_6to4": ({}, None, 6, 4),       # case_<B_cfg>to<B_run>
            **{f"{name}_4to1": ({"SB_FORCE_VARIANT": str(f)}, PICKED.get(f), 4, 1) for f, name in enumerate(FORMS)},
            "conv01_4to1": (*STAGES["conv01"], 4, 1), "conv01_4to3": (*STAGES["conv01"], 4, 3),
            "frame_view_4to1": (*STAGES["frame_view"], 4, 1), "conv_first_4to1": (*STAGES["conv_first"], 4, 1)}


@pytest.mark.parametrize("case", list(C4_CASES))
def test_batch_audit_c4(case, capfd, monkeypatch):
    """C4 UNet, 200 x 232 uint8 frames: autotuned, every tensor-core form forced, each first-layer stage pinned."""
    env, expect, b_cfg, b_run = C4_CASES[case]
    rows = _audit(_c4(), 1, _frames((b_run, 200, 232, 1), 21), 0, capfd, monkeypatch, env, expect, max_batch=b_cfg)
    stage = case.rsplit("_", 1)[0]
    if stage in STAGE_ENGINE:
        assert _first_engine(rows) == STAGE_ENGINE[stage]


@pytest.mark.parametrize("stage", list(STAGES))
def test_batch_audit_c4_float_frames(stage, capfd, monkeypatch):
    """Float frames in [0, 1]: the <float> instantiations of k_conv01, k_first_view and k_conv_first."""
    env, expect = STAGES[stage]
    imgs = np.random.default_rng(22).uniform(0, 1, (1, 200, 232, 1)).astype(np.float32)
    rows = _audit(_c4(), 1, imgs, 0, capfd, monkeypatch, env, expect, max_batch=4)
    if stage in STAGE_ENGINE:
        assert _first_engine(rows) == STAGE_ENGINE[stage]


@pytest.mark.parametrize("case", ["autotuned", "resident"])
@pytest.mark.parametrize("b_run", [1, 5])
def test_batch_audit_c3_instance(case, b_run, capfd, monkeypatch):
    """C3's centered-instance net configured at 16 crops of 160 x 160 and run on a few: the top-down pattern."""
    env, expect = ({}, None) if case == "autotuned" else ({"SB_FORCE_VARIANT": "1"}, PICKED[1])
    _audit(C3_INSTANCE, 1, _frames((b_run, 160, 160, 1), 23), 0, capfd, monkeypatch, env, expect, max_batch=16)


@pytest.mark.parametrize("precision", [0, 2])
def test_batch_audit_resnet50(precision, capfd, monkeypatch):
    """ResNet50 with k4 transposed convs, 3 -> 1; in precision 0 the stem runs through its space-to-depth view."""
    rows = _audit(_resnet("tconv_concat"), 3, _frames((1, 150, 176, 3), 24), precision, capfd, monkeypatch, max_batch=3)
    if precision == 0:
        assert _first_engine(rows) == "tc"


@pytest.mark.parametrize("dtype", ["uint8", "float32"])
def test_batch_audit_hourglass(dtype, capfd, monkeypatch):
    """The 7x7/2 stem through its space-to-depth view (k_s2d_view<uint8 / float>), plain preprocessing, 3 -> 2."""
    imgs = _frames((2, 120, 136, 3), 25)
    if dtype == "float32":
        imgs = (imgs / np.float32(255)).astype(np.float32)
    rows = _audit(HOURGLASS, 3, imgs, 0, capfd, monkeypatch, max_batch=3)
    assert _first_engine(rows) == "tc"


def test_batch_audit_bilinear_resized_rgb(capfd, monkeypatch):
    """RGB frames into a gray model at input_scale 0.5: k_preprocess's resize, then the view of the preprocessed buffer."""
    rows = _audit(BILINEAR_RGB, 1, _frames((1, 300, 346, 3), 26), 0, capfd, monkeypatch, input_scale=0.5, max_batch=3)
    assert _first_engine(rows) == "tc"


@pytest.mark.parametrize("case", ["autotuned", "resident"])
def test_batch_audit_c4_precision2(case, capfd, monkeypatch):
    """Precision 2, 4 -> 1: k_conv_first's split store, and the resident form (the only other one open to precision 2)."""
    env, expect = ({}, None) if case == "autotuned" else ({"SB_FORCE_VARIANT": "1"}, PICKED[1])
    _audit(_c4(), 1, _frames((1, 200, 232, 1), 27), 2, capfd, monkeypatch, env, expect, max_batch=4)


def test_batch_audit_c4_precision1(capfd, monkeypatch):
    """The fp32 CUDA-core path, 3 -> 1."""
    _audit(_c4(), 1, _frames((1, 200, 232, 1), 28), 1, capfd, monkeypatch, max_batch=3)


# ------------------------------------------------------------------------------------------------ batch composition
# The input stage pinned to k_conv01 over k_conv_first: the two input-stage choices whose arithmetic differs.  The conv
# forms stay autotuned per configuration; they are bit-identical to each other.
PINNED = {"SB_FORCE_CONV01": "1", "SB_DISABLE_FIRST_VIEW": "1"}


@functools.lru_cache(maxsize=None)
def _bench_weights():
    """bench.py's C4 weights, calibrated as the benchmark does on its own calibration frames."""
    import bench
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    weights = A.make_synthetic_weights(A.compile_model(bench.c4_spec(), 1), bench.SEED)
    calib = bench.make_frames(2, 500)
    cms0, pafs0 = DeviceModel(bench.c4_spec(), weights, input_channels=1, precision=0).forward(calib)
    return bench.calibrate_heads(weights, cms0, pafs0, len(calib))


def _model(b_cfg, hw, precision=0, env=()):
    import bench
    from sleap_b200.nn.model import DeviceModel
    with pytest.MonkeyPatch.context() as mp:
        for k, v in dict(env).items():
            mp.setenv(k, v)
        m = DeviceModel(bench.c4_spec(), _bench_weights(), input_channels=1, precision=precision)
        m.configure(b_cfg, hw, hw, 1)
    return m


def _run(model, frames, order):
    """{frame index: (cms, pafs)} of one forward over frames[order]."""
    cms, pafs = model.forward(np.ascontiguousarray(frames[list(order)]))
    return {f: (cms[i], pafs[i]) for i, f in enumerate(order)}


def _assert_same(ref, got, what):
    for f, (a, b) in got.items():
        for name, x, y in (("cms", ref[f][0], a), ("pafs", ref[f][1], b)):
            assert same_bits(x, y), (f"{what}: frame {f} {name} differs in {int((x != y).sum())} elements, "
                                     f"max |diff| {float(np.abs(x.astype(np.float64) - y).max()):.3g}")


def _bench_frames():
    import bench
    return bench.make_frames(8, 4242)


def test_heads_independent_of_batch_composition():
    """The benchmark's model (8 x 1024 x 1024, autotuned): the full 8, reversed, frames 0 and 7 alone, [f5, f2, f0]."""
    import bench
    frames = _bench_frames()
    model = _model(8, bench.H)
    ref = _run(model, frames, range(8))
    for order in (range(7, -1, -1), [0], [7], [5, 2, 0]):
        _assert_same(ref, _run(model, frames, order), f"B = {len(order)} {list(order)}")


@pytest.fixture(scope="module")
def pinned8():
    """(frames, heads) of the pinned model configured at 8 x 1024 x 1024."""
    import bench
    frames = _bench_frames()
    return frames, _run(_model(8, bench.H, env=PINNED), frames, range(8))


def test_heads_independent_of_configured_batch(pinned8):
    """Pinned input stage, configured at 8, 3 and 1 (each autotuned on its own): the same bits per frame, the ragged
    last batch of the B = 3 model included."""
    import bench
    frames, ref = pinned8
    m3 = _model(3, bench.H, env=PINNED)
    for chunk in ([0, 1, 2], [3, 4, 5], [6, 7]):
        _assert_same(ref, _run(m3, frames, chunk), f"configured at 3, B = {len(chunk)} {chunk}")
    m1 = _model(1, bench.H, env=PINNED)
    for f in range(8):
        _assert_same(ref, _run(m1, frames, [f]), "configured at 1")


def test_heads_independent_of_configured_batch_precision2():
    """Precision 2 on C4 at 512 x 512, configured at 4 and at 1."""
    frames = np.ascontiguousarray(_bench_frames()[:4, 256:768, 256:768])
    ref = _run(_model(4, 512, 2, PINNED), frames, range(4))
    m1 = _model(1, 512, 2, PINNED)
    for f in range(4):
        _assert_same(ref, _run(m1, frames, [f]), "precision 2 configured at 1")


CHILD = """
import sys
import numpy as np
import bench
from sleap_b200.nn.model import DeviceModel, load_weights_npz
d = sys.argv[1]
m = DeviceModel(bench.c4_spec(), load_weights_npz(d + "/weights.npz"), input_channels=1, precision=0)
m.configure(8, bench.H, bench.W, 1)
cms, pafs = m.forward(np.load(d + "/frames.npy"))
np.savez(d + "/heads.npz", cms=cms, pafs=pafs)
"""


def test_heads_independent_of_pdl(pinned8, tmp_path):
    """The pinned 8-frame model without programmatic dependent launch (the switch is read once per process, so in a
    child interpreter) gives the same bits."""
    from sleap_b200.nn.model import save_weights_npz
    frames, ref = pinned8
    save_weights_npz(str(tmp_path / "weights.npz"), _bench_weights())
    np.save(tmp_path / "frames.npy", frames)
    env = dict(os.environ, SB_DISABLE_PDL="1", PYTHONPATH=ROOT, **PINNED)
    flags = ["-s"] if sys.flags.no_user_site else []
    r = subprocess.run([sys.executable, *flags, "-c", CHILD, str(tmp_path)], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    z = np.load(tmp_path / "heads.npz")
    _assert_same(ref, {f: (z["cms"][f], z["pafs"][f]) for f in range(8)}, "SB_DISABLE_PDL=1")


def test_topdown_record_independent_of_batch():
    """Fused top-down (sb_infer_topdown), precision 0, 6 crops per frame and 4 crops per instance-network call: the
    middle of three frames has its crops in chunks shared with both neighbours, alone they are one full chunk and a
    ragged one, and the centroid network runs at 1 of its 3 configured frames.  The frame's record is the same bits."""
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.inference import TopDownPredictor
    from sleap_b200.nn.model import DeviceModel
    ccfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=2, middle_block=True, up_interpolate=True)
    cspec = dict(backbone="unet", backbone_cfg=ccfg, head_type="centroid", part_names=None, edges=None,
                 heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
    icfg = dict(filters=8, filters_rate=2, max_stride=16, output_stride=4, middle_block=True, up_interpolate=False)
    ispec = dict(backbone="unet", backbone_cfg=icfg, head_type="centered_instance", part_names=list("abcd"), edges=None,
                 heads=[dict(name="CenteredInstanceConfmapsHead", channels=4, output_stride=4)])
    cmodel, imodel = (DeviceModel(s, la.synthetic_weights(A.compile_model(s, 1), seed), input_channels=1, precision=0)
                      for s, seed in ((cspec, 51), (ispec, 53)))
    imgs = np.random.default_rng(8).integers(0, 256, size=(3, 192, 224, 1), dtype=np.uint8)
    thr = float(np.median(cmodel.forward(imgs)[0]))              # far more than 6 local maxima above it in every frame
    pred = TopDownPredictor(cmodel, imodel, crop_size=64, peak_threshold=thr, integral_refinement=True, batch_size=3,
                            max_instances=6)
    im = pred.inference_model
    im.instance_peaks.peak_threshold = -1e9
    im.instance_peaks.max_crops_per_call = 4
    assert im._can_fuse()
    three = im.predict_on_batch(imgs)
    assert three["n_valid"].tolist() == [6, 6, 6]
    one = im.predict_on_batch(imgs[1:2])
    assert cmodel.configured_for[0] == 3 and imodel.configured_for[0] == 4
    assert int(one["n_valid"][0]) == 6
    for k in ("centroids", "centroid_vals", "instance_peaks", "instance_peak_vals"):
        a, b = np.ascontiguousarray(three[k][1, :6]), np.ascontiguousarray(one[k][0, :6])
        assert same_bits(a, b), f"{k}: {a} vs {b}"
