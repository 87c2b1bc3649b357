"""The float64 per-element layer audit (tests/layer_audit.py, driven by test_gpu_layer_audit._audit) on the networks
that test_gpu_layer_audit.py does not reach:

  * the secondary benchmark configurations at their real widths (tools/bench_configs.py): C3's centered-instance UNet
    (24 .. 384 channels: Cout 24 through the generic epilogue, the N = 192 instantiation, padded 256-wide N tiles) with
    every tensor-core form forced in turn, C3's centroid UNet (the C1 / C2 backbone), C5's full-width hourglass
    (256 .. 768 channels, 10 - 12 K chunks, conv -> ReLU -> BN over several N tiles, a 46-channel head);
  * a filters_rate 1.5 UNet (16 / 24 / 36 / 54 / 81): the fp16 CUDA-core kernels with odd widths and odd concat offsets;
  * the trained fixture models under tests/golden/models on their committed frames;
  * precision 1, the fp32 CUDA-core path, on the networks of test_gpu_layer_audit.py.

Each case runs the production run and the all-buffers run, gated as in test_gpu_layer_audit.py (_gate)."""
import numpy as np
import pytest

import reference_models as rm
from test_gpu_layer_audit import _audit, _c4, _frames, _resnet

pytestmark = pytest.mark.gpu

FL13 = [f"n{i}" for i in range(13)]
FORMS = {"streaming": "0", "resident": "1", "halo": "2", "wide": "3"}


def _unet(filters, max_stride, output_stride, **kw):
    return dict(filters=filters, filters_rate=2, max_stride=max_stride, output_stride=output_stride, middle_block=True,
                up_interpolate=True, stacks=1, **kw)


# tools/bench_configs.py topdown()
C3_INSTANCE = dict(backbone="unet", backbone_cfg=dict(_unet(24, 16, 4), up_interpolate=False), head_type="centered_instance",
                   part_names=FL13, edges=None, heads=[dict(name="CenteredInstanceConfmapsHead", channels=13, output_stride=4)])
C3_CENTROID = dict(backbone="unet", backbone_cfg=_unet(16, 16, 2), head_type="centroid", part_names=None, edges=None,
                   heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
# tools/bench_configs.py hourglass()
C5_HOURGLASS = dict(backbone="hourglass", backbone_cfg=dict(stem_stride=4, max_stride=64, output_stride=4, stem_filters=128,
                                                            filters=256, filter_increase=128, stacks=3),
                    head_type="multi_instance", part_names=None, edges=None,
                    heads=[dict(name="MultiInstanceConfmapsHead", channels=24, output_stride=4),
                           dict(name="PartAffinityFieldsHead", channels=46, output_stride=4)])
UNET_RATE15 = dict(backbone="unet", backbone_cfg=dict(filters=16, filters_rate=1.5, max_stride=16, output_stride=2,
                                                      middle_block=True, up_interpolate=False, stacks=1),
                   head_type="multi_instance", part_names=None, edges=None,
                   heads=[dict(name="MultiInstanceConfmapsHead", channels=5, output_stride=2),
                          dict(name="PartAffinityFieldsHead", channels=8, output_stride=4)])


@pytest.mark.parametrize("case", ["autotuned", "streaming", "resident", "halo", "wide"])
def test_audit_c3_instance(case, capfd, monkeypatch):
    """C3's centered-instance net on 5 uint8 crops of 160 x 160 (10 x 10 deepest maps), autotuned and with each
    tensor-core form forced; a forced form must have run on at least one op."""
    env = {} if case == "autotuned" else {"SB_FORCE_VARIANT": FORMS[case]}
    expect = None if case in ("autotuned", "streaming") else f"-> {case}"
    _audit(C3_INSTANCE, 1, _frames((5, 160, 160, 1), 11), 0, capfd, monkeypatch, env, expect)


def test_audit_c3_instance_precision2(capfd, monkeypatch):
    _audit(C3_INSTANCE, 1, _frames((5, 160, 160, 1), 12), 2, capfd, monkeypatch)


@pytest.mark.parametrize("precision", [0, 2])
def test_audit_c3_centroid(precision, capfd, monkeypatch):
    """C3's centroid net (the C1 / C2 backbone): bilinear decoder, output stride 2, a 1-channel head, frames resized by
    0.5 in PREPROCESS (400 x 464 -> 200 x 232, padded to 208 x 240)."""
    _audit(C3_CENTROID, 1, _frames((2, 400, 464, 1), 13), precision, capfd, monkeypatch, input_scale=0.5)


@pytest.mark.parametrize("case", ["autotuned", "streaming", "precision2"])
def test_audit_c5_hourglass(case, capfd, monkeypatch):
    """C5's hourglass at full width on one 176 x 232 RGB frame: the stem runs on a frame padded to 192 x 256 and the
    tiles of every stride are partial."""
    env = {"SB_FORCE_VARIANT": "0"} if case == "streaming" else {}
    _audit(C5_HOURGLASS, 3, _frames((1, 176, 232, 3), 14), 2 if case == "precision2" else 0, capfd, monkeypatch, env)


@pytest.mark.parametrize("precision", [0, 2])
def test_audit_unet_rate15(precision, capfd, monkeypatch):
    _audit(UNET_RATE15, 1, _frames((2, 200, 232, 1), 15), precision, capfd, monkeypatch)


FIXTURE_FRAMES = {"minimal_instance": "minimal_instance", "min_tracks_2node": "tracks_2node", "minimal_robot": "robot"}


def _fixture_case(name):
    """(spec, weights, in_ch, input_scale, frames): the committed frames of the fixture's dataset; for a centered-instance
    model the window around the first ground-truth instance that the model sees as a crop_size crop after input scaling."""
    cfg, spec, w, in_ch = rm.load_fixture_model(name)
    scale = float(cfg["data"]["preprocessing"].get("input_scaling") or 1.0)
    imgs, gt = rm.frames(FIXTURE_FRAMES[name.split(".")[0]])
    if spec["head_type"] in ("centered_instance", "multi_class_topdown"):
        side = int(round(cfg["data"]["instance_cropping"]["crop_size"] / scale))
        cy, cx = (int(round(float(v))) for v in np.nanmean(gt[0, 0], axis=0)[::-1])
        y0 = min(max(cy - side // 2, 0), imgs.shape[1] - side)
        x0 = min(max(cx - side // 2, 0), imgs.shape[2] - side)
        imgs = np.ascontiguousarray(imgs[:1, y0:y0 + side, x0:x0 + side])
    return spec, w, in_ch, scale, imgs


@pytest.mark.parametrize("precision", [0, 1, 2])
@pytest.mark.parametrize("name", ["minimal_instance.bottomup", "minimal_instance.centroid", "minimal_instance.centered_instance",
                                  "minimal_instance.centered_instance_with_scaling", "minimal_robot.single_instance",
                                  "min_tracks_2node.bottomup_multiclass", "min_tracks_2node.topdown_multiclass"])
def test_audit_trained_fixture(name, precision, capfd, monkeypatch):
    """Trained weights on real frames: odd widths (filters_rate 1.5), their concat offsets, bilinear decoders."""
    spec, w, in_ch, scale, imgs = _fixture_case(name)
    _audit(spec, in_ch, imgs, precision, capfd, monkeypatch, input_scale=scale, weights=w)


BILINEAR_RGB = dict(backbone="unet", backbone_cfg=_unet(16, 16, 2), head_type="multi_instance", part_names=None, edges=None,
                    heads=[dict(name="MultiInstanceConfmapsHead", channels=6, output_stride=2),
                           dict(name="PartAffinityFieldsHead", channels=10, output_stride=4)])
HOURGLASS = dict(backbone="hourglass", head_type="multi_instance", part_names=None, edges=None,
                 backbone_cfg=dict(stem_stride=4, max_stride=32, output_stride=4, stem_filters=16, filters=32, filter_increase=32, stacks=2),
                 heads=[dict(name="MultiInstanceConfmapsHead", channels=6, output_stride=4),
                        dict(name="PartAffinityFieldsHead", channels=10, output_stride=4)])
LEAP = dict(backbone="leap", backbone_cfg=dict(max_stride=8, output_stride=2, filters=16, filters_rate=2, up_interpolate=False, stacks=1),
            head_type="multi_instance", part_names=None, edges=None,
            heads=[dict(name="MultiInstanceConfmapsHead", channels=5, output_stride=2),
                   dict(name="PartAffinityFieldsHead", channels=8, output_stride=4)])


@pytest.mark.parametrize("model", ["c4", "unet_bilinear_resized_rgb", "hourglass", "resnet50_tconv_concat",
                                   "resnet50_interp_add", "leap"])
def test_audit_precision1(model, capfd, monkeypatch):
    """The fp32 CUDA-core path (the strict reference of bench.c4_parity and the full-size tests), on the networks and
    frames of test_gpu_layer_audit.py.  Nothing is fused in precision 1, so both runs fetch every buffer."""
    spec, in_ch, imgs, scale = {
        "c4": (_c4(), 1, _frames((3, 200, 232, 1), 1), 1.0),
        "unet_bilinear_resized_rgb": (BILINEAR_RGB, 1, _frames((2, 300, 346, 3), 3), 0.5),
        "hourglass": (HOURGLASS, 3, _frames((2, 120, 136, 3), 5), 1.0),
        "resnet50_tconv_concat": (_resnet("tconv_concat"), 3, _frames((2, 150, 176, 3), 4), 1.0),
        "resnet50_interp_add": (_resnet("interp_add"), 3, _frames((1, 150, 176, 3), 4), 1.0),
        "leap": (LEAP, 1, _frames((3, 96, 112, 1), 6), 1.0)}[model]
    rows = _audit(spec, in_ch, imgs, 1, capfd, monkeypatch, input_scale=scale)
    assert {r["out"] for r in rows} <= {"f32", "exact"}
    assert {r["engine"] for r in rows if r["steps"]} == {"cuda"}
    print(f"== {model} p1: largest worst = {max(r['worst'] for r in rows):.3g}")
