"""ResNet / LEAP backbones on the host: graph compiler structure against the reference's known answers
(tests/nn/architectures/test_resnet.py, test_leap.py), training_config.json dispatch, the BatchNormalization fold,
and the oracle's output shapes.  No GPU."""
import numpy as np
import pytest
import torch

import backbone_oracle as bo
from oracle.convnet import conv2d_same
from sleap_b200.nn import architectures as A
from sleap_b200.nn import oplist as ol


def _resnet(version="ResNet50", weights="random", max_stride=32, up=None, output_stride=None):
    os_ = output_stride or max_stride
    return dict(backbone="resnet", backbone_cfg=dict(version=version, weights=weights, max_stride=max_stride, output_stride=os_,
                                                     upsampling=up),
                head_type="x", heads=[dict(name="H", channels=1, output_stride=os_)], part_names=None, edges=None)


def _counts(cm, head_cin):
    total = A.count_params(cm) - (head_cin + 1)            # minus the 1x1 head
    bn = sum(L["c"] for L in cm.layers if L["kind"] == "bn")
    return total - 2 * bn, total                            # trainable (moving mean / var excluded), total


@pytest.mark.parametrize("version,weights,trainable,total", [
    ("ResNet50", "random", 23528320, 23581440), ("ResNet50", "frozen", 23534592, 23587712),
    ("ResNet101", "random", 42546560, 42651904), ("ResNet152", "random", 58213248, 58364672)])
def test_resnet_param_counts(version, weights, trainable, total):
    cm = A.compile_model(_resnet(version, weights), 1)
    assert _counts(cm, 2048) == (trainable, total)


def test_resnet_strides_and_layer_names():
    cm = A.compile_model(_resnet(), 1)
    names = [L["name"] for L in cm.layers]
    for n in ("conv1_conv", "conv1_bn", "conv2_block1_0_conv", "conv2_block3_3_bn", "conv4_block6_3_bn", "conv5_block3_3_conv"):
        assert n in names
    bufs = {int(r[1]): int(r[2]) for r in cm.records if r[0] == ol.BUFFER}
    assert max(bufs.values()) == 32
    # max_stride 16: conv5 keeps stride 1 (its dilation reaches only 1x1 convs and is dropped)
    cm16 = A.compile_model(_resnet(max_stride=16), 1)
    assert max(int(r[2]) for r in cm16.records if r[0] == ol.BUFFER) == 16
    assert _counts(cm16, 2048) == _counts(cm, 2048)


def test_resnet_oracle_shapes():
    spec = _resnet()
    w = A.make_synthetic_weights(A.compile_model(spec, 1), 0)
    x = torch.zeros((1, 1, 160, 160))
    out, feats, st = bo.resnet_forward(x, spec["backbone_cfg"], w)
    assert tuple(out.shape) == (1, 2048, 5, 5) and st == 32
    spec16 = _resnet(max_stride=16)
    out16, _, _ = bo.resnet_forward(x, spec16["backbone_cfg"], w)
    assert tuple(out16.shape) == (1, 2048, 10, 10)
    up = dict(method="transposed_conv", skip_connections=None, block_stride=2, filters=64, filters_rate=1, refine_convs=2,
              batch_norm=True, transposed_conv_kernel_size=4)
    specu = _resnet(up=up, output_stride=4)
    wu = A.make_synthetic_weights(A.compile_model(specu, 1), 0)
    outu, mids, stu = bo.resnet_forward(x, specu["backbone_cfg"], wu)
    assert tuple(outu.shape) == (1, 64, 40, 40) and stu == 4 and [s for _, s in mids] == [32, 16, 8, 4]


def test_leap_param_counts_and_shape():
    spec = dict(backbone="leap", backbone_cfg=dict(max_stride=8, output_stride=1, filters=64, filters_rate=2, up_interpolate=False),
                head_type="x", heads=[dict(name="H", channels=1, output_stride=1)], part_names=None, edges=None)
    cm = A.compile_model(spec, 1)
    assert A.count_params(cm) - (128 + 1) == 10768896
    assert "stack0_dec0_s8_to_s4_trans_conv" in [L["name"] for L in cm.layers]
    w = A.make_synthetic_weights(cm, 0)
    out, mids, st = bo.leap_forward(torch.zeros((1, 1, 192, 192)), spec["backbone_cfg"], w)
    assert tuple(out.shape) == (1, 128, 192, 192) and len(mids) == 3
    spec_i = dict(spec, backbone_cfg=dict(max_stride=8, output_stride=1, filters=8, filters_rate=2, up_interpolate=True))
    assert A.count_params(A.compile_model(spec_i, 1)) - (16 + 1) == 120272


def _cfg(backbone, bcfg):
    bb = {"unet": None, "hourglass": None, "resnet": None, "leap": None, "pretrained_encoder": None}
    bb[backbone] = bcfg
    heads = {"multi_instance": {"confmaps": {"part_names": list("abc"), "output_stride": 4},
                                "pafs": {"edges": [["a", "b"], ["b", "c"]], "output_stride": 8}},
             "single_instance": None, "centroid": None, "centered_instance": None}
    return {"backbone": bb, "heads": heads}


def test_spec_from_config_resnet_leap_and_pretrained_encoder():
    up = dict(method="transposed_conv", skip_connections="concatenate", block_stride=2, filters=64, filters_rate=1,
              refine_convs=2, batch_norm=True, transposed_conv_kernel_size=4)
    spec = A.spec_from_config(_cfg("resnet", dict(version="ResNet50", weights="frozen", upsampling=up, max_stride=32, output_stride=4)))
    assert spec["backbone"] == "resnet" and [h["output_stride"] for h in spec["heads"]] == [4, 8]
    assert [h["channels"] for h in spec["heads"]] == [3, 4]
    cm = A.compile_model(spec, 3)
    assert cm.max_stride == 32 and cm.head_strides == {"MultiInstanceConfmapsHead": 4, "PartAffinityFieldsHead": 8}
    pre = next(r for r in cm.records if r[0] == ol.PREPROCESS)
    assert pre[19] == ol.PRE_IMAGENET_CAFFE and pre[8] == 3           # 3-channel caffe-normalised network input
    # trained on grayscale frames (1-channel Keras input): colour frames are converted to gray before tile_channels
    pre = next(r for r in A.compile_model(spec, 1).records if r[0] == ol.PREPROCESS)
    assert pre[19] == ol.PRE_IMAGENET_CAFFE_GRAY and pre[8] == 3
    spec = A.spec_from_config(_cfg("leap", dict(max_stride=16, output_stride=4, filters=16, filters_rate=2, up_interpolate=True)))
    assert spec["backbone"] == "leap" and A.compile_model(spec, 1).max_stride == 16
    with pytest.raises(ValueError, match="pretrained_encoder"):
        A.spec_from_config(_cfg("pretrained_encoder", dict(encoder="efficientnetb0")))
    bad = dict(up, block_stride=4)
    with pytest.raises(ValueError, match="block_stride"):
        A.compile_model(A.spec_from_config(_cfg("resnet", dict(version="ResNet50", weights="random", upsampling=bad,
                                                                max_stride=32, output_stride=4))), 1)


def test_records_stem_pool_residual_tconv():
    up = dict(method="transposed_conv", skip_connections="add", block_stride=2, filters=64, filters_rate=1, refine_convs=1,
              batch_norm=True, transposed_conv_kernel_size=4)
    cm = A.compile_model(_resnet(up=up, output_stride=4), 1)
    convs = [r for r in cm.records if r[0] == ol.CONV]
    stem = convs[0]
    assert stem[9] == 7 and stem[10] == 2 and stem[11] & ol.F_EXPLICIT_PAD and (stem[16], stem[17]) == (3, 3)
    assert any(r[0] == ol.POOL and r[9] == 3 for r in cm.records)
    assert all(r[9] == 4 for r in cm.records if r[0] == ol.TCONV)
    # every bottleneck's last 1x1 conv carries its shortcut; the ADD after it is flagged, with the block's ReLU
    recs = list(cm.records)
    n_res = 0
    for i, r in enumerate(recs):
        if r[0] == ol.CONV and r[11] & ol.F_RESIDUAL:
            n_res += 1
            add = recs[i + 1]
            assert add[0] == ol.ADD and add[11] & ol.F_FUSED_ADD and (add[6], add[7]) == (r[22], r[23])
    assert n_res == 16 + 3          # 16 blocks + the three 1x1 projections of the add skips (1024 / 512 / 256 -> 64)


def test_bn_fold_equals_conv_then_bn():
    """Packed weights of a folded conv == the unfolded conv + BatchNormalization (oracle), within 1e-6 relative."""
    spec = _resnet(max_stride=32)
    cm = A.compile_model(spec, 1)
    rng = np.random.default_rng(0)
    w = A.make_synthetic_weights(cm, 1)
    for L in cm.layers:
        if L["kind"] == "bn":
            c = L["c"]
            w[L["name"]] = dict(gamma=rng.uniform(0.5, 1.5, c).astype(np.float32), beta=rng.normal(0, 0.3, c).astype(np.float32),
                                mean=rng.normal(0, 0.3, c).astype(np.float32), var=rng.uniform(0.2, 2.0, c).astype(np.float32))
        elif L["kind"] == "conv":
            w[L["name"]]["bias"] = rng.normal(0, 0.2, L["cout"]).astype(np.float32)
    blob = cm.pack_weights(w)
    x = torch.from_numpy(rng.normal(size=(1, 64, 12, 12)).astype(np.float32))
    for name, bn_name in (("conv2_block1_2_conv", "conv2_block1_2_bn"), ("conv2_block1_3_conv", "conv2_block1_3_bn")):
        L = next(l for l in cm.layers if l["name"] == name)
        slot = cm._w_slots[name]
        k = blob[slot["w"]:slot["w"] + L["k"] ** 2 * L["cin"] * L["cout"]].reshape(L["k"], L["k"], L["cin"], L["cout"])
        b = blob[slot["b"]:slot["b"] + L["cout"]]
        xi = x[:, :L["cin"]] if L["cin"] <= 64 else torch.cat([x] * (L["cin"] // 64), 1)
        want = bo.bn(conv2d_same(xi, w[name]["kernel"], w[name]["bias"], 1), w[bn_name], bo.RESNET_EPS)
        got = conv2d_same(xi, k, b, 1)
        assert (got - want).abs().max().item() <= 1e-5 * want.abs().max().item()     # fp32 sums in a different order
        assert np.abs(k - w[name]["kernel"] * (w[bn_name]["gamma"] / np.sqrt(w[bn_name]["var"] + np.float32(1.001e-5)))).max() \
            <= 1e-6 * np.abs(k).max()


def test_leap_stacked_needs_symmetric_encoder_decoder():
    """EncoderDecoder.make_backbone (encoder_decoder.py:633-639): stacks > 1 with output_stride != 1 is refused."""
    cfg = dict(max_stride=8, output_stride=2, filters=8, filters_rate=2, up_interpolate=True, stacks=2)
    spec = dict(backbone="leap", backbone_cfg=cfg, head_type="x", heads=[dict(name="H", channels=1, output_stride=2)],
                part_names=None, edges=None)
    with pytest.raises(ValueError, match="symmetric"):
        A.compile_model(spec, 1)
    spec["backbone_cfg"] = dict(cfg, output_stride=1)
    spec["heads"][0]["output_stride"] = 1
    assert A.compile_model(spec, 1).max_stride == 8
