"""Oracle forward pass of the ResNet (v1, with UpsamplingStack) and LEAP backbones (torch CPU float32).

Test infrastructure only, written from the reference source independently of the graph compiler:
  sleap/nn/architectures/resnet.py:88-702     make_resnet_model, block_v1, stack_v1, make_backbone_fn,
                                               tile_channels, imagenet_preproc_v1, ResNetv1.make_backbone
  sleap/nn/architectures/upsampling.py:90-259 UpsamplingStack.make_stack
  sleap/nn/architectures/leap.py:14-131       LeapCNN on encoder_decoder.EncoderDecoder
  sleap/nn/model.py:325-364                   head taps by output stride
BatchNormalization is applied as its own layer after the conv (not folded), so that comparing against the device
checks the compiler's fold.  Keras layer semantics: ZeroPadding2D + VALID convs / pools, Conv2DTranspose SAME,
UpSampling2D bilinear (half-pixel centres), BatchNormalization(epsilon).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle.convnet import _t, conv2d_same, conv2d_transpose_same, maxpool2_same, upsample2

RESNET_EPS = 1.001e-5
KERAS_EPS = 1e-3
CAFFE_MEAN_BGR = (103.939, 116.779, 123.68)
STACKS = {"ResNet50": (3, 4, 6, 3), "ResNet101": (3, 4, 23, 3), "ResNet152": (3, 8, 36, 3)}


def conv_valid(x, p, stride=1, pad=0):
    """ZeroPadding2D(pad) + Conv2D(padding='valid')."""
    if pad:
        x = F.pad(x, (pad, pad, pad, pad))
    b = p.get("bias")
    return F.conv2d(x, _t(p["kernel"]).permute(3, 2, 0, 1).contiguous(), None if b is None else _t(b), stride=stride)


def bn(x, p, eps):
    scale = _t(p["gamma"]) / torch.sqrt(_t(p["var"]) + eps)
    return (x - _t(p["mean"]).view(1, -1, 1, 1)) * scale.view(1, -1, 1, 1) + _t(p["beta"]).view(1, -1, 1, 1)


def maxpool3_zero_pad(x):
    """ZeroPadding2D(1) + MaxPooling2D(3, strides=2, padding='valid'): the padding value is 0, not -inf."""
    return F.max_pool2d(F.pad(x, (1, 1, 1, 1)), 3, 2)


def imagenet_caffe(x):
    """tile_channels (1 -> 3) + imagenet_preproc_v1: x * 255, RGB -> BGR, minus the caffe means."""
    if x.shape[1] == 1:
        x = x.repeat(1, 3, 1, 1)
    x = x * 255.0
    x = x.flip(1)
    return x - torch.tensor(CAFFE_MEAN_BGR, dtype=torch.float32).view(1, 3, 1, 1)


def resnet_forward(x, cfg, w):
    """ResNetv1.make_backbone -> (main output, intermediate features [(tensor, stride)], output stride)."""
    max_stride = cfg.get("max_stride", 32)
    if cfg.get("weights", "frozen") != "random":
        x = imagenet_caffe(x)

    def cb(t, name, stride=1, pad=0, relu=True):
        y = bn(conv_valid(t, w[name + "_conv"], stride, pad) if w[name + "_conv"]["kernel"].shape[0] != 3
               else conv2d_same(t, w[name + "_conv"]["kernel"], w[name + "_conv"].get("bias"), stride), w[name + "_bn"], RESNET_EPS)
        return F.relu(y) if relu else y

    feats = []
    x = cb(x, "conv1", stride=2, pad=3)
    feats.append((x, 2))
    x = maxpool3_zero_pad(x)
    feats.append((x, 4))
    cur = 4
    for si, (n_blocks, s1) in enumerate(zip(STACKS[cfg.get("version", "ResNet50")], (1, 2, 2, 2))):
        if cur < max_stride:
            cur *= s1
            stride = s1
        else:
            stride = 1                # dilated 1x1 convs: same as undilated
        for b in range(1, n_blocks + 1):
            name = f"conv{si + 2}_block{b}"
            st = stride if b == 1 else 1
            sc = cb(x, name + "_0", stride=st, relu=False) if b == 1 else x
            y = cb(x, name + "_1", stride=st)
            y = cb(y, name + "_2")
            y = cb(y, name + "_3", relu=False)
            x = F.relu(sc + y)
        feats.append((x, cur))
    up = cfg.get("upsampling")
    if not up:
        return x, feats, max_stride
    skips = feats[2:] if up.get("skip_connections") else []
    transposed = up.get("method", "interpolation") == "transposed_conv"
    filters, rate = up.get("filters", 64), up.get("filters_rate", 1)
    mids = [(x, max_stride)]
    cur = max_stride
    for blk in range(int(round(math.log2(max_stride / cfg["output_stride"])))):
        new = cur // 2
        pre = f"upsample_s{cur}_to_s{new}"
        if transposed:
            p = w[pre + "_trans_conv"]
            x = conv2d_transpose_same(x, p["kernel"], p.get("bias"), 2)
            if up.get("batch_norm", True):
                x = bn(x, w[pre + "_bn"], KERAS_EPS)
            x = F.relu(x)
        else:
            x = upsample2(x, "bilinear")
        cur = new
        for (t, st) in skips:
            if st == cur:
                if up["skip_connections"] == "add":
                    if t.shape[1] != x.shape[1]:
                        t = conv2d_same(t, w[pre + "_skip_conv1x1"]["kernel"], w[pre + "_skip_conv1x1"].get("bias"), 1)
                    x = t + x
                else:
                    x = torch.cat([t, x], dim=1)
                break
        for i in range(int(up.get("refine_convs", 2))):
            p = w[pre + f"_refine{i}_conv"]
            x = conv2d_same(x, p["kernel"], p.get("bias"), 1)
            if up.get("batch_norm", True):
                x = bn(x, w[pre + f"_refine{i}_bn"], KERAS_EPS)
            x = F.relu(x)
        mids.append((x, cur))
    return x, mids, cur


def leap_forward(x, cfg, w):
    filters, rate = cfg.get("filters", 64), cfg.get("filters_rate", 2)
    down = int(round(math.log2(cfg["max_stride"])))
    up = int(round(math.log2(cfg["max_stride"] / cfg["output_stride"])))
    cur = 1
    for i in range(down):
        for j in range(3):
            p = w[f"stack0_enc{i}_conv{j}"]
            x = F.relu(conv2d_same(x, p["kernel"], p.get("bias"), 1))
        x = maxpool2_same(x)
        cur *= 2
    mids = []
    for i in range(up):
        mids.append((x, cur))
        pre = f"stack0_dec{i}_s{cur}_to_s{cur // 2}"
        if cfg.get("up_interpolate", False):
            x = upsample2(x, "bilinear")
        else:
            p = w[pre + "_trans_conv"]
            x = F.relu(conv2d_transpose_same(x, p["kernel"], p.get("bias"), 2))
        for j in range(2):
            p = w[pre + f"_refine_conv{j}"]
            x = F.relu(conv2d_same(x, p["kernel"], p.get("bias"), 1))
        cur //= 2
    return x, mids, cur


def model_forward(images_nhwc, spec, weights):
    """Backbone + 1x1 linear heads (model.py:325-364) -> list of NHWC float32 arrays, one per head."""
    x = _t(images_nhwc).permute(0, 3, 1, 2).contiguous()
    with torch.no_grad():
        fwd = resnet_forward if spec["backbone"] == "resnet" else leap_forward
        main, mids, out_stride = fwd(x, spec["backbone_cfg"], weights)
        res = []
        for h in spec["heads"]:
            feat = main if h["output_stride"] == out_stride else next(t for (t, st) in mids if st == h["output_stride"])
            p = weights[h["name"]]
            res.append(conv2d_same(feat, p["kernel"], p.get("bias"), 1).permute(0, 2, 3, 1).contiguous().numpy())
    return res
