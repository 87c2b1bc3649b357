"""Host-side graph compiler: reference model config -> flat op-list + weight blob for libsleapb200.

Restates the *topology* (not the execution) of the reference's Keras graph builders:
  sleap/nn/architectures/unet.py:43-278          UNet block stacks and from_config
  sleap/nn/architectures/encoder_decoder.py:94-144, 275-399, 508-676
  sleap/nn/architectures/hourglass.py:17-305
  sleap/nn/architectures/resnet.py:88-702         ResNet50 / 101 / 152 (v1) with the UpsamplingStack decoder
  sleap/nn/architectures/upsampling.py:90-259
  sleap/nn/architectures/leap.py:14-131           LeapCNN
  sleap/nn/heads.py:42-63, sleap/nn/model.py:104-364 (head taps by output stride, output order)
Layer names follow the reference's Keras layer names so that weights exported from a
``best_model.h5`` map 1:1 (``{layer_name: {"kernel", "bias", ...}}``, Keras layouts).

Concatenated skip connections are realised by construction: the producer of each part writes
straight into its channel slice of the concat buffer, so no concat kernel exists.

Backbones: UNet, hourglass, ResNet (v1, ``resnet``) and LEAP (``leap``).  ``pretrained_encoder`` models are not
supported: their encoders are built by the third-party ``segmentation_models`` package, whose layer graph is not part
of the reference and so cannot be restated and checked here.
"""
import math
from typing import Dict, List, Optional

import numpy as np

from sleap_b200.nn import oplist as ol

BN_EPS = 1e-3  # Keras BatchNormalization default
RESNET_BN_EPS = 1.001e-5   # resnet.py: every BatchNormalization of the ResNet backbone
RESNET_STACKS = {"ResNet50": (3, 4, 6, 3), "ResNet101": (3, 4, 23, 3), "ResNet152": (3, 8, 36, 3)}
IMAGENET_CAFFE_MEAN_BGR = (103.939, 116.779, 123.68)   # resnet.py imagenet_preproc_v1

HEAD_CLASS_NAMES = {
    "single_instance": "SingleInstanceConfmapsHead",
    "centroid": "CentroidConfmapsHead",
    "centered_instance": "CenteredInstanceConfmapsHead",
    "multi_instance": "MultiInstanceConfmapsHead",
}


class _T:
    """Symbolic tensor."""
    __slots__ = ("id", "C", "stride", "f32", "buf", "coff", "name")

    def __init__(self, id, C, stride, f32=False, name=""):
        self.id, self.C, self.stride, self.f32, self.name = id, C, stride, f32, name
        self.buf, self.coff = None, 0


class GraphBuilder:
    def __init__(self):
        self.tensors: List[_T] = []
        self.sym_ops = []          # (kind, dict)
        self.layers = []           # (name, kind, shape info) for weight enumeration

    def tensor(self, C, stride, f32=False, name=""):
        t = _T(len(self.tensors), C, stride, f32, name)
        self.tensors.append(t)
        return t

    def conv(self, x, filters, k, name, stride=1, relu=True, bn=None, f32_out=False, bn_pre=None, bn_eps=BN_EPS, pad=None):
        """``bn``: BatchNormalization AFTER the ReLU (hourglass), applied as the epilogue affine.  ``bn_pre``:
        BatchNormalization BEFORE the ReLU (ResNet, upsampling stack), folded into the kernel and bias at pack time.
        ``pad``: explicit (top, left) zero padding (bottom / right follow from the output size), None = TF SAME."""
        y = self.tensor(filters, x.stride * stride, f32_out, name)
        self.sym_ops.append(("conv", dict(x=x, y=y, k=k, stride=stride, relu=relu, bn=bn, name=name, pad=pad)))
        self.layers.append(dict(name=name, kind="conv", k=k, cin=x.C, cout=filters))
        if bn:
            self.layers.append(dict(name=bn, kind="bn", c=filters, eps=BN_EPS))
        if bn_pre:
            self.layers[-1]["fold_bn"] = bn_pre
            self.layers.append(dict(name=bn_pre, kind="bn", c=filters, eps=bn_eps, folded=True))
        return y

    def tconv(self, x, filters, name, k=3, bn_pre=None, bn_eps=BN_EPS):
        y = self.tensor(filters, x.stride // 2, False, name)
        self.sym_ops.append(("tconv", dict(x=x, y=y, k=k, name=name)))
        self.layers.append(dict(name=name, kind="tconv", k=k, cin=x.C, cout=filters))
        if bn_pre:
            self.layers[-1]["fold_bn"] = bn_pre
            self.layers.append(dict(name=bn_pre, kind="bn", c=filters, eps=bn_eps, folded=True))
        return y

    def pool(self, x, name="pool", k=2):
        """k = 2: MaxPool2D(2, 2, SAME); k = 3: ZeroPadding2D(1) + MaxPool2D(3, 2) (ResNet stem)."""
        y = self.tensor(x.C, x.stride * 2, False, name)
        self.sym_ops.append(("pool", dict(x=x, y=y, k=k)))
        return y

    def upsample(self, x, bilinear, name="up"):
        y = self.tensor(x.C, x.stride // 2, False, name)
        self.sym_ops.append(("up", dict(x=x, y=y, bilinear=bilinear)))
        return y

    def add(self, a, b, name="add", relu=False):
        y = self.tensor(a.C, a.stride, False, name)
        self.sym_ops.append(("add", dict(a=a, b=b, y=y, relu=relu)))
        return y

    def concat(self, parts, name="concat"):
        y = self.tensor(sum(p.C for p in parts), parts[0].stride, False, name)
        self.sym_ops.append(("concat", dict(parts=list(parts), y=y)))
        return y


# ------------------------------------------------------------------------------------------
def unet_blocks(cfg):
    """UNet.from_config (unet.py:250-278)."""
    stem_blocks = 0
    if cfg.get("stem_stride"):
        stem_blocks = int(math.log2(cfg["stem_stride"]))
    down_blocks = int(math.log2(cfg["max_stride"])) - stem_blocks
    up_blocks = int(math.log2(cfg["max_stride"] / cfg["output_stride"]))
    return stem_blocks, down_blocks, up_blocks


def build_unet(g: GraphBuilder, x: _T, cfg):
    """Returns (outputs per stack, intermediate decoder features per stack, output stride)."""
    filters, rate = cfg["filters"], cfg.get("filters_rate", 2)
    convs = cfg.get("convs_per_block", 2)
    middle = cfg.get("middle_block", True)
    interp = cfg.get("up_interpolate", False)
    contraction = cfg.get("block_contraction", False)
    stacks = cfg.get("stacks", 1)
    ksz = cfg.get("kernel_size", 3)
    stem_k = cfg.get("stem_kernel_size", 7)
    stem_blocks, down_blocks, up_blocks = unet_blocks(cfg)

    stem_output = []
    if stem_blocks > 0:
        for b in range(stem_blocks):
            bf = int(filters * rate ** b)
            if b > 0:
                x = g.pool(x, f"stem{b}_pool")
            for i in range(convs):
                x = g.conv(x, bf, stem_k, f"stem{b}_conv{i}")
        x = g.pool(x, f"stem{stem_blocks}_last_pool")
        stem_output = [x]
    stem_stride = x.stride

    outs, mids = [], []
    for s in range(stacks):
        feats = []

        def note(t):
            if t.stride not in [f.stride for f in feats]:
                feats.append(t)

        bi = 0
        for b in range(down_blocks):
            bf = int(filters * rate ** (b + stem_blocks))
            if b > 0:
                x = g.pool(x, f"stack{s}_enc{bi}_pool")
            for i in range(convs):
                x = g.conv(x, bf, ksz, f"stack{s}_enc{bi}_conv{i}")
            note(x)
            bi += 1
        x = g.pool(x, f"stack{s}_enc{bi}_last_pool")
        note(x)
        bi += 1
        if middle:
            if convs > 1:
                bf = int(filters * rate ** (down_blocks + stem_blocks))
                for i in range(convs - 1):
                    x = g.conv(x, bf, ksz, f"stack{s}_enc{bi}_middle_expand_conv{i}")
                note(x)
                bi += 1
            bf = int(filters * rate ** (down_blocks + stem_blocks - (1 if contraction else 0)))
            x = g.conv(x, bf, ksz, f"stack{s}_enc{bi}_middle_contract_conv0")
            note(x)
            bi += 1
        skips = stem_output + feats[:-1]

        inter = []
        for b in range(up_blocks):
            inter.append(x)
            cur, nxt = x.stride, x.stride // 2
            f_in = int(filters * rate ** (down_blocks + stem_blocks - 1 - b))
            f_out = int(filters * rate ** (down_blocks + stem_blocks - 2 - b)) if contraction else f_in
            prefix = f"stack{s}_dec{b}_s{cur}_to_s{nxt}"
            if interp:
                x = g.upsample(x, True, prefix + "_interp_bilinear")
            else:
                x = g.tconv(x, f_in, prefix + "_trans_conv")
            skip = next((t for t in skips if t.stride == nxt), None)
            if skip is not None:
                x = g.concat([skip, x], prefix + "_skip_concat")
            for i in range(convs):
                x = g.conv(x, f_in if i == 0 else f_out, ksz, prefix + f"_refine_conv{i}")
        outs.append(x)
        mids.append(inter)
    return outs, mids


def build_hourglass(g: GraphBuilder, x: _T, cfg):
    stem_stride = cfg.get("stem_stride", 4)
    stem_blocks = int(math.log2(stem_stride))
    down_blocks = int(math.log2(cfg.get("max_stride", 64))) - stem_blocks
    up_blocks = int(math.log2(cfg.get("max_stride", 64) / cfg.get("output_stride", 4)))
    stem_filters = cfg.get("stem_filters", 128)
    filters = cfg.get("filters", 256)
    inc = cfg.get("filter_increase", 128)
    stacks = cfg.get("stacks", 3)

    def cbn(t, f, prefix, k=3, stride=1):   # hourglass.conv: Conv2D(relu) -> BatchNormalization
        return g.conv(t, f, k, prefix + "_conv", stride=stride, relu=True, bn=prefix + "_bn")

    x = cbn(x, stem_filters, "stem0_conv7x7", k=7, stride=2 if stem_stride == 4 else 1)
    x = cbn(x, 2 * stem_filters, "stem0_conv3x3")
    if stem_stride > 1:
        x = g.pool(x, "stem0_pool")
    x = cbn(x, filters, "stem0_conv3x3_out")
    stem_output = [x]
    outs, mids = [], []
    for s in range(stacks):
        feats = []
        for b in range(down_blocks):
            x = g.pool(x, f"stack{s}_enc{b}_pool")
            x = cbn(x, filters + b * inc, f"stack{s}_enc{b}_conv")
            if x.stride not in [f.stride for f in feats]:
                feats.append(x)
        skips = stem_output + feats[:-1]
        inter = []
        for b in range(up_blocks):
            inter.append(x)
            nxt = x.stride // 2
            f = filters + (down_blocks - b - 1) * inc
            prefix = f"stack{s}_dec{b}"
            skip = next(t for t in skips if t.stride == nxt)
            x = cbn(x, f, prefix + "_conv")
            x = g.upsample(x, False, prefix + "_nearest")
            xs = cbn(skip, f, prefix + "_skip")
            x = g.add(x, xs, prefix + "_skip_add")
        outs.append(x)
        mids.append(inter)
    return outs, mids


def build_resnet(g: GraphBuilder, x: _T, cfg):
    """ResNetv1.make_backbone (resnet.py): stem, stacks of bottleneck blocks (block_v1 / stack_v1), optional
    UpsamplingStack.  Layer names are the flat Keras names (``conv1_conv``, ``conv2_block1_0_conv``, ...)."""
    version = cfg.get("version", "ResNet50")
    if version not in RESNET_STACKS:
        raise ValueError(f"Invalid ResNet version in the configuration: {version}")
    max_stride = int(cfg.get("max_stride", 32))
    if max_stride not in (4, 8, 16, 32):
        raise ValueError(f"ResNet max_stride must be 4, 8, 16 or 32, got {max_stride}.")
    eps = RESNET_BN_EPS

    def cbn(t, f, k, name, stride=1, relu=True, pad=None):
        return g.conv(t, f, k, name + "_conv", stride=stride, relu=relu, bn_pre=name + "_bn", bn_eps=eps, pad=pad)

    # stem: ZeroPadding2D(3) + Conv2D(7, s2, VALID) -- 3|3 padding, not SAME's 2|3 -- BN, ReLU; then ZeroPadding2D(1) +
    # MaxPooling2D(3, s2, VALID)
    x = cbn(x, 64, 7, "conv1", stride=2, pad=(3, 3))
    feats = [x]
    x = g.pool(x, "pool1_pool", k=3)
    feats.append(x)

    def block(t, filters, stride, shortcut, name):
        # the 1x1 convs are VALID; with kernel 1 and an even input (every buffer is a multiple of the stride) VALID and
        # SAME coincide: padding 0|0
        sc = cbn(t, 4 * filters, 1, name + "_0", stride=stride, relu=False, pad=(0, 0)) if shortcut else t
        y = cbn(t, filters, 1, name + "_1", stride=stride, pad=(0, 0))
        y = cbn(y, filters, 3, name + "_2")
        y = cbn(y, 4 * filters, 1, name + "_3", relu=False)
        return g.add(sc, y, name + "_add", relu=True)

    cur = 4
    for si, (filters, n_blocks, stride1) in enumerate(zip((64, 128, 256, 512), RESNET_STACKS[version], (1, 2, 2, 2))):
        if cur < max_stride:
            cur *= stride1
        else:
            # make_backbone_fn: the stack's stride becomes 1 and its dilation_rate doubles.  The dilation only reaches the
            # first block's 1x1 convs (_0_conv, _1_conv), where it has no effect, so it is dropped here.
            stride1 = 1
        for b in range(1, n_blocks + 1):
            x = block(x, filters, stride1 if b == 1 else 1, b == 1, f"conv{si + 2}_block{b}")
        feats.append(x)

    up = cfg.get("upsampling")
    if not up:
        return [x], [feats]
    if int(up.get("block_stride", 2)) != 2:
        raise ValueError("Upsampling block_stride other than 2 is not supported.")
    transposed = up.get("method", "interpolation") == "transposed_conv"
    skip_mode = up.get("skip_connections")
    filters, rate = up.get("filters", 64), up.get("filters_rate", 1)
    refine, bn, tk = int(up.get("refine_convs", 2)), bool(up.get("batch_norm", True)), int(up.get("transposed_conv_kernel_size", 4))
    if transposed and tk not in (3, 4):
        raise ValueError(f"Transposed convolution kernel size {tk} is not supported (3 or 4).")
    skip_sources = feats[2:] if skip_mode else []          # the stack outputs (intermediate_feats[2:])
    mids = [x]
    cur = max_stride
    n_up = int(round(math.log2(max_stride / cfg["output_stride"])))
    for blk in range(n_up):
        new = cur // 2
        prefix = f"upsample_s{cur}_to_s{new}"
        f = int(filters * rate ** blk)
        if transposed:
            # Conv2DTranspose -> (BatchNormalization, Keras default eps) -> ReLU: BN folded, ReLU in the epilogue
            x = g.tconv(x, f, prefix + "_trans_conv", k=tk, bn_pre=prefix + "_bn" if bn else None)
        else:
            x = g.upsample(x, True, prefix + "_interp")
        cur = new
        skip = next((t for t in skip_sources if t.stride == cur), None)
        if skip is not None:
            if skip_mode == "add":
                src = skip if skip.C == x.C else g.conv(skip, x.C, 1, prefix + "_skip_conv1x1", relu=False)
                x = g.add(src, x, prefix + "_skip_add")
            else:
                x = g.concat([skip, x], prefix + "_skip_concat")
        for i in range(refine):
            x = g.conv(x, f, 3, prefix + f"_refine{i}_conv", bn_pre=prefix + f"_refine{i}_bn" if bn else None)
        mids.append(x)
    return [x], [mids]


def build_leap(g: GraphBuilder, x: _T, cfg):
    """LeapCNN.from_config (leap.py) on EncoderDecoder: 3 convs + 2x2 max-pool per down block, transposed conv k3 s2
    (or bilinear x2) + 2 refine convs per up block, no skip connections."""
    filters, rate = cfg.get("filters", 64), cfg.get("filters_rate", 2)
    down = int(round(math.log2(cfg["max_stride"])))
    up = int(round(math.log2(cfg["max_stride"] / cfg["output_stride"])))
    interp = cfg.get("up_interpolate", False)
    if cfg.get("stacks", 1) > 1 and cfg["output_stride"] != 1:       # EncoderDecoder.make_backbone (encoder_decoder.py:633-639)
        raise ValueError("If using a stacked configuration, the backbone must define symmetric encoder and decoder. "
                         "Create a stem for initial downsampling if an output stride > 1 is desired.")
    outs, mids = [], []
    for s in range(cfg.get("stacks", 1)):
        for i in range(down):
            for j in range(3):
                x = g.conv(x, int(filters * rate ** i), 3, f"stack{s}_enc{i}_conv{j}")
            x = g.pool(x, f"stack{s}_enc{i}_pool")
        inter = []
        for i, e in enumerate(range(up, 0, -1)):
            inter.append(x)
            f = int(filters * rate ** e)
            prefix = f"stack{s}_dec{i}_s{x.stride}_to_s{x.stride // 2}"
            x = g.upsample(x, True, prefix + "_interp_bilinear") if interp else g.tconv(x, f, prefix + "_trans_conv")
            for j in range(2):
                x = g.conv(x, f, 3, prefix + f"_refine_conv{j}")
        outs.append(x)
        mids.append(inter)
    return outs, mids


def resnet_pretrained(spec) -> bool:
    """``weights != "random"`` (the default "frozen" included): the graph starts with tile_channels (1 -> 3) and
    imagenet_preproc_v1."""
    return spec["backbone"] == "resnet" and spec["backbone_cfg"].get("weights", "frozen") != "random"


# ------------------------------------------------------------------------------------------
def spec_from_config(model_cfg: dict, skeleton_nodes=None, skeleton_edges=None):
    """``training_config.json["model"]`` -> internal spec.

    spec = {"backbone": "unet"|"hourglass"|"resnet"|"leap", "backbone_cfg": {...}, "head_type": str,
            "heads": [{"name", "channels", "output_stride"}...], "part_names", "edges"}
    Mirrors Model.from_config (model.py:104-305): head list order = [confmaps, pafs, (offsets)].
    """
    bb = {k: v for k, v in model_cfg["backbone"].items() if v is not None}
    if len(bb) != 1:
        raise ValueError("Backbone architecture (config.model.backbone) was not specified.")
    bname, bcfg = next(iter(bb.items()))
    if bname == "pretrained_encoder":
        raise ValueError("Backbone 'pretrained_encoder' is not supported: its encoder is built by the third-party "
                         "segmentation_models package, whose layer graph this library cannot restate and check.")
    if bname not in ("unet", "hourglass", "resnet", "leap"):
        raise ValueError(f"Backbone '{bname}' is outside the scope of this build (UNet / hourglass / ResNet / LEAP only).")
    hd = {k: v for k, v in model_cfg["heads"].items() if v is not None}
    if len(hd) != 1:
        raise ValueError("Head configuration (config.model.heads) was not specified.")
    htype, hcfg = next(iter(hd.items()))
    heads, part_names, edges = [], None, None
    if htype in ("single_instance", "centered_instance"):
        part_names = hcfg.get("part_names") or skeleton_nodes
        if part_names is None:
            raise ValueError("Skeleton must be provided when the head configuration is incomplete.")
        heads.append(dict(name=HEAD_CLASS_NAMES[htype], channels=len(part_names), output_stride=hcfg["output_stride"]))
        if hcfg.get("offset_refinement"):
            heads.append(dict(name="OffsetRefinementHead", channels=2 * len(part_names), output_stride=hcfg["output_stride"]))
    elif htype == "centroid":
        heads.append(dict(name=HEAD_CLASS_NAMES[htype], channels=1, output_stride=hcfg["output_stride"]))
        if hcfg.get("offset_refinement"):
            heads.append(dict(name="OffsetRefinementHead", channels=2, output_stride=hcfg["output_stride"]))
    elif htype == "multi_instance":
        cm, paf = hcfg["confmaps"], hcfg["pafs"]
        part_names = cm.get("part_names") or skeleton_nodes
        edges = paf.get("edges") or skeleton_edges
        if part_names is None or edges is None:
            raise ValueError("Skeleton must be provided when the head configuration is incomplete.")
        heads.append(dict(name="MultiInstanceConfmapsHead", channels=len(part_names), output_stride=cm["output_stride"]))
        heads.append(dict(name="PartAffinityFieldsHead", channels=2 * len(edges), output_stride=paf["output_stride"]))
        if cm.get("offset_refinement"):
            heads.append(dict(name="OffsetRefinementHead", channels=2 * len(part_names), output_stride=cm["output_stride"]))
    elif htype == "multi_class_topdown":                                    # model.py:258-296
        cm, cv = hcfg["confmaps"], hcfg["class_vectors"]
        part_names = cm.get("part_names") or skeleton_nodes
        classes = cv.get("classes")
        if part_names is None:
            raise ValueError("Skeleton must be provided when the head configuration is incomplete.")
        if classes is None:
            raise ValueError("Classes must be provided when the head configuration is incomplete.")
        heads.append(dict(name="CenteredInstanceConfmapsHead", channels=len(part_names), output_stride=cm["output_stride"]))
        # ClassVectorsHead (heads.py:431-460): global max pool / flatten -> Dense + ReLU x num_fc_layers -> Dense + softmax.
        # Not a convolution: the engine exposes the feature map it taps ("vector" head); its dense layers run in the fused
        # top-down multi-class step (k_class_vectors), or on the host after DeviceModel.forward
        heads.append(dict(name="ClassVectorsHead", channels=len(classes), output_stride=cv["output_stride"], vector=True,
                          num_fc_layers=int(cv.get("num_fc_layers", 1)), num_fc_units=int(cv.get("num_fc_units", 64)),
                          global_pool=bool(cv.get("global_pool", True))))
        if cm.get("offset_refinement"):
            heads.append(dict(name="OffsetRefinementHead", channels=2 * len(part_names), output_stride=cm["output_stride"]))
    elif htype == "multi_class_bottomup":                                   # model.py:219-256
        cm, cls_cfg = hcfg["confmaps"], hcfg["class_maps"]
        part_names = cm.get("part_names") or skeleton_nodes
        classes = cls_cfg.get("classes")
        if part_names is None:
            raise ValueError("Skeleton must be provided when the head configuration is incomplete.")
        if classes is None:
            raise ValueError("Classes must be provided when the head configuration is incomplete.")
        heads.append(dict(name="MultiInstanceConfmapsHead", channels=len(part_names), output_stride=cm["output_stride"]))
        # ClassMapsHead: 1x1 conv + sigmoid (heads.py:336-338); the sigmoid is applied by the inference layer
        heads.append(dict(name="ClassMapsHead", channels=len(classes), output_stride=cls_cfg["output_stride"], activation="sigmoid"))
        if cm.get("offset_refinement"):
            heads.append(dict(name="OffsetRefinementHead", channels=2 * len(part_names), output_stride=cm["output_stride"]))
    else:
        raise ValueError(f"Head type '{htype}' is outside the scope of this build.")
    bcfg = dict(bcfg)
    bcfg["output_stride"] = heads[0]["output_stride"]     # model.py:301
    spec = dict(backbone=bname, backbone_cfg=bcfg, head_type=htype, heads=heads,
                part_names=list(part_names) if part_names else None,
                edges=[tuple(e) for e in edges] if edges else None)
    if htype == "multi_class_bottomup":
        spec["classes"] = list(hcfg["class_maps"]["classes"])
    if htype == "multi_class_topdown":
        spec["classes"] = list(hcfg["class_vectors"]["classes"])
    return spec


class CompiledModel:
    """Result of ``compile_model``: the op-list records + layer table (+ weights once packed)."""

    def __init__(self):
        self.records = []            # list of int32[SB_OP_WORDS]
        self.layers = []             # weight-bearing layers in graph order
        self.n_buffers = 0
        self.input_buffer = 0
        self.head_buffers: Dict[str, int] = {}
        self.head_strides: Dict[str, int] = {}
        self.vector_taps: Dict[str, dict] = {}    # "vector" heads: the feature map they read (buffer, channel offset, C, planes)
        self.input_channels = 1
        self.max_stride = 1
        self.spec = None
        self._w_slots = {}           # layer name -> dict of blob offsets
        self.n_weights = 0
        self.flops_per_pixel = 0.0   # conv MACs*2 per network-input pixel (for rooflines)

    def ops_array(self):
        return np.ascontiguousarray(np.stack(self.records).astype(np.int32))

    def folded_kernel_bias(self, L, weights):
        """Kernel (kh, kw, Cin, Cout) and bias of a conv / transposed conv in float32, with a BatchNormalization that
        follows it before the activation folded in: W' = W * s, b' = b * s + t (s, t: bn_affine)."""
        p = weights[L["name"]]
        kern = np.asarray(p["kernel"], np.float32)
        if L["kind"] == "tconv":
            kern = np.transpose(kern, (0, 1, 3, 2))     # (kh,kw,Cout,Cin) -> (kh,kw,Cin,Cout)
        assert kern.shape == (L["k"], L["k"], L["cin"], L["cout"]), (L["name"], kern.shape)
        bias = p.get("bias")
        bias = np.zeros((L["cout"],), np.float32) if bias is None else np.asarray(bias, np.float32)
        if L.get("fold_bn"):
            bn = next(B for B in self.layers if B["name"] == L["fold_bn"])
            scale, shift = bn_affine(weights[bn["name"]], bn["eps"])
            kern = (kern * scale).astype(np.float32)
            bias = (bias * scale + shift).astype(np.float32)
        return kern, bias

    def pack_weights(self, weights: Dict[str, Dict[str, np.ndarray]]) -> np.ndarray:
        """Keras-layout weights dict -> flat float32 blob in the kernel layouts.  BatchNormalization layers before an
        activation are folded into the conv before them (before precision 2's hi / lo split of the weights)."""
        blob = np.zeros((self.n_weights,), np.float32)
        for L in self.layers:
            if L.get("folded"):
                continue
            slot = self._w_slots[L["name"]]
            p = weights[L["name"]]
            if L["kind"] in ("conv", "tconv"):
                kern, bias = self.folded_kernel_bias(L, weights)
                if "expand" in L:        # precision 2: input rows in the physical order of the split input, [Wh | Wl | Wh]
                    src, part = L["expand"]
                    wh = kern.astype(np.float16).astype(np.float32)
                    wl = (kern - wh).astype(np.float16).astype(np.float32)
                    kern = np.where((part == 1)[None, None, :, None], wl[:, :, src, :], wh[:, :, src, :])
                blob[slot["w"]:slot["w"] + kern.size] = kern.reshape(-1)
                blob[slot["b"]:slot["b"] + L["cout"]] = bias
            else:  # bn -> affine (scale, shift), exact Keras inference formula
                scale, shift = bn_affine(p, L["eps"])
                blob[slot["scale"]:slot["scale"] + L["c"]] = scale
                blob[slot["shift"]:slot["shift"] + L["c"]] = shift
        return blob


def bn_affine(p, eps):
    """BatchNormalization (inference) as a per-channel affine: scale = gamma / sqrt(var + eps), shift = beta - mean * scale."""
    scale = (np.asarray(p["gamma"], np.float32) / np.sqrt(np.asarray(p["var"], np.float32) + np.float32(eps))).astype(np.float32)
    shift = (np.asarray(p["beta"], np.float32) - np.asarray(p["mean"], np.float32) * scale).astype(np.float32)
    return scale, shift


def _compile_identity(spec: dict, input_channels: int, input_scale: float, pad_to_stride: Optional[int]) -> CompiledModel:
    """``backbone="identity"``: the network is ``Lambda(lambda x: x)`` named after the head, as in the reference's
    layer tests (tests/nn/test_inference.py:218-220, 270-274, 556-558): the preprocessed frame IS the head output.
    One float32 buffer, one PREPROCESS op; only meaningful with the fp32 precision path."""
    cm = CompiledModel()
    head = spec["heads"][0]
    if head["channels"] != input_channels:
        raise ValueError("identity backbone: head channels must equal the input channels")
    cm.records = [ol.buffer_record(0, 1, input_channels, 1, 1), ol.preprocess_record(0, input_channels, float(input_scale), int(pad_to_stride or 1))]
    cm.n_buffers = 1
    cm.head_buffers = {head["name"]: 0}
    cm.head_strides = {head["name"]: 1}
    cm.spec, cm.input_channels, cm.max_stride = spec, input_channels, int(pad_to_stride or 1)
    cm.n_weights = 1                                  # the C-ABI wants a non-empty weight blob
    return cm


def compile_model(spec: dict, input_channels: int, input_scale: float = 1.0, pad_to_stride: Optional[int] = None,
                  split: bool = False) -> CompiledModel:
    """``split=True`` lays the graph out for precision 2 (split-fp16 activations on the tensor cores): every fp16 tensor of
    C channels occupies 3C physical channels [lo | hi | hi] (csrc/sb_kernels_direct.cuh: st_split), the preprocessed
    frame stays fp32, and ``pack_weights`` expands every consumer conv's input rows to [Wh | Wl | Wh] in the physical
    channel order of its input (concat buffers interleave the triples of their parts).  Records carry physical
    channel counts / offsets, except ``out_C`` of CONV / TCONV which stays the GEMM N (logical C_out)."""
    if spec["backbone"] == "identity":
        return _compile_identity(spec, input_channels, input_scale, pad_to_stride)
    g = GraphBuilder()
    net_c = input_channels
    pre_mode = ol.PRE_PLAIN
    if resnet_pretrained(spec):
        # tile_channels + imagenet_preproc_v1: the buffer after PREPROCESS has 3 caffe-normalised BGR channels.
        # ``input_channels`` is the channel count of the model's Keras input (its training frames): 1 -> colour frames
        # are converted to gray and the gray plane is tiled (PRE_IMAGENET_CAFFE_GRAY); 3 -> grayscale frames are tiled.
        net_c = 3
        pre_mode = ol.PRE_IMAGENET_CAFFE_GRAY if input_channels == 1 else ol.PRE_IMAGENET_CAFFE
    x0 = g.tensor(net_c, 1, False, "input")
    if spec["backbone"] == "unet":
        outs, mids = build_unet(g, x0, spec["backbone_cfg"])
        max_stride = spec["backbone_cfg"]["max_stride"]
    elif spec["backbone"] == "resnet":
        outs, mids = build_resnet(g, x0, spec["backbone_cfg"])
        max_stride = int(spec["backbone_cfg"].get("max_stride", 32))
    elif spec["backbone"] == "leap":
        outs, mids = build_leap(g, x0, spec["backbone_cfg"])
        max_stride = spec["backbone_cfg"]["max_stride"]
    else:
        outs, mids = build_hourglass(g, x0, spec["backbone_cfg"])
        max_stride = spec["backbone_cfg"].get("max_stride", 64)
    out_stride = outs[-1].stride
    # heads on the LAST stack only (inference.py:2885-2888; SURVEY Appendix A.15)
    head_t, vec_t = {}, {}
    for hd in spec["heads"]:
        if hd["output_stride"] == out_stride:
            feat = outs[-1]
        else:
            feat = next((t for t in mids[-1] if t.stride == hd["output_stride"]), None)
            if feat is None:
                raise ValueError(f"Could not find a feature activation for output at stride {hd['output_stride']}.")
        if hd.get("vector"):
            vec_t[hd["name"]] = feat
            continue
        head_t[hd["name"]] = g.conv(feat, hd["channels"], 1, hd["name"], relu=False, f32_out=True)

    # ---- placement: concat parts become slices of the concat buffer ----
    bufs = []   # (C, stride, f32)

    def new_buf(C, stride, f32):
        bufs.append((C, stride, f32))
        return len(bufs) - 1

    if split:
        x0.f32 = True            # the preprocessed frame stays fp32 (first conv on the CUDA cores, exact)

    def pc(t):                   # physical channels of a tensor
        return t.C if (not split or t.f32) else 3 * t.C

    concat_parts = {}            # tensor id -> parts (for the physical channel map of split tensors)

    def phys_map(t):
        """(src, part) per physical channel: logical source channel and plane 0 = lo (pairs with Wh), 1 = hi (pairs with
        Wl), 2 = hi (pairs with Wh): the correction terms first in K order (see st_split in csrc/sb_kernels_direct.cuh)."""
        if not split or t.f32:
            return np.arange(t.C), np.zeros(t.C, np.int64)
        if t.id in concat_parts:
            srcs, parts, off = [], [], 0
            for p in concat_parts[t.id]:
                s_, p_ = phys_map(p)
                srcs.append(s_ + off)
                parts.append(p_)
                off += p.C
            return np.concatenate(srcs), np.concatenate(parts)
        return np.tile(np.arange(t.C), 3), np.repeat(np.arange(3), t.C)

    x0.buf, x0.coff = new_buf(x0.C, 1, x0.f32), 0
    copies_before = {}   # sym op index -> list of (src tensor, dst buf, dst coff)
    for idx, (kind, o) in enumerate(g.sym_ops):
        if kind == "concat":
            y = o["y"]
            concat_parts[y.id] = list(o["parts"])
            y.buf, y.coff = new_buf(pc(y), y.stride, False), 0
            off = 0
            for p in o["parts"]:
                if p.buf is None:
                    p.buf, p.coff = y.buf, off
                else:
                    copies_before.setdefault(idx, []).append((p, y.buf, off))
                off += pc(p)
    for t in g.tensors:
        if t.buf is None:
            t.buf, t.coff = new_buf(pc(t), t.stride, t.f32), 0

    cm = CompiledModel()
    cm.spec = spec
    cm.input_channels = input_channels
    cm.max_stride = max_stride
    cm.n_buffers = len(bufs)
    for i, (C, stride, f32) in enumerate(bufs):
        cm.records.append(ol.buffer_record(i, stride, C, f32, 1 if i == 0 else 0))
    cm.records.append(ol.preprocess_record(0, net_c, input_scale, pad_to_stride or max_stride, pre_mode))

    # ---- weights layout ----
    if split:
        by_name = {L["name"]: L for L in g.layers}
        for kind, o in g.sym_ops:
            if kind in ("conv", "tconv") and not o["x"].f32:
                src, part = phys_map(o["x"])
                by_name[o["name"]]["expand"] = (src, part)
    off = 0
    for L in g.layers:
        if L.get("folded"):
            continue
        if L["kind"] in ("conv", "tconv"):
            n = L["k"] * L["k"] * (len(L["expand"][0]) if "expand" in L else L["cin"]) * L["cout"]
            cm._w_slots[L["name"]] = dict(w=off, b=off + n)
            off += n + L["cout"]
        else:
            cm._w_slots[L["name"]] = dict(scale=off, shift=off + L["c"])
            off += 2 * L["c"]
        off = (off + 3) // 4 * 4
    cm.n_weights = off
    cm.layers = g.layers

    def n_readers(t):
        n = 0
        for kind_, o_ in g.sym_ops:
            ins = o_["parts"] if kind_ == "concat" else ([o_["a"], o_["b"]] if kind_ == "add" else [o_["x"]])
            n += sum(1 for u in ins if u is t)
        return n

    tapped = {t.id for t in vec_t.values()}
    flops = 0.0
    fused_pools, fused_adds = set(), set()
    for idx, (kind, o) in enumerate(g.sym_ops):
        for (src, dbuf, dcoff) in copies_before.get(idx, []):
            cm.records.append(ol.copy_record(src.buf, src.coff, pc(src), dbuf, dcoff))
        if kind == "conv":
            x, y = o["x"], o["y"]
            slot = cm._w_slots[o["name"]]
            bn = cm._w_slots[o["bn"]] if o["bn"] else None
            # a 2x2 max-pool that directly follows is offered to the conv's epilogue (the POOL record
            # stays in the list, flagged, and only runs when the conv took the CUDA-core path)
            pool_buf, pool_coff = -1, 0
            if idx + 1 < len(g.sym_ops) and g.sym_ops[idx + 1][0] == "pool" and g.sym_ops[idx + 1][1]["x"] is y \
                    and not copies_before.get(idx + 1) and o["stride"] == 1 and not y.f32:
                py = g.sym_ops[idx + 1][1]["y"]
                pool_buf, pool_coff = py.buf, py.coff
                fused_pools.add(idx + 1)
            # an ADD right after this conv with this conv's output as one operand, which nothing else reads: offered to
            # the conv's epilogue (residual add + the ADD's ReLU); the ADD record stays, flagged, for the CUDA-core path
            res = None
            if idx + 1 < len(g.sym_ops) and g.sym_ops[idx + 1][0] == "add" and not copies_before.get(idx + 1) \
                    and not y.f32 and not o["relu"] and not o["bn"] and pool_buf < 0:
                ao = g.sym_ops[idx + 1][1]
                other = ao["b"] if ao["a"] is y else (ao["a"] if ao["b"] is y else None)
                if other is not None and other is not y and n_readers(y) == 1 and y.id not in tapped:
                    res = (other.buf, other.coff, ao["y"].buf, ao["y"].coff)
                    fused_adds.add(idx + 1)
            cm.records.append(ol.conv_record(x.buf, x.coff, pc(x), y.buf, y.coff, y.C, o["k"], o["stride"],
                                             relu=o["relu"], w_off=slot["w"], b_off=slot["b"],
                                             bn_scale_off=bn["scale"] if bn else -1, bn_shift_off=bn["shift"] if bn else -1,
                                             pool_buf=pool_buf, pool_coff=pool_coff, pad=o.get("pad"), res=res))
            flops += 2.0 * o["k"] * o["k"] * x.C * y.C / (y.stride ** 2)
        elif kind == "tconv":
            x, y = o["x"], o["y"]
            slot = cm._w_slots[o["name"]]
            cm.records.append(ol.tconv_record(x.buf, x.coff, pc(x), y.buf, y.coff, y.C, w_off=slot["w"], b_off=slot["b"], k=o["k"]))
            flops += 2.0 * o["k"] ** 2 * x.C * y.C / (x.stride ** 2)     # 2*k*k*Cin*Cout MACs per *input* pixel (Keras count)
        elif kind == "pool":
            cm.records.append(ol.pool_record(o["x"].buf, o["x"].coff, pc(o["x"]), o["y"].buf, o["y"].coff,
                                             fused=idx in fused_pools, k=o["k"]))
        elif kind == "up":
            cm.records.append(ol.upsample_record(o["x"].buf, o["x"].coff, pc(o["x"]), o["y"].buf, o["y"].coff, o["bilinear"]))
        elif kind == "add":
            cm.records.append(ol.add_record(o["a"].buf, o["a"].coff, o["b"].buf, o["b"].coff, pc(o["a"]), o["y"].buf, o["y"].coff,
                                            relu=o["relu"], fused=idx in fused_adds))
        elif kind == "concat":
            pass
    cm.flops_per_pixel = flops
    for hd in spec["heads"]:
        cm.head_strides[hd["name"]] = hd["output_stride"]
        if hd["name"] in vec_t:
            t = vec_t[hd["name"]]
            cm.vector_taps[hd["name"]] = dict(buf=t.buf, coff=t.coff, C=t.C, planes=3 if (split and not t.f32) else 1,
                                              buf_C=bufs[t.buf][0], f32=bool(t.f32))
            continue
        cm.head_buffers[hd["name"]] = head_t[hd["name"]].buf
    return cm


def make_synthetic_weights(cm: CompiledModel, seed: int) -> Dict[str, Dict[str, np.ndarray]]:
    """SURVEY 8(d) canonical synthetic model: He-normal kernels N(0, 2/fan_in), zero biases,
    BN gamma=1 beta=0 mean=0 var=1; ``numpy.random.default_rng(seed)``.  Keras layouts."""
    rng = np.random.default_rng(seed)
    w = {}
    for L in cm.layers:
        if L["kind"] == "conv":
            std = math.sqrt(2.0 / (L["k"] * L["k"] * L["cin"]))
            w[L["name"]] = dict(kernel=(rng.standard_normal((L["k"], L["k"], L["cin"], L["cout"])) * std).astype(np.float32),
                                bias=np.zeros((L["cout"],), np.float32))
        elif L["kind"] == "tconv":
            # effective fan-in of a k s2 transposed conv is ~ (k^2/4) * Cin taps per output pixel
            std = math.sqrt(2.0 / (L["k"] ** 2 / 4.0 * L["cin"]))
            w[L["name"]] = dict(kernel=(rng.standard_normal((L["k"], L["k"], L["cout"], L["cin"])) * std).astype(np.float32),
                                bias=np.zeros((L["cout"],), np.float32))
        else:
            c = L["c"]
            w[L["name"]] = dict(gamma=np.ones((c,), np.float32), beta=np.zeros((c,), np.float32),
                                mean=np.zeros((c,), np.float32), var=np.ones((c,), np.float32))
    return w


def count_params(cm: CompiledModel) -> int:
    n = 0
    for L in cm.layers:
        if L["kind"] in ("conv", "tconv"):
            n += L["k"] * L["k"] * L["cin"] * L["cout"] + L["cout"]
        else:
            n += 4 * L["c"]
    return n
