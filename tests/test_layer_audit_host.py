"""CPU tests of the float64 op-list interpreter and per-element checker (tests/layer_audit.py).

* The interpreter is the network: chained on its own outputs from the frame, it reproduces the float32 oracles, also
  on the secondary benchmark networks at full width, a filters_rate 1.5 UNet and a trained fixture model.
* The checker is sensitive: an emulation of a correct device (truncating fp32 accumulation per K = 16 step, fp32
  epilogue, round-to-nearest stores) passes; each planted fault fails.  The same for precision 1 with an emulation of
  the fp32 CUDA-core kernels (fma in k_conv_direct's order, fp32 epilogue and stores)."""
import numpy as np
import pytest

import backbone_oracle as bo
import layer_audit as la
import reference_models as rm
from oracle import convnet, preprocess as opre
from sleap_b200.nn import architectures as A
from sleap_b200.nn import oplist as ol


def _interpret_heads(spec, in_ch, imgs, split=False, seed=3, precision=None, weights=None):
    cm = A.compile_model(spec, in_ch, split=split)
    w = weights if weights is not None else la.synthetic_weights(A.compile_model(spec, in_ch), seed)
    kinds = [2 if r[0] in (ol.CONV, ol.TCONV) else 0 for r in cm.records if r[0] != ol.BUFFER]   # fp32 operands
    aud = la.Audit(cm, cm.pack_weights(w), (2 if split else 0) if precision is None else precision, imgs, kinds)
    buf = la.interpret(aud, "exact")
    return [buf[cm.head_buffers[h["name"]]] for h in spec["heads"]], w


UNET = dict(backbone="unet", head_type="multi_instance", part_names=None, edges=None,
            backbone_cfg=dict(filters=8, filters_rate=2, max_stride=8, output_stride=2, middle_block=True, up_interpolate=False, stacks=1),
            heads=[dict(name="MultiInstanceConfmapsHead", channels=3, output_stride=2),
                   dict(name="PartAffinityFieldsHead", channels=4, output_stride=4)])
HOURGLASS = dict(backbone="hourglass", head_type="multi_instance", part_names=None, edges=None,
                 backbone_cfg=dict(stem_stride=4, max_stride=16, output_stride=4, stem_filters=8, filters=16, filter_increase=8, stacks=2),
                 heads=[dict(name="MultiInstanceConfmapsHead", channels=3, output_stride=4),
                        dict(name="PartAffinityFieldsHead", channels=4, output_stride=4)])
RESNET = dict(backbone="resnet", head_type="multi_instance", part_names=None, edges=None,
              backbone_cfg=dict(version="ResNet50", weights="frozen", max_stride=32, output_stride=4,
                                upsampling=dict(method="transposed_conv", skip_connections="concatenate", block_stride=2, filters=32,
                                                filters_rate=1, refine_convs=1, batch_norm=True, transposed_conv_kernel_size=4)),
              heads=[dict(name="MultiInstanceConfmapsHead", channels=3, output_stride=4),
                     dict(name="PartAffinityFieldsHead", channels=4, output_stride=8)])
LEAP = dict(backbone="leap", head_type="multi_instance", part_names=None, edges=None,
            backbone_cfg=dict(max_stride=8, output_stride=2, filters=8, filters_rate=2, up_interpolate=False, stacks=1),
            heads=[dict(name="MultiInstanceConfmapsHead", channels=3, output_stride=2),
                   dict(name="PartAffinityFieldsHead", channels=4, output_stride=4)])


# The secondary benchmark networks at their real widths (tools/bench_configs.py): C3's centered-instance UNet (channels
# 24 .. 384, transposed convs) and C5's hourglass (stem 128, filters 256 + 128 per level, 3 stacks, max stride 64)
C3_INSTANCE = dict(backbone="unet", head_type="centered_instance", part_names=[f"n{i}" for i in range(13)], edges=None,
                   backbone_cfg=dict(filters=24, filters_rate=2, max_stride=16, output_stride=4, middle_block=True,
                                     up_interpolate=False, stacks=1),
                   heads=[dict(name="CenteredInstanceConfmapsHead", channels=13, output_stride=4)])
C5_HOURGLASS = dict(backbone="hourglass", head_type="multi_instance", part_names=None, edges=None,
                    backbone_cfg=dict(stem_stride=4, max_stride=64, output_stride=4, stem_filters=128, filters=256,
                                      filter_increase=128, stacks=3),
                    heads=[dict(name="MultiInstanceConfmapsHead", channels=24, output_stride=4),
                           dict(name="PartAffinityFieldsHead", channels=46, output_stride=4)])
# filters_rate 1.5: widths 16 / 24 / 36 / 54 / 81, so most convs run on the CUDA cores and concat slices sit at odd offsets
UNET_RATE15 = dict(backbone="unet", head_type="multi_instance", part_names=None, edges=None,
                   backbone_cfg=dict(filters=16, filters_rate=1.5, max_stride=16, output_stride=2, middle_block=True,
                                     up_interpolate=False, stacks=1),
                   heads=[dict(name="MultiInstanceConfmapsHead", channels=5, output_stride=2),
                          dict(name="PartAffinityFieldsHead", channels=8, output_stride=4)])
FIXTURE = "min_tracks_2node.bottomup_multiclass"       # trained, filters 8, rate 1.5 (8 / 12 / 18 / 27 / 40), bilinear


@pytest.mark.parametrize("name", ["unet", "hourglass", "resnet", "leap", "c3_instance", "c5_hourglass", "unet_rate15",
                                  "fixture"])
def test_interpreter_is_the_network(name):
    weights = None
    if name == "fixture":
        _, spec, weights, in_ch = rm.load_fixture_model(FIXTURE)
    else:
        spec, in_ch = {"unet": (UNET, 1), "hourglass": (HOURGLASS, 3), "resnet": (RESNET, 3), "leap": (LEAP, 1),
                       "c3_instance": (C3_INSTANCE, 1), "c5_hourglass": (C5_HOURGLASS, 3), "unet_rate15": (UNET_RATE15, 1)}[name]
    B = 1 if name == "c5_hourglass" else 2
    imgs = np.random.default_rng(1).integers(0, 256, size=(B, 40, 56, in_ch), dtype=np.uint8)
    got, w = _interpret_heads(spec, in_ch, imgs, weights=weights)
    ms = spec["backbone_cfg"]["max_stride"]
    x = opre.preprocess(imgs, ensure_gray=in_ch == 1, pad_stride=ms)
    want = (bo.model_forward(x, spec, w) if name in ("resnet", "leap") else convnet.model_forward(x, spec, w))
    for g, ref in zip(got, want):
        assert g.shape == ref.shape
        assert np.abs(g - ref).max() <= 1e-4 * np.abs(ref).max()


@pytest.mark.parametrize("name", ["unet", "hourglass"])
def test_interpreter_precision1_op_list_is_the_network(name):
    """Audit(precision=1): every buffer fp32, every conv on the CUDA cores; chained from the frame it is the network."""
    spec, in_ch = {"unet": (dict(UNET, backbone_cfg=dict(UNET["backbone_cfg"], up_interpolate=True)), 1),
                   "hourglass": (HOURGLASS, 3)}[name]
    imgs = np.random.default_rng(5).integers(0, 256, size=(1, 40, 56, in_ch), dtype=np.uint8)
    got, w = _interpret_heads(spec, in_ch, imgs, precision=1)
    x = opre.preprocess(imgs, ensure_gray=in_ch == 1, pad_stride=spec["backbone_cfg"]["max_stride"])
    for g, ref in zip(got, convnet.model_forward(x, spec, w)):
        assert g.shape == ref.shape
        assert np.abs(g - ref).max() <= 1e-4 * np.abs(ref).max()


@pytest.mark.parametrize("name", ["unet", "hourglass", "resnet"])
def test_interpreter_split_op_list_is_the_plain_one(name):
    """On the split op list ([lo | hi | hi] tensors, [Wh | Wl | Wh] rows, fp32 frame) the interpreter gives the same
    logical maps as on the plain op list, up to the dropped lo * Wl term (2^-22 relative)."""
    spec, in_ch = {"unet": (UNET, 1), "hourglass": (HOURGLASS, 3), "resnet": (RESNET, 3)}[name]
    imgs = np.random.default_rng(2).integers(0, 256, size=(1, 40, 56, in_ch), dtype=np.uint8)
    plain, _ = _interpret_heads(spec, in_ch, imgs)
    split, _ = _interpret_heads(spec, in_ch, imgs, split=True)
    for a, b in zip(plain, split):
        assert np.abs(a - b).max() <= 2e-6 * np.abs(a).max()


# ---------------------------------------------------------------------------------------------- checker sensitivity
def _trunc32(a):
    r = a.astype(np.float32)
    over = np.abs(r.astype(np.float64)) > np.abs(a)
    r[over] = np.nextafter(r[over], np.float32(0))
    return r.astype(np.float64)


def _r32(a):
    return np.asarray(a, np.float64).astype(np.float32).astype(np.float64)


def emulate(fault=None, fault_op=-1):
    """conv_fn of la.interpret emulating the tensor-core path: fp16 operands, an fp32 accumulator truncated after every
    K = 16 step (tap-major, 16-channel chunks), residual, bias, ReLU, BN in fp32.  ``fault`` plants one bug in op
    ``fault_op``."""
    def conv_fn(aud, i, x, res, relu):
        op = aud.ops[i]
        k, st = int(op[9]), int(op[10])
        w, b = aud._weights(op, x.shape[3], aud.engine(i) in ("tc", "conv01"))
        if i == fault_op and fault == "bias":
            b = np.roll(b, -1)                       # bias read from the neighbouring channel
        ob = aud.shape(int(op[6]))
        if op[0] == ol.TCONV:
            acc = _trunc32(la.tconv64(x, w, k))
        else:
            Hin, Win = x.shape[1:3]
            pt = int(op[16]) if op[11] & ol.F_EXPLICIT_PAD else max((ob[1] - 1) * st + k - Hin, 0) // 2
            pl = int(op[17]) if op[11] & ol.F_EXPLICIT_PAD else max((ob[2] - 1) * st + k - Win, 0) // 2
            if i == fault_op and fault == "cross_frame":      # frame 0's bottom SAME-pad row read from frame 1's first row
                x = np.concatenate([x, np.concatenate([x[1:2, :1], np.zeros_like(x[1:, :1])])], axis=1)
            elif i == fault_op and fault == "wrong_frame":    # frame 1's input read from frame 0's slot
                x = np.concatenate([x[:1], x[:1], x[2:]])
            acc = np.zeros(ob[:3] + (w.shape[3],))
            for ky in range(k):
                for kx in range(k):
                    for c0 in range(0, x.shape[3], 16):
                        wt = np.zeros_like(w)
                        wt[ky, kx, c0:c0 + 16] = w[ky, kx, c0:c0 + 16]
                        part = la.conv64(x, wt, st, pt, pl, ob[1], ob[2])
                        if i == fault_op and fault == "tap" and (ky, kx) == (1, 1):
                            part[:, 0, 0] = 0                # one tap missing on the corner pixel
                        acc = _trunc32(acc + part)
        v = acc
        if res is not None:
            v = _r32(v + res) if fault != "double_round" else la.f16(v) + res
        v = _r32(v + b)
        if relu is None:
            relu = bool(op[11] & ol.F_RELU)
        if relu:
            v = np.maximum(v, 0)
        if op[11] & ol.F_BN:
            sc = aud.blob[int(op[14]):int(op[14]) + int(op[8])].astype(np.float64)
            sh = aud.blob[int(op[15]):int(op[15]) + int(op[8])].astype(np.float64)
            v = _r32(_r32(v * sc) + sh)
        if i == fault_op and fault == "rz":           # round toward zero on the fp16 store
            h = la.f16(v)
            v = np.where(np.abs(h) > np.abs(v), np.nextafter(h.astype(np.float16), np.float16(0)).astype(np.float64), h)
        return v
    return conv_fn


def _toy():
    """frame -> conv a (1 -> 16, 3x3, the fused first block's conv0) -> conv b (16 -> 16, dead full-resolution output,
    fused 2x2 pool into channels 0-15 of a 32-channel buffer) -> conv c (channels 0-15 -> 16-31 of the same buffer) ->
    conv d (1x1, 32 -> 16, residual = conv c, fused ADD with ReLU) -> fp32 1x1 head."""
    rng = np.random.default_rng(7)
    parts, offs = [], []

    def add(*shape, scale=1.0):
        offs.append(sum(p.size for p in parts))
        parts.append((rng.standard_normal(shape) * scale).astype(np.float32).reshape(-1))
        return offs[-1]
    wa, ba = add(3, 3, 1, 16, scale=0.5), add(16, scale=0.1)
    wb, bb = add(3, 3, 16, 16, scale=(2 / 144) ** 0.5), add(16, scale=0.1)
    wc, bc = add(3, 3, 16, 16, scale=(2 / 144) ** 0.5), add(16, scale=0.1)
    wd, bd = add(1, 1, 32, 16, scale=(2 / 32) ** 0.5), add(16, scale=0.1)
    wh, bh = add(1, 1, 16, 5, scale=0.25), add(5, scale=0.1)
    blob = np.concatenate(parts)
    recs = [ol.buffer_record(0, 1, 1, 0, 1), ol.buffer_record(1, 1, 16, 0, 0), ol.buffer_record(2, 1, 16, 0, 0),
            ol.buffer_record(3, 2, 32, 0, 0), ol.buffer_record(4, 2, 16, 0, 0), ol.buffer_record(5, 2, 16, 0, 0),
            ol.buffer_record(6, 2, 5, 1, 0),
            ol.preprocess_record(0, 1, 1.0, 2),
            ol.conv_record(0, 0, 1, 1, 0, 16, 3, 1, True, wa, ba),
            ol.conv_record(1, 0, 16, 2, 0, 16, 3, 1, True, wb, bb, pool_buf=3, pool_coff=0),
            ol.pool_record(2, 0, 16, 3, 0, fused=True),
            ol.conv_record(3, 0, 16, 3, 16, 16, 3, 1, True, wc, bc),
            ol.conv_record(3, 0, 32, 4, 0, 16, 1, 1, False, wd, bd, res=(3, 16, 5, 0)),
            ol.add_record(4, 0, 3, 16, 16, 5, 0, relu=True, fused=True),
            ol.conv_record(5, 0, 16, 6, 0, 5, 1, 1, False, wh, bh)]

    class CM:
        records = recs
    frames = rng.integers(0, 256, size=(2, 24, 40, 1), dtype=np.uint8)
    kinds = [0, 1, 1, 0, 1, 1, 0, 1]
    return CM, blob, frames, kinds


def _passes(aud, dev):
    try:
        rows = aud.run(dev, production=True)
    except AssertionError:
        return False
    return all(r["worst"] <= 1 and r.get("missed", 0) == 0 for r in rows)


def _dev(aud, fault=None, fault_op=-1):
    buf = la.interpret(aud, "device", production=True, conv_fn=emulate(fault, fault_op))
    return {b: a.astype(np.float32) for b, a in buf.items() if b not in aud.internal_buffers(True)}


def test_checker_passes_faithful_emulation():
    cm, blob, frames, kinds = _toy()
    aud = la.Audit(cm, blob, 0, frames, kinds, conv01=True)
    assert aud.internal_buffers(True) == {0, 1, 2, 4}      # frame, conv0, dead conv1, conv d (residual fused)
    rows = aud.run(_dev(aud), production=True)
    assert {r["what"] for r in rows} >= {"pool(conv)", "conv3x3/1", "conv1x1/1 +res", "conv1x1/1"}
    for r in rows:
        assert r["worst"] <= 1 and r.get("missed", 0) == 0, r


@pytest.mark.parametrize("fault", ["tap", "bias", "rz", "pool_partner", "slice_off", "double_round", "cross_frame",
                                   "wrong_frame"])
def test_checker_catches_planted_fault(fault):
    """cross_frame / wrong_frame: the bugs a run below the configured batch can hide, where the slots past the last frame
    hold an earlier call's data -- a SAME-pad row read from the next frame, a frame's input read from another slot."""
    cm, blob, frames, kinds = _toy()
    aud = la.Audit(cm, blob, 0, frames, kinds, conv01=True)
    op_c, op_d = 4, 5
    if fault in ("tap", "bias", "rz", "cross_frame", "wrong_frame"):
        dev = _dev(aud, fault, op_c)
    elif fault == "double_round":
        dev = _dev(aud, fault, op_d)
    else:
        buf = la.interpret(aud, "device", production=True, conv_fn=emulate())
        dev = {b: a.astype(np.float32) for b, a in buf.items() if b not in aud.internal_buffers(True)}
        if fault == "pool_partner":                     # max of the horizontal partner only
            full = buf[2]
            dev[3][..., 0:16] = np.maximum(full[:, 0::2, 0::2], full[:, 0::2, 1::2])
        else:                                           # conv c written 8 channels off
            dev[3][..., 8:24] = buf[3][..., 16:32]
    assert _passes(aud, _dev(aud)), "the faithful emulation must pass"
    assert not _passes(aud, dev), f"planted fault {fault!r} not caught"


def test_bias_ignores_relu_zero_crossings():
    """A ReLU output whose pre-activation lies within the bound of 0 is 0 on one side and small on the other: that is not
    a rounding bias, and one such element must not swamp the mean signed error; round toward zero still shows in it."""
    ref = np.maximum(np.random.default_rng(0).normal(0, 1, 8192), 0)
    e_pre = np.full_like(ref, 1e-3)
    dev = la.f16(ref)
    z = np.flatnonzero(ref == 0)
    dev[z[0]] = la.f16(5e-4)                              # reference 0, device just above
    r = la.check(dev, ref, e_pre, "f16")
    assert r["worst"] <= 1 and abs(r["bias"]) < 0.01, r
    h = la.f16(ref)
    rz = np.where(np.abs(h) > np.abs(ref), np.nextafter(h.astype(np.float16), np.float16(0)).astype(np.float64), h)
    assert la.check(rz, ref, e_pre, "f16")["bias"] < -0.2


def test_checker_catches_dropped_lo_plane():
    """Precision 2: a producer that stores hi but leaves lo at zero."""
    spec = dict(UNET, backbone_cfg=dict(UNET["backbone_cfg"], filters=16))
    cm = A.compile_model(spec, 1, split=True)
    w = la.synthetic_weights(A.compile_model(spec, 1), 4)
    imgs = np.random.default_rng(3).integers(0, 256, size=(1, 32, 48, 1), dtype=np.uint8)
    kinds = [1 if r[0] in (ol.CONV, ol.TCONV) else 0 for r in cm.records if r[0] != ol.BUFFER]
    kinds[1] = 2                                        # the first conv reads the fp32 frame on the CUDA cores
    aud = la.Audit(cm, cm.pack_weights(w), 2, imgs, kinds)
    dev = _dev(aud)
    assert _passes(aud, dev)
    op = next(o for o in aud.ops if o[0] == ol.CONV and o[3] >= 48 and int(o[6]) in dev and not aud.bufs[int(o[6])]["f32"])
    b, coff, C = int(op[6]), int(op[7]), int(op[8])
    dev[b][..., coff:coff + C] = 0
    assert not _passes(aud, dev)


def test_unfetched_output_is_an_error():
    """A conv writing another slice of a buffer the production run does not fetch (here the dead full-resolution output
    of conv b) is reported, not silently skipped."""
    cm, blob, frames, kinds = _toy()
    recs = list(cm.records)
    recs[2] = ol.buffer_record(2, 1, 32, 0, 0)                           # conv b's buffer gains a second slice
    extra = ol.conv_record(1, 0, 16, 2, 16, 16, 3, 1, True, int(recs[9][12]), int(recs[9][13]))
    recs = recs[:11] + [extra] + recs[11:]                               # after conv b's fused pool

    class CM2:
        records = recs
    aud = la.Audit(CM2, blob, 0, frames, kinds[:4] + [1] + kinds[4:], conv01=True)
    dev = {b: np.zeros(aud.shape(b), np.float32) for b in aud.bufs if b not in aud.internal_buffers(True)}
    with pytest.raises(AssertionError, match="nothing checks it"):
        aud.run(dev, production=True)


# ------------------------------------------------------------------------------ checker sensitivity, precision 1 (fp32)
def emulate32(fault=None, fault_op=-1):
    """conv_fn of la.interpret emulating the fp32 CUDA-core path: k_conv_direct's fma order (8-channel chunks, then
    taps, then the chunk's channels; each fma rounded to fp32), then + bias, ReLU, BN in fp32.  A transposed conv is
    the float64 value rounded once.  ``fault`` plants one bug in op ``fault_op``."""
    def conv_fn(aud, i, x, res, relu):
        op = aud.ops[i]
        k, st = int(op[9]), int(op[10])
        w, b = aud._weights(op, x.shape[3], False)
        bug = fault if i == fault_op else None
        if bug == "bias":
            b = np.roll(b, -1)
        ob = aud.shape(int(op[6]))
        if op[0] == ol.TCONV:
            acc = _r32(la.tconv64(x, w, k))
        else:
            Hin, Win = x.shape[1:3]
            pt = int(op[16]) if op[11] & ol.F_EXPLICIT_PAD else max((ob[1] - 1) * st + k - Hin, 0) // 2
            pl = int(op[17]) if op[11] & ol.F_EXPLICIT_PAD else max((ob[2] - 1) * st + k - Win, 0) // 2
            Hp, Wp = (ob[1] - 1) * st + k, (ob[2] - 1) * st + k
            xp = np.zeros((x.shape[0], Hp, Wp, x.shape[3]))
            h, ww = min(Hin, Hp - pt), min(Win, Wp - pl)
            xp[:, pt:pt + h, pl:pl + ww] = x[:, :h, :ww]
            acc = np.zeros(ob[:3] + (w.shape[3],))
            for c0 in range(0, x.shape[3], 8):
                for ky in range(k):
                    for kx in range(k):
                        win = xp[:, ky:ky + st * (ob[1] - 1) + 1:st, kx:kx + st * (ob[2] - 1) + 1:st]
                        for c in range(c0, min(c0 + 8, x.shape[3])):
                            part = win[..., c:c + 1] * w[ky, kx, c]
                            if bug == "tap" and (ky, kx) == (1, 1):
                                part[:, 0, 0] = 0                # one tap missing on the corner pixel
                            acc = _r32(acc + part)
        v = _r32(acc + b)
        if relu is None:
            relu = bool(op[11] & ol.F_RELU)
        if relu:
            v = np.maximum(v, 0)
        if op[11] & ol.F_BN:
            sc = aud.blob[int(op[14]):int(op[14]) + int(op[8])].astype(np.float64)
            sh = aud.blob[int(op[15]):int(op[15]) + int(op[8])].astype(np.float64)
            v = _r32(_r32(v * sc) + (sh if bug != "bn_shift" else 0.0))
        if bug == "half_store":                     # an fp16 round trip on the fp32 path
            v = la.f16(v)
        return v
    return conv_fn


def _toy32():
    """fp32 op list: frame -> conv a (3x3, 1 -> 12, ReLU + BN) -> 2x2 pool -> conv b (3x3, 12 -> 20, channels 0-19 of a
    28-channel buffer) and conv c (1x1, 12 -> 8, channels 20-27) -> bilinear x2 of conv b, transposed conv of conv b,
    nearest x2 of conv c -> ADD (ReLU) of the two 20-channel maps -> 1x1 head."""
    rng = np.random.default_rng(11)
    parts = []

    def add(*shape, scale=1.0, loc=0.0):
        parts.append((loc + rng.standard_normal(shape) * scale).astype(np.float32).reshape(-1))
        return sum(p.size for p in parts[:-1])
    wa, ba = add(3, 3, 1, 12, scale=0.5), add(12, scale=0.1)
    sa, ha = add(12, scale=0.2, loc=1.0), add(12, scale=0.3)
    wb, bb = add(3, 3, 12, 20, scale=(2 / 108) ** 0.5), add(20, scale=0.1)
    wc, bc = add(1, 1, 12, 8, scale=(2 / 12) ** 0.5), add(8, scale=0.1)
    wt, bt = add(3, 3, 20, 20, scale=(2 / 80) ** 0.5), add(20, scale=0.1)
    wh, bh = add(1, 1, 20, 3, scale=0.25), add(3, scale=0.1)
    blob = np.concatenate(parts)
    recs = [ol.buffer_record(0, 1, 1, 0, 1), ol.buffer_record(1, 1, 12, 0, 0), ol.buffer_record(2, 2, 12, 0, 0),
            ol.buffer_record(3, 2, 28, 0, 0), ol.buffer_record(4, 1, 20, 0, 0), ol.buffer_record(5, 1, 20, 0, 0),
            ol.buffer_record(6, 1, 8, 0, 0), ol.buffer_record(7, 1, 20, 0, 0), ol.buffer_record(8, 1, 3, 1, 0),
            ol.preprocess_record(0, 1, 1.0, 2),
            ol.conv_record(0, 0, 1, 1, 0, 12, 3, 1, True, wa, ba, bn_scale_off=sa, bn_shift_off=ha),
            ol.pool_record(1, 0, 12, 2, 0),
            ol.conv_record(2, 0, 12, 3, 0, 20, 3, 1, True, wb, bb),
            ol.conv_record(2, 0, 12, 3, 20, 8, 1, 1, False, wc, bc),
            ol.upsample_record(3, 0, 20, 4, 0, bilinear=True),
            ol.tconv_record(3, 0, 20, 5, 0, 20, wt, bt),
            ol.upsample_record(3, 20, 8, 6, 0, bilinear=False),
            ol.add_record(4, 0, 5, 0, 20, 7, 0, relu=True),
            ol.conv_record(7, 0, 20, 8, 0, 3, 1, 1, False, wh, bh)]

    class CM:
        records = recs
    frames = rng.integers(0, 256, size=(2, 24, 40, 1), dtype=np.uint8)
    kinds = [0, 2, 0, 2, 2, 0, 2, 0, 0, 2]
    return CM, blob, frames, kinds


def _dev32(aud, fault=None, fault_op=-1):
    buf = la.interpret(aud, "device", conv_fn=emulate32(fault, fault_op))
    return {b: a.astype(np.float32) for b, a in buf.items()}


def test_checker_passes_faithful_fp32_emulation():
    cm, blob, frames, kinds = _toy32()
    aud = la.Audit(cm, blob, 1, frames, kinds)
    assert aud.internal_buffers(True) == set() and all(b["f32"] for b in aud.bufs.values())
    rows = aud.run(_dev32(aud), production=True)
    assert [r["what"] for r in rows] == ["preprocess", "conv3x3/1 +bn", "pool2", "conv3x3/1", "conv1x1/1", "upsample-bilinear",
                                         "tconv", "upsample-nearest", "add", "conv1x1/1"]
    assert {r["out"] for r in rows} == {"f32", "exact"} and {r["engine"] for r in rows if r["steps"]} == {"cuda"}
    for r in rows:
        assert r["worst"] <= 1, r
    conv = {r["op"]: r for r in rows}
    assert conv[1]["steps"] == 9 and conv[3]["steps"] == 9 * 12 and conv[6]["steps"] == 4 * 20     # taps x C_in fma


@pytest.mark.parametrize("fault", ["tap", "bias", "slice_off", "bn_shift", "half_store", "pool_partner", "bilinear_as_nearest",
                                   "add_operand"])
def test_checker_catches_planted_fp32_fault(fault):
    cm, blob, frames, kinds = _toy32()
    aud = la.Audit(cm, blob, 1, frames, kinds)
    op_a, op_b = 1, 3
    if fault in ("tap", "bias", "half_store"):
        dev = _dev32(aud, fault, op_b)
    elif fault == "bn_shift":                           # the BN shift dropped from conv a's epilogue
        dev = _dev32(aud, fault, op_a)
    else:
        dev = _dev32(aud)
        if fault == "slice_off":                        # conv c written one channel off, over conv b's last channel
            dev[3][..., 19:27] = dev[3][..., 20:28].copy()
        elif fault == "pool_partner":                   # max of the horizontal partner only
            full = dev[1]
            dev[2][...] = np.maximum(full[:, 0::2, 0::2], full[:, 0::2, 1::2])
        elif fault == "bilinear_as_nearest":            # the bilinear flag ignored
            dev[4][...] = la.upsample64(dev[3][..., :20].astype(np.float64), False)
        else:                                           # the ADD reads conv b's bilinear map twice
            dev[7][...] = np.maximum(2 * dev[4], 0)
    assert _passes(aud, _dev32(aud)), "the faithful emulation must pass"
    assert not _passes(aud, dev), f"planted fault {fault!r} not caught"
