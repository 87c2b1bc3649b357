"""Every op of the fp16 and split-precision forwards against a float64 recompute from the device's own inputs
(tests/layer_audit.py), per element, against a bound derived from the kernel's arithmetic.

Each model is audited in two runs:
  * production: every buffer except those internal to a fusion is fetched, and the run must launch exactly the kernels of
    a heads-only forward (plus one k_half_to_float per fetched fp16 buffer); fused ops are checked through what they
    produce (pooled tensors, the residual sum, the first block's pooled output from the frame);
  * all buffers: every buffer is fetched (dead stores written, the residual ADD and the first block's two convs separate),
    which audits each of those ops on its own.
Gates per checked output: worst |err| / bound <= 1; no miss where the bound decides the fp16 rounding; and for larger
outputs the exact-match fraction and the mean signed error in fp16 ulps, at
thresholds set from the H100 measurement with margin (see the constants)."""
import re
import time
from ctypes import byref, c_int, c_void_p

import numpy as np
import pytest

import layer_audit as la

pytestmark = pytest.mark.gpu

# Measured on one H100 80GB HBM3 (400 W power limit) over every case of this file, outputs of >= STAT_MIN_N elements:
# exact-match fraction >= 0.748 (the fused first block's pooled output, checked through its hidden conv0; every directly
# checked output >= 0.99), |mean signed error| <= 0.116 ulp.  Round toward zero on the store gives about -0.5 ulp.  The
# lo-plane bias of precision 2 is printed but not gated: it reached -3.3 ulp(lo) on a ResNet 3x3 layer, so it does not
# separate a correct lo rounding from a wrong one there.
EXACT_MIN = 0.70
BIAS_MAX = 0.2
STAT_MIN_N = 4096          # outputs with fewer elements are gated by the bound and the decided roundings only


def _op_kinds(model, B, H, W, C):
    import torch
    from sleap_b200 import _lib
    dev = torch.zeros((B, H, W, C), dtype=torch.uint8, device="cuda")
    n = len(model.cm.records)
    ms, kind, fl = np.zeros(n, np.float32), np.zeros(n, np.int32), np.zeros(n, np.float64)
    cnt = c_int(0)
    model.handle.call("sb_model_profile_ops", model.model_id, c_void_p(dev.data_ptr()), B, n, _lib.ptr(ms), _lib.ptr(kind),
                      _lib.ptr(fl), byref(cnt))
    return kind[:cnt.value]


def _fetch(model, aud, imgs, ids):
    from sleap_b200._lib import ptr
    outs = [np.zeros((imgs.shape[0],) + aud.shape(b)[1:], np.float32) for b in ids]
    ptrs = (c_void_p * len(outs))(*[o.ctypes.data for o in outs])
    model.handle.call("sb_model_forward", model.model_id, ptr(np.ascontiguousarray(imgs)), int(imgs.dtype == np.uint8),
                      imgs.shape[0], len(outs), ptr(np.asarray(ids, np.int32)), ptrs)
    return dict(zip(ids, outs))


def _forms(err):
    forms = {}
    for m in re.finditer(r"\[sb_conv_tc\] op (\d+) launch \d+[^:]*:.*-> (\w+)", err):
        forms.setdefault(int(m.group(1)), set()).add(m.group(2))
    for m in re.finditer(r"\[sb_conv_tc\] op (\d+) first layer:.*-> (\w+)", err):
        forms.setdefault(int(m.group(1)), set()).add(m.group(2))
    return forms


def _gate(rows, label):
    for r in rows:
        tag = f"{label}: op {r['op']} {r['what']}"
        assert r["worst"] <= 1.0, f"{tag}: worst err / bound {r['worst']:.3g} at {r.get('where')}"
        assert r.get("missed", 0) == 0, f"{tag}: {r['missed']} elements differ from fp16(reference) where the bound decides the rounding, first (index, device, reference, e_pre) = {r.get('miss_at')}"
        if r.get("out") == "f16" and r["n"] >= STAT_MIN_N:
            assert r["exact"] >= EXACT_MIN, f"{tag}: exact-match fraction {r['exact']:.4f}"
            assert abs(r["bias"]) <= BIAS_MAX, f"{tag}: mean signed error {r['bias']:.4f} ulp, largest (index, device, reference, e_pre, ulps) = {r.get('bias_at')}"


def _audit(spec, in_ch, imgs, precision, capfd, monkeypatch, env=(), expect=None, all_buffers=True, input_scale=1.0, seed=5,
           weights=None, max_batch=None):
    """``weights``: a weight dict (e.g. a trained model's); None = la.synthetic_weights(seed).
    ``max_batch``: configure (and autotune) at this batch and audit ``imgs`` at their own, smaller batch, after a poison
    forward of ``max_batch`` other frames (constant 255, or floats around 50) with every buffer fetched, so that every
    slot past the audited frames, the fusion-internal buffers included, holds stale data of another magnitude."""
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    t0 = time.time()
    monkeypatch.setenv("SB_DEBUG", "1")
    for k, v in dict(env).items():
        monkeypatch.setenv(k, v)
    w = weights if weights is not None else la.synthetic_weights(A.compile_model(spec, in_ch, input_scale, split=precision == 2), seed)
    model = DeviceModel(spec, w, input_channels=in_ch, input_scale=input_scale, precision=precision)
    B, H, W, C = imgs.shape
    capfd.readouterr()
    model.configure(max_batch or B, H, W, C)
    err = capfd.readouterr().err
    if expect:
        assert expect in err, f"{expect!r} never ran"
    if dict(env).get("SB_FORCE_VARIANT") == "0":
        picked = re.findall(r"\[sb_conv_tc\] op \d+ launch \d+[^:]*:.*-> (\w+)", err)
        assert picked and set(picked) == {"streaming"}, set(picked)
    kinds = _op_kinds(model, B, H, W, C)
    aud = la.Audit(model.cm, model.cm.pack_weights(w), precision, imgs, kinds, conv01="-> fused" in err)
    forms = _forms(err)
    label = f"{spec['backbone']} p{precision} {dict(env)}"
    if max_batch:
        assert max_batch > B
        label += f" {imgs.dtype} B {max_batch} -> {B}"
        poison = (np.full((max_batch, H, W, C), 255, np.uint8) if imgs.dtype == np.uint8 else
                  np.random.default_rng(seed).uniform(45, 55, (max_batch, H, W, C)).astype(np.float32))
        _fetch(model, aud, poison, list(aud.bufs))

    # (a) production run: the benchmark's kernels
    internal = aud.internal_buffers(True)
    ids = [b for b in aud.bufs if b not in internal]
    model.forward(imgs)
    l0 = model.handle.gpu_launches(); model.forward(imgs); l_heads = model.handle.gpu_launches() - l0
    l0 = model.handle.gpu_launches(); dev = _fetch(model, aud, imgs, ids); l_prod = model.handle.gpu_launches() - l0
    n_half = sum(1 for b in ids if not aud.bufs[b]["f32"])
    assert l_prod == l_heads + n_half, (l_prod, l_heads, n_half)
    rows = aud.run(dev, production=True)
    print(f"\n== {label}: production run, {B} x {H}x{W}x{C}, {len(rows)} outputs checked\n" + la.format_rows(rows, forms))
    _gate(rows, label + " production")
    if all_buffers:
        ids = [b for b in aud.bufs if b not in aud.internal_buffers(False)]
        rows = aud.run(_fetch(model, aud, imgs, ids), production=False)
        print(f"== {label}: all-buffers run\n" + la.format_rows(rows, forms))
        _gate(rows, label + " all buffers")
    print(f"== {label}: {time.time() - t0:.1f} s")
    return rows


def _c4():
    import bench
    return bench.c4_spec()


def _frames(shape, seed):
    return np.random.default_rng(seed).integers(0, 256, size=shape, dtype=np.uint8)


@pytest.mark.parametrize("case", ["autotuned", "streaming", "halo", "conv01"])
def test_audit_c4(case, capfd, monkeypatch):
    """C4 UNet, precision 0, 200 x 232 frames (net 224 x 256: partial tiles from stride 8 on)."""
    env, expect, B = {"autotuned": ({}, None, 3), "streaming": ({"SB_FORCE_VARIANT": "0"}, None, 1),
                      "halo": ({"SB_FORCE_VARIANT": "2"}, "-> halo", 3), "conv01": ({"SB_FORCE_CONV01": "1"}, "-> fused", 1)}[case]
    _audit(_c4(), 1, _frames((B, 200, 232, 1), 1), 0, capfd, monkeypatch, env, expect, all_buffers=case == "autotuned")


def test_audit_c4_precision2(capfd, monkeypatch):
    _audit(_c4(), 1, _frames((2, 200, 232, 1), 2), 2, capfd, monkeypatch)


def test_audit_unet_bilinear_resized_rgb(capfd, monkeypatch):
    """Bilinear upsampling, output stride 2, RGB frames into a gray model at input_scale 0.5 (rgb -> gray + resize in
    PREPROCESS, then the Toeplitz view of the preprocessed buffer), a frame that is not a multiple of the max stride."""
    cfg = dict(filters=16, filters_rate=2, max_stride=16, output_stride=2, middle_block=True, up_interpolate=True, stacks=1)
    spec = dict(backbone="unet", backbone_cfg=cfg, head_type="multi_instance", part_names=None, edges=None,
                heads=[dict(name="MultiInstanceConfmapsHead", channels=6, output_stride=2),
                       dict(name="PartAffinityFieldsHead", channels=10, output_stride=4)])
    _audit(spec, 1, _frames((2, 300, 346, 3), 3), 0, capfd, monkeypatch, input_scale=0.5)


def _resnet(up):
    ups = {"tconv_concat": dict(method="transposed_conv", skip_connections="concatenate", block_stride=2, filters=64, filters_rate=1,
                                refine_convs=2, batch_norm=True, transposed_conv_kernel_size=4),
           "interp_add": dict(method="interpolation", skip_connections="add", block_stride=2, filters=64, filters_rate=1,
                              refine_convs=1, batch_norm=False, transposed_conv_kernel_size=4)}[up]
    cfg = dict(version="ResNet50", weights="frozen", max_stride=32, output_stride=4, upsampling=ups)
    return dict(backbone="resnet", backbone_cfg=cfg, head_type="multi_instance", part_names=None, edges=None,
                heads=[dict(name="MultiInstanceConfmapsHead", channels=5, output_stride=4),
                       dict(name="PartAffinityFieldsHead", channels=8, output_stride=8)])


@pytest.mark.parametrize("precision", [0, 2])
@pytest.mark.parametrize("up", ["tconv_concat", "interp_add"])
def test_audit_resnet50(up, precision, capfd, monkeypatch):
    """Stem through the space-to-depth view with ImageNet preprocessing (precision 0), the zero-padded 3x3/2 pool,
    stride-2 1x1 convs, fused residual epilogues, k4 transposed-conv phases, BN folded and in the generic epilogue."""
    B = 1 if up == "interp_add" else 2
    _audit(_resnet(up), 3, _frames((B, 150, 176, 3), 4), precision, capfd, monkeypatch)


@pytest.mark.parametrize("precision", [0, 2])
def test_audit_hourglass(precision, capfd, monkeypatch):
    """conv -> ReLU -> BN, nearest x2, additive skips, the 7x7/2 stem."""
    spec = dict(backbone="hourglass", head_type="multi_instance", part_names=None, edges=None,
                backbone_cfg=dict(stem_stride=4, max_stride=32, output_stride=4, stem_filters=16, filters=32, filter_increase=32, stacks=2),
                heads=[dict(name="MultiInstanceConfmapsHead", channels=6, output_stride=4),
                       dict(name="PartAffinityFieldsHead", channels=10, output_stride=4)])
    _audit(spec, 3, _frames((2, 120, 136, 3), 5), precision, capfd, monkeypatch)


def test_audit_leap(capfd, monkeypatch):
    cfg = dict(max_stride=8, output_stride=2, filters=16, filters_rate=2, up_interpolate=False, stacks=1)
    spec = dict(backbone="leap", backbone_cfg=cfg, head_type="multi_instance", part_names=None, edges=None,
                heads=[dict(name="MultiInstanceConfmapsHead", channels=5, output_stride=2),
                       dict(name="PartAffinityFieldsHead", channels=8, output_stride=4)])
    _audit(spec, 1, _frames((3, 96, 112, 1), 6), 0, capfd, monkeypatch)


def test_split_store_bit_exact_when_the_accumulation_is_exact(capfd, monkeypatch):
    """Precision 2's lo plane, bit for bit.  The bound above is wider than lo's own rounding, so here the data make the
    tensor-core accumulation exact: frame -> 1x1 conv (CUDA cores, fp32, weights 1) -> split tensor x in [192, 256) on a
    2^-14 grid (hi + lo represent it exactly) -> 3x3 conv on the tensor cores whose output columns each have three +1 or
    three -1 weights, + a bias on the same grid, with its 2x2 max-pool fused.  Every partial sum is a multiple of 2^-14
    below 2^24 units, so the fp32 accumulator is exact whatever it truncates; away from the border v lies in [512, 832)
    and v - hi needs up to 13 bits: the epilogue must store hi = fp16_rn(v) and lo = fp16_rn(v - hi) exactly, in the conv output and the pool."""
    from sleap_b200 import _lib
    from sleap_b200.nn import oplist as ol
    rng = np.random.default_rng(31)
    q = 2.0 ** -14
    B, H, W = 2, 40, 56
    b1 = (rng.integers(0, 32 / q, 16) * q).astype(np.float32)
    w2 = np.zeros((3, 3, 16, 16), np.float32)
    for co in range(16):
        sign = 1.0 if co % 2 == 0 else -1.0
        for t in rng.choice(9 * 16, 3, replace=False):
            w2[t // 48, (t // 16) % 3, t % 16, co] = sign
    b2 = (np.where(np.arange(16) % 2 == 0, 1, -1) * rng.integers(0, 64 / q, 16) * q).astype(np.float32)
    w2x = np.concatenate([w2, np.zeros_like(w2), w2], axis=2)          # [Wh | Wl | Wh] rows, Wl = 0 (fp16-exact weights)
    blob = np.concatenate([np.ones(16, np.float32), b1, w2x.reshape(-1), b2]).astype(np.float32)
    o2 = 32
    recs = [ol.buffer_record(0, 1, 1, 1, 1), ol.buffer_record(1, 1, 48, 0, 0), ol.buffer_record(2, 1, 48, 0, 0),
            ol.buffer_record(3, 2, 48, 0, 0), ol.preprocess_record(0, 1, 1.0, 2),
            ol.conv_record(0, 0, 1, 1, 0, 16, 1, 1, False, 0, 16),
            ol.conv_record(1, 0, 48, 2, 0, 16, 3, 1, False, o2, o2 + w2x.size, pool_buf=3, pool_coff=0),
            ol.pool_record(2, 0, 48, 3, 0, fused=True)]
    ops = np.ascontiguousarray(np.stack(recs).astype(np.int32))
    imgs = (192 + rng.integers(0, 32 / q, size=(B, H, W, 1)) * q).astype(np.float32)
    monkeypatch.setenv("SB_DEBUG", "1")
    h = _lib.Handle(0)
    try:
        mid = c_int(-1)
        h.call("sb_load_model", _lib.ptr(ops), ops.shape[0], _lib.ptr(blob), int(blob.size), 2, byref(mid))
        capfd.readouterr()
        h.call("sb_model_configure", mid.value, B, H, W, 1)
        assert "[sb_conv_tc] op 2 launch" in capfd.readouterr().err          # the 3x3 conv runs on the tensor cores
        outs = [np.zeros((B, H, W, 48), np.float32), np.zeros((B, H // 2, W // 2, 48), np.float32)]
        ptrs = (c_void_p * 2)(*[o.ctypes.data for o in outs])
        h.call("sb_model_forward", mid.value, _lib.ptr(imgs), 0, B, 2, _lib.ptr(np.asarray([2, 3], np.int32)), ptrs)
    finally:
        h.close()
    x = imgs.astype(np.float64) + b1.astype(np.float64)
    v = la.conv64(x, w2.astype(np.float64), 1, 1, 1, H, W) + b2
    assert np.all(np.abs(v) < 2.0 ** 24 * q)
    for got, ref in ((outs[0], v), (outs[1], la.pool2(v))):
        hi = la.f16(ref)
        lo = la.f16(ref - hi)
        assert np.mean(lo != ref - hi) > 0.1            # lo really is rounded in a good share of the elements
        assert np.array_equal(got[..., 16:32], hi) and np.array_equal(got[..., 32:48], hi)
        bad = got[..., 0:16] != lo
        assert not bad.any(), f"{int(bad.sum())} lo values differ, first {got[..., 0:16][bad][:4]} vs {lo[bad][:4]}"
