"""Shared harness of the tensor-core conv tests (sb_conv_tc.cu): op lists that put one conv or transposed conv on the
tensor cores, and ``forced_equal``, which checks that a forced kernel form ran and is bit-identical to the streaming
form 0.

Forms (SB_FORCE_VARIANT=n forces form n where it is eligible): 0 streaming k_conv_wg, 1 persistent k_conv_wg_p with
resident weights, 2 halo-patch k_conv_wg_h, 3 wide halo-patch k_conv_wg_hw, 4 fused transposed conv k_tconv_wg_hw."""
from ctypes import byref, c_int, c_void_p

import numpy as np

PICKED = {1: "-> resident", 2: "-> halo", 3: "-> wide", 4: "-> tconv-fused"}


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def forced_equal(run, form, monkeypatch, capfd, check_ran=True):
    """run() under SB_DEBUG with SB_FORCE_VARIANT=0 and =form; asserts from the autotune lines that form `form` ran
    (check_ran; form 4: that the fused form ran exactly when forced) and that every output of the two runs is equal bit
    for bit.  Returns the form-0 outputs."""
    monkeypatch.setenv("SB_DEBUG", "1")
    outs = {}
    for f in (0, form):
        monkeypatch.setenv("SB_FORCE_VARIANT", str(f))
        capfd.readouterr()
        outs[f] = run()
        err = capfd.readouterr().err
        if form == 4:
            assert (PICKED[4] in err) == (f == 4), "the fused form did not run exactly when forced"
        elif f == form and check_ran:
            assert PICKED[form] in err, f"form {form} never ran"
    for a, b in zip(outs[0], outs[form]):
        assert same_bits(a, b), float(np.abs(a.astype(np.float64) - b).max())
    return outs[0]


class Layer:
    """An op list (frame -> conv0 (3x3, 1 -> cin, CUDA-core) -> ... -> the layer under test), its weights and frames.
    w1 / b1: the weights of the layer under test."""

    def __init__(self, recs, blob, imgs, shapes, ids, crop, w1, b1):
        self.ops = np.ascontiguousarray(np.stack(recs).astype(np.int32))
        self.blob, self.imgs, self.shapes, self.ids, self.crop, self.w1, self.b1 = blob, imgs, shapes, ids, crop, w1, b1

    def run(self, ids=None, probe=None):
        """The requested buffers (default: the layer's outputs; a concat buffer cut to the layer's slice) of one forward
        on a fresh handle.  probe(handle, model_id), if given, runs after the forward and its result is returned too."""
        from sleap_b200 import _lib
        ids = self.ids if ids is None else ids
        B, H, W, _ = self.imgs.shape
        h = _lib.Handle(0)
        mid = c_int(-1)
        h.call("sb_load_model", _lib.ptr(self.ops), self.ops.shape[0], _lib.ptr(self.blob), int(self.blob.size), 0, byref(mid))
        h.call("sb_model_configure", mid.value, B, H, W, 1)
        outs = [np.zeros(self.shapes[i], np.float32) for i in ids]
        ptrs = (c_void_p * len(ids))(*[o.ctypes.data for o in outs])
        h.call("sb_model_forward", mid.value, _lib.ptr(self.imgs), 0, B, len(ids), _lib.ptr(np.asarray(ids, np.int32)), ptrs)
        extra = probe(h, mid.value) if probe else None
        h.close()
        outs = [o[..., self.crop[i]] if i in self.crop else o for i, o in zip(ids, outs)]
        return outs if probe is None else (outs, extra)

    __call__ = run


def conv_layer(cin, cout, hw, B, k=3, relu=True, f32_out=False, pool=None, out_slice=False, in_slice=False):
    """frame -> conv0 (3x3, 1 -> cin) -> conv1 (k x k, cin -> cout, the layer under test).  f32_out: conv1 writes fp32.
    pool: None, "dead" (fused 2x2 max-pool, only the pooled tensor requested: conv1's own stores are skipped) or "alive"
    (both requested).  out_slice / in_slice: conv1 writes / reads a channel slice of a wider concat buffer.
    Buffers: 1 = conv0's output, 2 = conv1's, 3 = the pool's."""
    from sleap_b200.nn import oplist as ol
    rng = np.random.default_rng(7 * cin + cout + k)
    H, W = hw
    in_off, in_tot = (8, cin + 24) if in_slice else (0, cin)
    out_off, out_tot = (16, cout + 48) if out_slice else (0, cout)
    recs = [ol.buffer_record(0, 1, 1, 0, 1), ol.buffer_record(1, 1, in_tot, 0, 0), ol.buffer_record(2, 1, out_tot, f32_out, 0)]
    if pool:
        recs.append(ol.buffer_record(3, 2, cout, 0, 0))
    recs.append(ol.preprocess_record(0, 1, 1.0, 2 if pool else 1))
    w0 = (rng.standard_normal((3, 3, 1, cin)) * 0.5).astype(np.float32)
    b0 = rng.normal(0, 0.1, cin).astype(np.float32)
    w1 = (rng.standard_normal((k, k, cin, cout)) * np.sqrt(2.0 / (k * k * cin))).astype(np.float32)
    b1 = rng.normal(0, 0.1, cout).astype(np.float32)
    blob = np.concatenate([w0.reshape(-1), b0, w1.reshape(-1), b1]).astype(np.float32)
    o1 = w0.size + cin
    recs.append(ol.conv_record(0, 0, 1, 1, in_off, cin, 3, 1, True, 0, w0.size))
    recs.append(ol.conv_record(1, in_off, cin, 2, out_off, cout, k, 1, relu, o1, o1 + w1.size, pool_buf=3 if pool else -1))
    if pool:
        recs.append(ol.pool_record(2, out_off, cout, 3, 0, fused=True))
    imgs = rng.uniform(0, 1, size=(B, H, W, 1)).astype(np.float32)
    ids = [3] if pool == "dead" else ([2, 3] if pool == "alive" else [2])
    shapes = {1: (B, H, W, in_tot), 2: (B, H, W, out_tot), 3: (B, H // 2, W // 2, cout)}
    crop = {1: slice(in_off, in_off + cin), 2: slice(out_off, out_off + cout)}
    return Layer(recs, blob, imgs, shapes, ids, crop, w1, b1)


def tconv_layer(cin, cout, hw, B, out_slice=False, in_slice=False):
    """frame (H x W) -> conv0 (3x3, 1 -> cin) -> 2x2 max-pool -> tconv (k3 s2, cin -> cout, ReLU, the layer under test) on
    the H / 2 x W / 2 grid -> fp16 output at H x W (buffer 3).  out_slice / in_slice: the tconv writes / reads a channel
    slice of a wider concat buffer."""
    from sleap_b200.nn import oplist as ol
    rng = np.random.default_rng(5 * cin + cout)
    H, W = hw
    in_off, in_tot = (8, cin + 24) if in_slice else (0, cin)
    out_off, out_tot = (16, cout + 48) if out_slice else (0, cout)
    recs = [ol.buffer_record(0, 1, 1, 0, 1), ol.buffer_record(1, 1, cin, 0, 0), ol.buffer_record(2, 2, in_tot, 0, 0),
            ol.buffer_record(3, 1, out_tot, 0, 0), ol.preprocess_record(0, 1, 1.0, 2)]
    w0 = (rng.standard_normal((3, 3, 1, cin)) * 0.5).astype(np.float32)
    b0 = rng.normal(0, 0.1, cin).astype(np.float32)
    w1 = (rng.standard_normal((3, 3, cin, cout)) * np.sqrt(2.0 / (4 * cin))).astype(np.float32)
    b1 = rng.normal(0, 0.1, cout).astype(np.float32)
    blob = np.concatenate([w0.reshape(-1), b0, w1.reshape(-1), b1]).astype(np.float32)
    o1 = w0.size + cin
    recs.append(ol.conv_record(0, 0, 1, 1, 0, cin, 3, 1, True, 0, w0.size))
    recs.append(ol.pool_record(1, 0, cin, 2, in_off))
    recs.append(ol.tconv_record(2, in_off, cin, 3, out_off, cout, o1, o1 + w1.size))
    imgs = rng.uniform(0, 1, size=(B, H, W, 1)).astype(np.float32)
    return Layer(recs, blob, imgs, {3: (B, H, W, out_tot)}, [3], {3: slice(out_off, out_off + cout)}, w1, b1)


def model_run(spec, in_ch, imgs, precision, seed=3):
    """run() of a whole network on the device with non-trivial biases and BN statistics (every epilogue term is exercised)."""
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    cm = A.compile_model(spec, in_ch)
    w = A.make_synthetic_weights(cm, seed)
    rng = np.random.default_rng(seed + 1)
    for L in cm.layers:
        if L["kind"] in ("conv", "tconv"):
            w[L["name"]]["bias"] = rng.normal(0, 0.1, size=L["cout"]).astype(np.float32)
        else:
            c = L["c"]
            g = 0.3 if L["name"].endswith("_3_bn") else 1.0
            w[L["name"]] = dict(gamma=(g * rng.uniform(0.5, 1.5, c)).astype(np.float32), beta=rng.normal(0, 0.1, c).astype(np.float32),
                                mean=rng.normal(0, 0.1, c).astype(np.float32), var=rng.uniform(0.5, 1.5, c).astype(np.float32))

    def run():
        return [np.asarray(x) for x in DeviceModel(spec, w, input_channels=in_ch, precision=precision).forward(imgs)]
    return run


def c4_run(seed):
    """run() of the benchmark's C4 UNet (16 -> 512 channels, output stride 4, pooled encoder convs whose full-resolution
    outputs are dead, three k3 decoder tconvs) at 2 x 256 x 256 with the benchmark's weights."""
    import bench
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    spec = bench.c4_spec()
    w = A.make_synthetic_weights(A.compile_model(spec, 1), bench.SEED)
    imgs = np.random.default_rng(seed).integers(0, 256, size=(2, 256, 256, 1), dtype=np.uint8)

    def run():
        return [np.asarray(x) for x in DeviceModel(spec, w, input_channels=1, precision=0).forward(imgs)]
    return run


def resnet50_run(B, seed):
    """run() of ResNet50 at B x 128 x 96 x 3 with 4x4 transposed-conv upsampling: residual 1x1 convs with the ADD in their
    epilogue, stride-2 1x1 convs, BN-folded 3x3 bottleneck convs of 64-512 channels, k4 transposed convs."""
    ups = dict(method="transposed_conv", skip_connections="concatenate", block_stride=2, filters=64, filters_rate=1,
               refine_convs=2, batch_norm=True, transposed_conv_kernel_size=4)
    cfg = dict(version="ResNet50", weights="frozen", max_stride=32, output_stride=4, upsampling=ups)
    heads = [dict(name="MultiInstanceConfmapsHead", channels=5, output_stride=4),
             dict(name="PartAffinityFieldsHead", channels=8, output_stride=8)]
    spec = dict(backbone="resnet", backbone_cfg=cfg, head_type="multi_instance", heads=heads, part_names=None, edges=None)
    imgs = np.random.default_rng(seed).integers(0, 256, size=(B, 128, 96, 3), dtype=np.uint8)
    return model_run(spec, 3, imgs, 0)
