"""The halo form of the tensor-core convolution (k_conv_wg_h, form 2 in sb_conv_tc.cu) is byte-identical to the streaming
form 0.

SB_FORCE_VARIANT=2 forces the halo form where it is eligible (3x3 stride-1 convs, C_in <= 64, C_out 16..64 in the fp16
fast-epilogue shape); each case asserts from the SB_DEBUG autotune lines that it actually ran, and compares the raw bits
of every requested tensor with the SB_FORCE_VARIANT=0 run."""
from ctypes import byref, c_int, c_void_p

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _halo_vs_streaming(run, monkeypatch, capfd):
    """run() with the halo form forced and with the streaming form forced; the outputs must be equal bit for bit."""
    monkeypatch.setenv("SB_DEBUG", "1")
    outs = {}
    for f in ("0", "2"):
        monkeypatch.setenv("SB_FORCE_VARIANT", f)
        capfd.readouterr()
        outs[f] = run()
        err = capfd.readouterr().err
        if f == "2":
            assert "-> halo" in err, "the halo form never ran"
    for a, b in zip(outs["0"], outs["2"]):
        assert _same_bits(a, b), float(np.abs(a.astype(np.float64) - b).max())
    return outs["0"]


def _layer(cin, cout, hw, B, relu=True, pool=None, out_slice=False, in_slice=False):
    """frame -> conv0 (3x3, 1 -> cin) -> conv1 (3x3, cin -> cout, the layer under test; fp16 output).  pool: None, "dead"
    (fused 2x2 max-pool, only the pooled tensor requested: conv1's own stores are skipped) or "alive" (both requested).
    out_slice / in_slice: conv1 writes / reads a channel slice of a wider concat buffer."""
    from sleap_b200 import _lib
    from sleap_b200.nn import oplist as ol
    rng = np.random.default_rng(7 * cin + cout)
    H, W = hw
    in_off, in_tot = (8, cin + 24) if in_slice else (0, cin)
    out_off, out_tot = (16, cout + 48) if out_slice else (0, cout)
    recs = [ol.buffer_record(0, 1, 1, 0, 1), ol.buffer_record(1, 1, in_tot, 0, 0), ol.buffer_record(2, 1, out_tot, 0, 0)]
    if pool:
        recs.append(ol.buffer_record(3, 2, cout, 0, 0))
    recs.append(ol.preprocess_record(0, 1, 1.0, 2 if pool else 1))
    w0 = (rng.standard_normal((3, 3, 1, cin)) * 0.5).astype(np.float32)
    b0 = rng.normal(0, 0.1, cin).astype(np.float32)
    w1 = (rng.standard_normal((3, 3, cin, cout)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)
    b1 = rng.normal(0, 0.1, cout).astype(np.float32)
    blob = np.concatenate([w0.reshape(-1), b0, w1.reshape(-1), b1]).astype(np.float32)
    o1 = w0.size + cin
    recs.append(ol.conv_record(0, 0, 1, 1, in_off, cin, 3, 1, True, 0, w0.size))
    recs.append(ol.conv_record(1, in_off, cin, 2, out_off, cout, 3, 1, relu, o1, o1 + w1.size, pool_buf=3 if pool else -1))
    if pool:
        recs.append(ol.pool_record(2, out_off, cout, 3, 0, fused=True))
    ops = np.ascontiguousarray(np.stack(recs).astype(np.int32))
    imgs = rng.uniform(0, 1, size=(B, H, W, 1)).astype(np.float32)
    ids = [3] if pool == "dead" else ([2, 3] if pool == "alive" else [2])

    def run():
        h = _lib.Handle(0)
        mid = c_int(-1)
        h.call("sb_load_model", _lib.ptr(ops), ops.shape[0], _lib.ptr(blob), int(blob.size), 0, byref(mid))
        h.call("sb_model_configure", mid.value, B, H, W, 1)
        shapes = {2: (B, H, W, out_tot), 3: (B, H // 2, W // 2, cout)}
        outs = [np.zeros(shapes[i], np.float32) for i in ids]
        ptrs = (c_void_p * len(ids))(*[o.ctypes.data for o in outs])
        h.call("sb_model_forward", mid.value, _lib.ptr(imgs), 0, B, len(ids), _lib.ptr(np.asarray(ids, np.int32)), ptrs)
        h.close()
        # only conv1's slice of a concat buffer is written
        return [o[..., out_off:out_off + cout] if i == 2 else o for i, o in zip(ids, outs)]
    return run


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("cin,cout", [(16, 16), (16, 32), (24, 48), (32, 32), (32, 64), (48, 16), (64, 64), (64, 32)])
def test_halo_single_layers(cin, cout, B, monkeypatch, capfd):
    """Maps that are not a multiple of the 16 x 16 / 16 x 8 item in either direction."""
    out = _halo_vs_streaming(_layer(cin, cout, (40, 53), B), monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


@pytest.mark.parametrize("cin,cout", [(16, 32), (64, 64)])
def test_halo_no_relu(cin, cout, monkeypatch, capfd):
    out = _halo_vs_streaming(_layer(cin, cout, (24, 40), 2, relu=False), monkeypatch, capfd)
    assert (out[0] < 0).any()


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("pool", ["dead", "alive"])
@pytest.mark.parametrize("cin,cout", [(16, 16), (32, 32), (24, 48), (64, 64)])
def test_halo_pooled(cin, cout, pool, B, monkeypatch, capfd):
    """Fused 2x2 max-pool with conv1's own output dead (stores skipped) and requested; 36 x 50 leaves partial items."""
    out = _halo_vs_streaming(_layer(cin, cout, (36, 50), B, pool=pool), monkeypatch, capfd)
    assert all(np.abs(o).max() > 0 for o in out)


@pytest.mark.parametrize("cin,cout,hw", [(16, 32, (6, 10)), (64, 64, (4, 4)), (32, 48, (14, 12))])
def test_halo_smaller_than_one_item(cin, cout, hw, monkeypatch, capfd):
    out = _halo_vs_streaming(_layer(cin, cout, hw, 3), monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


@pytest.mark.parametrize("cin,cout,pool", [(32, 32, None), (16, 64, "alive"), (48, 32, None)])
def test_halo_concat_slices(cin, cout, pool, monkeypatch, capfd):
    """conv1 reads a channel slice of one concat buffer and writes a slice of another."""
    out = _halo_vs_streaming(_layer(cin, cout, (40, 48), 2, pool=pool, out_slice=True, in_slice=True), monkeypatch, capfd)
    assert np.abs(out[0]).max() > 0


def test_halo_c4_unet(monkeypatch, capfd):
    """The benchmark's C4 UNet (16 -> 512 channels, output stride 4, pooled encoder convs whose full-resolution outputs are
    dead) at 2 x 256 x 256: every output map byte-identical."""
    import bench
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    spec = bench.c4_spec()
    w = A.make_synthetic_weights(A.compile_model(spec, 1), bench.SEED)
    imgs = np.random.default_rng(23).integers(0, 256, size=(2, 256, 256, 1), dtype=np.uint8)

    def run():
        return [np.asarray(x) for x in DeviceModel(spec, w, input_channels=1, precision=0).forward(imgs)]
    out = _halo_vs_streaming(run, monkeypatch, capfd)
    assert all(np.isfinite(o).all() and np.abs(o).max() > 0 for o in out)
