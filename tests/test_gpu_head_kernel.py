"""k_head_1x1 (sb_conv_tc.cu), the kernel that writes every fp32 head output, against float64.

Each model is an op list: input -> 3x3 conv 1 -> C (fp16 buffer) -> one or more 1x1 heads reading channels
[in_coff, in_coff + cin) of that buffer into fp32 buffers.  Both the fp16 intermediate and the head outputs are read
back, and the reference is x16 @ W16 + b (+ ReLU) in float64 on the exact fp16 operands the kernel consumes.  The bound
is per element, |got - ref| <= 2^-19 * (sum_i |x_i w_i| + |b|) + 1e-7: loose for fp32 accumulation, but a dropped
K chunk, a stale ring slot, a wrong bias column or a shifted tail row is far outside it.

SB_DEBUG=1 makes head_launch print each head's launch shape once, so every case checks that k_head_1x1 really ran (or,
for shapes it cannot hold, that the op fell back to the implicit-GEMM conv kernel)."""
import re
from ctypes import byref, c_int, c_void_p

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

HEAD_RE = re.compile(r"\[sb_conv_tc\] head k_head_1x1: Cin (\d+) Cout (\d+) NT (\d+) KCH (\d+) n_ring (\d+) smem (\d+)")
SMEM_CAP = 200 * 1024


def head_fits(cin, cout):
    """Whether k_head_1x1 can hold a 1x1 head at all: the fp16 weight bank (<= 160 KB), the output staging, the bias and
    a ring of two staged items per warp fit in the 200 KB the kernel is configured for.  Otherwise the op runs on the
    implicit-GEMM conv kernel.  (How deep the ring is beyond 2 is a tuning choice the tests leave open.)"""
    nt, kch = (cout + 7) // 8, min(cin, 128)
    cout_pad = (cout + 15) // 16 * 16
    fixed = 8 * nt * (cin + 8) * 2 + 8 * 16 * (8 * nt + 1) * 4 + 8 * nt * 4
    stage = 8 * 16 * (kch + 8) * 2
    return cout_pad * (cin + 8) * 2 <= 160 * 1024 and fixed + 2 * stage <= SMEM_CAP


def _run_heads(cin, heads, B, hw, ctot=None, in_coff=0, seed=0):
    """heads: list of (out buffer, out_coff, cout, relu); out buffer i >= 2 has the channel count given by its heads.
    Returns (x16 as float32 [npix, ctot], {buffer: output [npix, C]}, [(w, b) per head])."""
    from sleap_b200 import _lib
    from sleap_b200.nn import oplist as ol
    rng = np.random.default_rng(seed)
    H, W = hw
    ctot = ctot or cin
    out_C = {}
    for ob, oc, cout, _ in heads:
        out_C[ob] = max(out_C.get(ob, 0), oc + cout)
    recs = [ol.buffer_record(0, 1, 1, 0, 1), ol.buffer_record(1, 1, ctot, 0, 0)]
    recs += [ol.buffer_record(ob, 1, c, 1, 0) for ob, c in sorted(out_C.items())]
    recs.append(ol.preprocess_record(0, 1, 1.0, 1))
    w0 = (rng.standard_normal((3, 3, 1, ctot)) * 0.5).astype(np.float32)
    b0 = rng.normal(0, 0.1, ctot).astype(np.float32)
    blob = [w0.reshape(-1), b0]
    off = w0.size + ctot
    recs.append(ol.conv_record(0, 0, 1, 1, 0, ctot, 3, 1, False, 0, w0.size))     # signed activations
    params = []
    for ob, oc, cout, relu in heads:
        w = (rng.standard_normal((cin, cout)) * np.sqrt(2.0 / cin)).astype(np.float32)
        b = rng.normal(0, 0.3, cout).astype(np.float32)
        recs.append(ol.conv_record(1, in_coff, cin, ob, oc, cout, 1, 1, relu, off, off + w.size))
        blob += [w.reshape(-1), b]
        off += w.size + cout
        params.append((w, b))
    blob = np.concatenate(blob).astype(np.float32)
    ops = np.ascontiguousarray(np.stack(recs).astype(np.int32))
    imgs = rng.uniform(0, 1, size=(B, H, W, 1)).astype(np.float32)
    h = _lib.Handle(0)
    try:
        mid = c_int(-1)
        h.call("sb_load_model", _lib.ptr(ops), ops.shape[0], _lib.ptr(blob), int(blob.size), 0, byref(mid))
        h.call("sb_model_configure", mid.value, B, H, W, 1)
        ids = [1] + sorted(out_C)
        outs = [np.zeros((B, H, W, ctot), np.float32)] + [np.zeros((B, H, W, out_C[ob]), np.float32) for ob in sorted(out_C)]
        ptrs = (c_void_p * len(ids))(*[o.ctypes.data for o in outs])
        h.call("sb_model_forward", mid.value, _lib.ptr(imgs), 0, B, len(ids), _lib.ptr(np.asarray(ids, np.int32)), ptrs)
    finally:
        h.close()
    n = B * H * W
    return outs[0].reshape(n, ctot), {ob: o.reshape(n, -1) for ob, o in zip(sorted(out_C), outs[1:])}, params


def _check(x16, outs, heads, params, cin, in_coff=0):
    x = x16[:, in_coff:in_coff + cin].astype(np.float64)
    for (ob, oc, cout, relu), (w, b) in zip(heads, params):
        w16 = w.astype(np.float16).astype(np.float64)
        ref = x @ w16 + b.astype(np.float64)
        bound = 2.0 ** -19 * (np.abs(x) @ np.abs(w16) + np.abs(b)) + 1e-7
        if relu:
            ref = np.maximum(ref, 0.0)
        got = outs[ob][:, oc:oc + cout].astype(np.float64)
        err = np.abs(got - ref)
        bad = np.argwhere(err > bound)
        assert bad.size == 0, (f"head {cin}->{cout} relu={relu}: {len(bad)} elements off, first (pixel, channel) {tuple(bad[0])}: "
                               f"got {got[tuple(bad[0])]}, want {ref[tuple(bad[0])]}")
        assert relu or np.abs(ref).max() > 0


def _check_ran(err, cin, couts):
    """couts: the heads in op-list order (op 0 is PREPROCESS, op 1 the 3x3 conv, head j is op 2 + j).  Each head that
    fits printed its k_head_1x1 launch (NT, KCH by its shape, a ring of 2-8 slots, at most 200 KB) and was not timed as a
    conv launch; each head that does not fit printed no launch and was timed as a conv launch of its own op."""
    seen = {}
    for m in HEAD_RE.finditer(err):
        c_in, c_out, nt, kch, ring, smem = map(int, m.groups())
        if c_in == cin:
            seen[c_out] = (nt, kch, ring, smem)
    for j, cout in enumerate(couts):
        conv_line = re.search(rf"\[sb_conv_tc\] op {2 + j} launch 0: .* -> (streaming|resident)", err)
        if not head_fits(cin, cout):
            assert cout not in seen, (cin, cout, seen.get(cout))
            assert conv_line, f"head {cin}->{cout} (op {2 + j}) never reached the conv kernel"
            continue
        assert cout in seen, f"k_head_1x1 did not run for {cin}->{cout}"
        assert not conv_line, conv_line.group(0)
        nt, kch, ring, smem = seen[cout]
        assert (nt, kch) == ((cout + 7) // 8, min(cin, 128)), seen[cout]
        assert 2 <= ring <= 8 and smem <= SMEM_CAP, seen[cout]


COUTS = (1, 8, 13, 16, 17, 24, 25, 32)
# (B, H, W): pixel counts 1920 (0 mod 16), 289 (1 mod 16), 1023 (15 mod 16), 15 (fewer than one tile)
GEOMS = {"full": (2, 24, 40), "tail1": (1, 17, 17), "tail15": (1, 31, 33), "tiny": (1, 3, 5)}


@pytest.mark.parametrize("geom", list(GEOMS))
@pytest.mark.parametrize("cin", [16, 32, 64, 128, 256, 384, 512, 1536, 2048, 2432])
def test_head_shapes(cin, geom, monkeypatch, capfd):
    """Every NT (1-4) x KCH (16-128) instantiation, one and several passes (Cin >= 256), linear stores, tail tiles, rings
    of 2 to 8 slots.  The wide inputs are the shapes whose weight bank leaves less than 110 KB for the ring: 1536 x 25-32
    and 2432 x 17-24 still fit a ring of 2 in 200 KB and must run on k_head_1x1, 2048-2432 x 25-32 fit none and must run
    on the conv kernel."""
    if cin in (1536, 2432):
        assert head_fits(cin, 32 if cin == 1536 else 24)
    if cin >= 2048:
        assert not head_fits(cin, 25)
    if geom == "tiny" and cin not in (16, 128, 512, 2048):
        pytest.skip("the 15-pixel frame runs on a subset of the input widths")
    monkeypatch.setenv("SB_DEBUG", "1")
    B, H, W = GEOMS[geom]
    flip = geom in ("tail1", "tiny")
    heads = [(2 + j, 0, cout, (j % 2 == 1) != flip) for j, cout in enumerate(COUTS)]
    capfd.readouterr()
    x16, outs, params = _run_heads(cin, heads, B, (H, W), seed=cin + len(geom))
    _check_ran(capfd.readouterr().err, cin, COUTS)
    _check(x16, outs, heads, params, cin)


@pytest.mark.parametrize("cin,ctot,in_coff", [(64, 96, 32), (128, 160, 16), (256, 272, 8)])
def test_head_channel_slice_and_shared_output(cin, ctot, in_coff, monkeypatch, capfd):
    """Heads reading a channel slice of a wider fp16 buffer, two pairs of heads sharing one fp32 buffer each (out_Ctot !=
    Cout: the NT <= 2 store path for 13 and 1 outputs, the NT > 2 path for 24 and 32), and one head owning its buffer."""
    monkeypatch.setenv("SB_DEBUG", "1")
    heads = [(2, 0, 13, False), (2, 13, 24, True), (3, 0, 1, True), (3, 1, 32, False), (4, 0, 8, False)]
    capfd.readouterr()
    x16, outs, params = _run_heads(cin, heads, 2, (21, 37), ctot=ctot, in_coff=in_coff, seed=ctot)
    _check_ran(capfd.readouterr().err, cin, (13, 24, 1, 32, 8))
    _check(x16, outs, heads, params, cin, in_coff)


def test_head_large_frame(monkeypatch, capfd):
    """2 x 256 x 256 pixels, 256 input channels: every warp walks several (tile, pass) items and its ring wraps."""
    monkeypatch.setenv("SB_DEBUG", "1")
    heads = [(2, 0, 13, False), (2, 13, 24, False), (3, 0, 32, True)]
    capfd.readouterr()
    x16, outs, params = _run_heads(256, heads, 2, (256, 256), seed=5)
    _check_ran(capfd.readouterr().err, 256, (13, 24, 32))
    _check(x16, outs, heads, params, 256)


def test_head_precision2_split_input(monkeypatch, capfd):
    """Precision 2: the PAF head reads 128 logical channels stored as 384 fp16 planes [lo | hi | hi], three 128-channel
    passes.  The network is checked against the fp32 oracle network at the precision-2 bar (1e-4 of the map maximum)."""
    from oracle import convnet, preprocess as opre
    from sleap_b200.nn import architectures as A
    from sleap_b200.nn.model import DeviceModel
    monkeypatch.setenv("SB_DEBUG", "1")
    spec = dict(backbone="unet", head_type="multi_instance", part_names=None, edges=None,
                backbone_cfg=dict(filters=16, filters_rate=2, max_stride=16, output_stride=4, middle_block=True, up_interpolate=False),
                heads=[dict(name="MultiInstanceConfmapsHead", channels=13, output_stride=4),
                       dict(name="PartAffinityFieldsHead", channels=24, output_stride=8)])
    cm = A.compile_model(spec, 1)
    w = A.make_synthetic_weights(cm, 8)
    rng = np.random.default_rng(9)
    for L in cm.layers:
        if L["kind"] in ("conv", "tconv"):
            w[L["name"]]["bias"] = rng.normal(0, 0.1, size=L["cout"]).astype(np.float32)
    imgs = rng.integers(0, 256, size=(2, 144, 112, 1), dtype=np.uint8)
    capfd.readouterr()
    got = DeviceModel(spec, w, input_channels=1, precision=2).forward(imgs)
    err = capfd.readouterr().err
    shapes = {(int(m.group(1)), int(m.group(2))): (int(m.group(4)), int(m.group(5))) for m in HEAD_RE.finditer(err)}
    assert (384, 24) in shapes and shapes[(384, 24)][0] == 128, shapes      # split input, three passes
    want = convnet.model_forward(opre.preprocess(imgs, ensure_gray=True, input_scale=1.0, pad_stride=16), spec, w)
    for g, x in zip(got, want):
        assert g.shape == x.shape
        rel = float(np.abs(g - x).max() / max(1.0, np.abs(x).max()))
        assert rel <= 1e-4, rel
