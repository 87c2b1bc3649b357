"""The persistent fused first block k_conv01 (sb_conv01.cu): frame -> conv0 (1 -> 16) -> conv1 (16 -> 16) -> 2x2 max-pool,
on shapes that stress its 32x16 work items, its non-swizzled conv0 planes and its per-CTA item walk."""
from ctypes import byref, c_int, c_void_p

import numpy as np
import pytest
from numpy.testing import assert_allclose

pytestmark = pytest.mark.gpu


def _first_block(H, W, B, as_float, relu, seed):
    from sleap_b200.nn import oplist as ol
    rng = np.random.default_rng(seed)
    w0 = (rng.standard_normal((3, 3, 1, 16)) * 0.5).astype(np.float32); b0 = (rng.standard_normal(16) * 0.1).astype(np.float32)
    w1 = (rng.standard_normal((3, 3, 16, 16)) * np.sqrt(2.0 / 144)).astype(np.float32); b1 = (rng.standard_normal(16) * 0.1).astype(np.float32)
    eye = np.eye(16, dtype=np.float32).reshape(1, 1, 16, 16)
    blob = np.concatenate([w0.reshape(-1), b0, w1.reshape(-1), b1, eye.reshape(-1), np.zeros(16, np.float32)]).astype(np.float32)
    o1 = w0.size + 16
    o2 = o1 + w1.size + 16
    # buffers: 0 input, 1 conv0 out, 2 conv1 out (dead), 3 pooled, 4 pooled copied to f32 by a 1x1 identity conv
    recs = [ol.buffer_record(0, 1, 1, 0, 1), ol.buffer_record(1, 1, 16, 0, 0), ol.buffer_record(2, 1, 16, 0, 0), ol.buffer_record(3, 2, 16, 0, 0),
            ol.buffer_record(4, 2, 16, 1, 0), ol.preprocess_record(0, 1, 1.0, 4),
            ol.conv_record(0, 0, 1, 1, 0, 16, 3, 1, relu, 0, w0.size),
            ol.conv_record(1, 0, 16, 2, 0, 16, 3, 1, relu, o1, o1 + w1.size, pool_buf=3, pool_coff=0),
            ol.pool_record(2, 0, 16, 3, 0, fused=True),
            ol.conv_record(3, 0, 16, 4, 0, 16, 1, 1, False, o2, o2 + 256)]
    ops = np.ascontiguousarray(np.stack(recs).astype(np.int32))
    if as_float:
        imgs = rng.random((B, H, W, 1)).astype(np.float32); xin = imgs
    else:
        imgs = rng.integers(0, 256, size=(B, H, W, 1), dtype=np.uint8); xin = imgs.astype(np.float32) * np.float32(1.0 / 255.0)
    return ops, blob, imgs, xin, (w0, b0, w1, b1)


def _run(ops, blob, imgs, as_float, fused, monkeypatch):
    from sleap_b200 import _lib
    B, H, W = imgs.shape[:3]
    Hn, Wn = -(-H // 4) * 4, -(-W // 4) * 4
    monkeypatch.setenv("SB_FORCE_CONV01", "1" if fused else "0")
    h = _lib.Handle(0)
    mid = c_int(-1)
    h.call("sb_load_model", _lib.ptr(ops), ops.shape[0], _lib.ptr(blob), int(blob.size), 0, byref(mid))
    h.call("sb_model_configure", mid.value, B, H, W, 1)
    outs = []
    ids = np.asarray([4], np.int32)
    for _ in range(2):                                   # the second launch reuses the first one's configuration
        out = np.full((B, Hn // 2, Wn // 2, 16), np.nan, np.float32)
        ptrs = (c_void_p * 1)(out.ctypes.data)
        h.call("sb_model_forward", mid.value, _lib.ptr(imgs), int(not as_float), B, 1, _lib.ptr(ids), ptrs)
        outs.append(out)
    n = h.gpu_launches()
    h.close()
    return outs, n


def _reference(xin, weights, relu):
    import torch
    import torch.nn.functional as F
    w0, b0, w1, b1 = weights
    B, H, W = xin.shape[:3]
    Hn, Wn = -(-H // 4) * 4, -(-W // 4) * 4
    act = (lambda t: torch.relu(t)) if relu else (lambda t: t)
    x = torch.from_numpy(np.pad(xin, ((0, 0), (0, Hn - H), (0, Wn - W), (0, 0)))).half().float().permute(0, 3, 1, 2)
    y0 = act(F.conv2d(x, torch.from_numpy(w0).half().float().permute(3, 2, 0, 1), torch.from_numpy(b0), padding=1)).half().float()
    y1 = act(F.conv2d(y0, torch.from_numpy(w1).half().float().permute(3, 2, 0, 1), torch.from_numpy(b1), padding=1)).half().float()
    return F.max_pool2d(y1, 2).permute(0, 2, 3, 1).numpy()


CASES = {
    "one_tile": ((16, 32), 1, False, True),            # exactly one work item: pins the conv0 plane layout / descriptors
    "edges": ((44, 100), 3, False, True),              # partial items in both directions (H, W not multiples of 16 / 32)
    "smaller_than_tile": ((8, 12), 1, False, True),
    "pitch_516": ((36, 516), 3, False, False),         # uint8 rows whose pitch is not a multiple of 16 bytes, no ReLU
    "float": ((40, 72), 3, True, True),
    "float_no_relu_b1": ((30, 50), 1, True, False),
    "many_items": ((512, 640), 3, False, True),        # every CTA walks several items
}


@pytest.mark.parametrize("case", list(CASES))
def test_first_block_persistent(case, monkeypatch):
    (H, W), B, as_float, relu = CASES[case]
    ops, blob, imgs, xin, weights = _first_block(H, W, B, as_float, relu, seed=H * 31 + W + B)
    got, n_fused = _run(ops, blob, imgs, as_float, True, monkeypatch)
    sep, n_sep = _run(ops, blob, imgs, as_float, False, monkeypatch)
    assert n_fused < n_sep                               # the fused kernel really ran
    assert np.array_equal(got[0], got[1])                # the second launch computes the same thing
    want = _reference(xin, weights, relu)
    scale = max(1.0, float(np.abs(want).max()))
    assert_allclose(got[1], want, atol=2.5e-3 * scale, rtol=0)   # one fp16 ulp of the intermediate through 144 taps
    assert_allclose(got[1], sep[1], atol=2.5e-3 * scale, rtol=0)
    assert np.mean(np.abs(got[1] - want) > 1e-3 * scale) < 1e-3
