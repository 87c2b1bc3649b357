"""Drop-in for ``sleap.nn.peak_finding`` (reference: sleap/nn/peak_finding.py).

Same function names, argument order and return tuples; inputs/outputs are NumPy arrays
(the reference returns tf.Tensors).  Every function runs as sm_90a CUDA kernels behind the
C-ABI (sleap_b200/csrc/sb_post.cu); nothing is computed on the CPU.
"""
from ctypes import c_int32, byref

import numpy as np

from sleap_b200 import _lib
from sleap_b200._lib import f32, i32, ptr

REFINE = {None: 0, "none": 0, "integral": 1, "local": 2}


def _refine_code(refinement):
    return REFINE.get(refinement, 0)  # unknown strings behave like None (peak_finding.py:381-386)


def find_offsets_local_direction(centered_patches, delta=0.25, handle=None):
    """sleap/nn/peak_finding.py:78-132.  (N,3,3,1) -> (N,2) [dx, dy]."""
    h = handle or _lib.default_handle()
    p = f32(centered_patches).reshape(-1, 3, 3, 1)
    out = np.zeros((p.shape[0], 2), np.float32)
    h.call("sb_find_offsets_local_direction", ptr(p), p.shape[0], float(delta), ptr(out))
    return out


def integral_regression(cms, xv, yv, handle=None):
    """sleap/nn/peak_finding.py:311-334.  cms (N,h,w,C) -> (x_hat, y_hat) each (N,C)."""
    h = handle or _lib.default_handle()
    cms = f32(cms)
    N, Hh, Ww, C = cms.shape
    xv, yv = f32(xv).reshape(-1), f32(yv).reshape(-1)
    x_hat = np.zeros((N, C), np.float32)
    y_hat = np.zeros((N, C), np.float32)
    h.call("sb_integral_regression", ptr(cms), N, Hh, Ww, C, ptr(xv), ptr(yv), ptr(x_hat), ptr(y_hat))
    return x_hat, y_hat


def _global(cms, threshold, refinement, patch, offsets, handle):
    h = handle or _lib.default_handle()
    cms = f32(cms)
    B, H, W, C = cms.shape
    off = None if offsets is None else f32(offsets).reshape(B, H, W, 2 * C)
    pts = np.zeros((B, C, 2), np.float32)
    vals = np.zeros((B, C), np.float32)
    h.call("sb_find_global_peaks", ptr(cms), B, H, W, C, float(threshold), _refine_code(refinement), int(patch),
           ptr(off), ptr(pts), ptr(vals))
    return pts, vals


def find_global_peaks_rough(cms, threshold=0.1, handle=None):
    """sleap/nn/peak_finding.py:193-246."""
    return _global(cms, threshold, None, 5, None, handle)


def find_global_peaks(cms, threshold=0.2, refinement=None, integral_patch_size=5, handle=None):
    """sleap/nn/peak_finding.py:337-420."""
    return _global(cms, threshold, refinement, integral_patch_size, None, handle)


def find_global_peaks_integral(cms, crop_size=5, threshold=0.2, handle=None):
    """sleap/nn/peak_finding.py:423-448."""
    return find_global_peaks(cms, threshold=threshold, refinement="integral", integral_patch_size=crop_size,
                             handle=handle)


def find_global_peaks_with_offsets(cms, offsets, threshold=0.2, handle=None):
    """sleap/nn/peak_finding.py:566-643."""
    return _global(cms, threshold, None, 5, offsets, handle)


def _local(cms, threshold, refinement, patch, offsets, handle, max_peaks_per_sample=None):
    h = handle or _lib.default_handle()
    cms = f32(cms)
    B, H, W, C = cms.shape
    if max_peaks_per_sample is None:
        # the reference is unbounded; a strict 8-neighbour maximum occupies a 2x2 block alone
        max_peaks_per_sample = max(1, ((H + 1) // 2) * ((W + 1) // 2) * C)
    cap = B * max_peaks_per_sample
    off = None if offsets is None else f32(offsets).reshape(B, H, W, 2 * C)
    pts = np.zeros((cap, 2), np.float32)
    vals = np.zeros((cap,), np.float32)
    si = np.zeros((cap,), np.int32)
    ci = np.zeros((cap,), np.int32)
    n = c_int32(0)
    flags = np.zeros((B,), np.int32)
    h.call("sb_find_local_peaks", ptr(cms), B, H, W, C, float(threshold), _refine_code(refinement), int(patch),
           ptr(off), int(max_peaks_per_sample), ptr(pts), ptr(vals), ptr(si), ptr(ci), byref(n), ptr(flags))
    k = n.value
    return pts[:k].copy(), vals[:k].copy(), si[:k].copy(), ci[:k].copy()


def find_local_peaks_rough(cms, threshold=0.2, handle=None):
    """sleap/nn/peak_finding.py:249-308."""
    return _local(cms, threshold, None, 5, None, handle)


def find_local_peaks(cms, threshold=0.2, refinement=None, integral_patch_size=5, handle=None):
    """sleap/nn/peak_finding.py:451-532."""
    return _local(cms, threshold, refinement, integral_patch_size, None, handle)


def find_local_peaks_integral(cms, crop_size=5, threshold=0.2, handle=None):
    """sleap/nn/peak_finding.py:535-563."""
    return find_local_peaks(cms, threshold=threshold, refinement="integral", integral_patch_size=crop_size,
                            handle=handle)


def find_local_peaks_with_offsets(cms, offsets, threshold=0.2, handle=None):
    """sleap/nn/peak_finding.py:646-707."""
    return _local(cms, threshold, None, 5, offsets, handle)


def crop_bboxes(images, bboxes, sample_inds, handle=None):
    """sleap/nn/peak_finding.py:135-190 for centred boxes (as produced by make_centered_bboxes):
    bboxes (n,4) y1,x1,y2,x2; crop size from the first box."""
    h = handle or _lib.default_handle()
    images = np.ascontiguousarray(images)
    bboxes = f32(bboxes).reshape(-1, 4)
    n = bboxes.shape[0]
    ch = int(np.round((bboxes[0, 2] - bboxes[0, 0]) + 1))
    cw = int(np.round((bboxes[0, 3] - bboxes[0, 1]) + 1))
    cent = np.stack([(bboxes[:, 1] + bboxes[:, 3]) * np.float32(0.5),
                     (bboxes[:, 0] + bboxes[:, 2]) * np.float32(0.5)], axis=1).astype(np.float32)
    is_u8 = images.dtype == np.uint8
    if not is_u8:
        images = f32(images)
    B, H, W, C = images.shape
    out = np.zeros((n, ch, cw, C), images.dtype)
    h.call("sb_crop_centered", ptr(images), int(is_u8), B, H, W, C, ptr(cent), ptr(i32(sample_inds)), n, ch, cw,
           ptr(out))
    return out
