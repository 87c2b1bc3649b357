"""Flow shift of the optical-flow trackers on the GPU (``sb_flow_*`` in include/sleap_b200.h, kernels in
sleap_b200/csrc/sb_flow.cu).

``DeviceFlow`` keeps the image pyramid and Scharr derivatives of the last ``ring`` frames on the device, keyed by
frame index, and shifts any number of (reference frame, point) pairs into the current frame with one launch: what
``cv2.calcOpticalFlowPyrLK`` computes per reference frame, with each frame's pyramid built once.
"""
import ctypes

import numpy as np

from sleap_b200 import _lib


class DeviceFlow:
    """Pyramidal Lucas-Kanade (``cv2.calcOpticalFlowPyrLK`` with ``winSize=(window_size, window_size)``,
    ``maxLevel=max_levels``, 30 iterations / eps 0.01) on gray frames resized by ``img_scale`` (1 or 0.5).

    Owns its own library handle (its own CUDA stream), so the tracker's thread never shares a handle with the
    inference that runs on another thread.  Calls on one ``DeviceFlow`` must come from one thread at a time.
    """

    def __init__(self, device=0, window_size: int = 21, max_levels: int = 3, img_scale: float = 1.0, ring: int = 7):
        self.handle = _lib.Handle(device)
        self.window_size, self.max_levels, self.img_scale = int(window_size), int(max_levels), float(img_scale)
        self.ring = 0
        self._id = None
        self._create(ring)

    def _create(self, ring: int):
        if self._id is not None:
            self.handle.call("sb_flow_destroy", self._id)
        fid = ctypes.c_int()
        self.handle.call("sb_flow_create", self.window_size, self.max_levels, ctypes.c_float(self.img_scale), int(ring),
                         ctypes.byref(fid))
        self._id, self.ring = fid.value, int(ring)

    def reserve(self, n_frames: int):
        """Make room for ``n_frames`` frames at once.  Growing the ring drops the frames it holds."""
        if n_frames > self.ring:
            self._create(n_frames)

    def add_frame(self, t: int, img: np.ndarray, replace: bool = True):
        """Upload frame ``t`` (uint8 (H, W), (H, W, 1) or BGR (H, W, 3)) and build its pyramid.  ``replace=False``
        keeps a frame already held under ``t`` and skips the upload."""
        img = np.ascontiguousarray(img, dtype=np.uint8)
        if img.ndim == 2:
            img = img[..., None]
        if img.ndim != 3:
            raise ValueError(f"frame of shape {img.shape}: expected (H, W) or (H, W, C)")
        self.handle.call("sb_flow_add_frame", self._id, int(t), _lib.ptr(img), img.shape[0], img.shape[1], img.shape[2],
                         int(bool(replace)))

    def shift(self, t: int, ref_t, pts: np.ndarray):
        """Move ``pts`` ((n, 2) float32, resized-frame pixels; point i belongs to frame ``ref_t[i]``) into frame ``t``.
        Returns (points (n, 2) float32, status (n,) uint8, err (n,) float32), as ``cv2.calcOpticalFlowPyrLK``."""
        pts = np.ascontiguousarray(pts, dtype=np.float32).reshape(-1, 2)
        ref_t = np.ascontiguousarray(ref_t, dtype=np.int64).reshape(-1)
        n = len(pts)
        if len(ref_t) != n:
            raise ValueError(f"{len(ref_t)} reference frame indices for {n} points")
        out, status, err = np.empty((n, 2), np.float32), np.empty(n, np.int32), np.empty(n, np.float32)
        self.handle.call("sb_flow_shift", self._id, int(t), n, _lib.ptr(ref_t), _lib.ptr(pts), _lib.ptr(out),
                         _lib.ptr(status), _lib.ptr(err))
        return out, status.astype(np.uint8), err

    def fetch_level(self, t: int, level: int):
        """(image (h, w) uint8, derivatives (h, w, 2) int16, number of levels) of pyramid level ``level`` of frame
        ``t``: what ``cv2.buildOpticalFlowPyramid(..., withDerivatives=True)`` returns for that level."""
        H, W, L = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        self.handle.call("sb_flow_fetch_level", self._id, int(t), int(level), None, None, ctypes.byref(H), ctypes.byref(W),
                         ctypes.byref(L))
        img, der = np.empty((H.value, W.value), np.uint8), np.empty((H.value, W.value, 2), np.int16)
        self.handle.call("sb_flow_fetch_level", self._id, int(t), int(level), _lib.ptr(img), _lib.ptr(der), ctypes.byref(H),
                         ctypes.byref(W), ctypes.byref(L))
        return img, der, L.value

    def close(self):
        if self._id is not None and self.handle is not None:
            self.handle.call("sb_flow_destroy", self._id)
            self._id = None
        if self.handle is not None:
            self.handle.close()
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
