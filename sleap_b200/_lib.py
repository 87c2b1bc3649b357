"""ctypes binding of libsleapb200.so (the C-ABI declared in include/sleap_b200.h).

The library is built in-tree by ``sleap_b200/build.py`` (``__graft_entry__.build()``).  Loading
works without a GPU (symbols resolve); creating a handle without a CUDA device raises
``SleapB200Error`` -- the product path never falls back to the CPU.
"""
import ctypes
import os
import threading
from ctypes import POINTER, c_char_p, c_float, c_int, c_int32, c_int64, c_uint8, c_void_p

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsleapb200.so")


class SleapB200Error(RuntimeError):
    pass


_lib = None
_lock = threading.Lock()

c_float_p = POINTER(c_float)
c_int32_p = POINTER(c_int32)


class BottomUpParams(ctypes.Structure):
    _fields_ = [
        ("cms_buffer", c_int32), ("pafs_buffer", c_int32), ("offsets_buffer", c_int32),
        ("cm_output_stride", c_int32), ("paf_output_stride", c_int32),
        ("peak_threshold", c_float), ("refinement", c_int32), ("integral_patch_size", c_int32),
        ("n_nodes", c_int32), ("n_edges", c_int32),
        ("edges", c_void_p), ("sorted_edge_inds", c_void_p), ("n_sorted", c_int32),
        ("n_line_points", c_int32),
        ("max_edge_length_ratio", c_float), ("dist_penalty_weight", c_float), ("min_line_scores", c_float),
        ("min_instance_peaks", c_int32), ("input_scale", c_float),
        ("max_peaks_per_sample", c_int32), ("max_node_peaks", c_int32), ("max_instances", c_int32),
    ]


class MultiClassParams(ctypes.Structure):
    _fields_ = [
        ("cms_buffer", c_int32), ("class_maps_buffer", c_int32), ("offsets_buffer", c_int32),
        ("cm_output_stride", c_int32), ("class_maps_output_stride", c_int32),
        ("peak_threshold", c_float), ("refinement", c_int32), ("integral_patch_size", c_int32),
        ("n_nodes", c_int32), ("n_classes", c_int32), ("input_scale", c_float),
        ("max_peaks_per_sample", c_int32), ("max_node_peaks", c_int32),
    ]


MAX_CLASSES = 128           # SB_MAX_CLASSES (include/sleap_b200.h)


class GlobalParams(ctypes.Structure):
    _fields_ = [
        ("cms_buffer", c_int32), ("offsets_buffer", c_int32), ("output_stride", c_int32),
        ("peak_threshold", c_float), ("refinement", c_int32), ("integral_patch_size", c_int32),
        ("input_scale", c_float),
    ]


class CentroidParams(ctypes.Structure):
    _fields_ = [
        ("cms_buffer", c_int32), ("offsets_buffer", c_int32), ("output_stride", c_int32),
        ("peak_threshold", c_float), ("refinement", c_int32), ("integral_patch_size", c_int32),
        ("input_scale", c_float), ("max_peaks_per_sample", c_int32),
    ]


class TopdownParams(ctypes.Structure):
    _fields_ = [("centroid_model", c_int32), ("instance_model", c_int32), ("centroid", CentroidParams), ("instance", GlobalParams),
                ("crop_size", c_int32), ("max_instances", c_int32), ("max_centroids_per_frame", c_int32),
                ("max_crops_per_call", c_int32), ("precrop_resize", c_float)]


class TopdownMultiClassParams(ctypes.Structure):
    _fields_ = [("topdown", TopdownParams), ("tap_buffer", c_int32), ("tap_channel_offset", c_int32), ("tap_channels", c_int32),
                ("tap_planes", c_int32), ("n_classes", c_int32), ("num_fc_layers", c_int32), ("num_fc_units", c_int32),
                ("global_pool", c_int32), ("dense_weights", c_void_p), ("n_dense_weights", c_int64)]


MAX_DENSE_WIDTH = 4096      # SB_MAX_DENSE_WIDTH (include/sleap_b200.h)


class TrackerParams(ctypes.Structure):
    _fields_ = [("maker", c_int32), ("similarity", c_int32), ("match", c_int32), ("track_window", c_int32),
                ("max_tracks", c_int32), ("max_tracking", c_int32), ("min_match_points", c_int32),
                ("min_new_track_points", c_int32), ("robust", ctypes.c_double), ("cull_target", c_int32),
                ("cull_use_iou", c_int32), ("cull_iou_threshold", ctypes.c_double), ("oks_errors", c_void_p),
                ("n_oks_errors", c_int32), ("oks_score_weighting", c_int32), ("oks_normalization", c_int32),
                ("n_nodes", c_int32), ("max_instances", c_int32), ("track_table", c_int32)]


# name -> argtypes (restype is always int unless noted)
_SIGS = {
    "sb_version": [],
    "sb_create": [c_int, POINTER(c_void_p)],
    "sb_destroy": [c_void_p],
    "sb_synchronize": [c_void_p],
    "sb_gpu_launches": [c_void_p],
    "sb_set_stream": [c_void_p, c_void_p],
    "sb_find_local_peaks": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_int, c_int, c_void_p,
                            c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sb_find_global_peaks": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_float, c_int, c_int, c_void_p,
                             c_void_p, c_void_p],
    "sb_crop_centered": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                         c_int, c_int, c_void_p],
    "sb_crop_centered_resized": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int,
                                 c_int, c_int, c_float, c_void_p],
    "sb_score_paf_lines_batch": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                 c_void_p, c_int, c_int, c_int, c_int, c_float, c_float, c_int, c_void_p,
                                 c_void_p, c_void_p, c_void_p],
    "sb_paf_lines": [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                     c_int, c_int, c_int, c_float, c_float, c_void_p, c_void_p, c_void_p],
    "sb_integral_regression": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                               c_void_p],
    "sb_find_offsets_local_direction": [c_void_p, c_void_p, c_int, c_float, c_void_p],
    "sb_linear_sum_assignment_batch": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p,
                                       c_void_p, c_void_p, c_void_p],
    "sb_group_instances_batch": [c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                 c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int,
                                 c_float, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "sb_load_model": [c_void_p, c_void_p, c_int, c_void_p, c_int64, c_int, POINTER(c_int)],
    "sb_model_configure": [c_void_p, c_int, c_int, c_int, c_int, c_int],
    "sb_model_forward": [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    "sb_model_profile_ops": [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "sb_model_forward_times": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    "sb_bottomup_configure": [c_void_p, c_int, POINTER(BottomUpParams)],
    "sb_infer_bottomup": [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sb_infer_bottomup_dev": [c_void_p, c_int, c_void_p, c_int],
    "sb_bottomup_submit": [c_void_p, c_int, c_void_p, c_int, c_int],
    "sb_bottomup_collect": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sb_get_post_stream": [c_void_p, POINTER(c_void_p)],
    "sb_bottomup_device_records": [c_void_p, c_int, POINTER(c_void_p)],
    "sb_bottomup_fetch_graph": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                c_void_p, c_void_p, c_void_p, c_void_p],
    "sb_bottomup_from_maps": [c_void_p, POINTER(BottomUpParams), c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int,
                              c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                              c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "sb_multiclass_configure": [c_void_p, c_int, POINTER(MultiClassParams)],
    "sb_infer_multiclass": [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "sb_multiclass_submit": [c_void_p, c_int, c_void_p, c_int, c_int],
    "sb_multiclass_collect": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "sb_multiclass_from_maps": [c_void_p, POINTER(MultiClassParams), c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int,
                                c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sb_gather_init": [c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "sb_gather_connect": [c_void_p, c_int, c_void_p],
    "sb_gather_enabled": [c_void_p, c_int],
    "sb_gather_consume_dev": [c_void_p, c_int, c_int64],
    "sb_gather_window": [c_void_p, c_int, c_int64, POINTER(c_void_p), POINTER(c_int64)],
    "sb_gather_collect": [c_void_p, c_int, c_int64, c_int, c_void_p, c_void_p],
    "sb_gather_status": [c_void_p, c_int, c_void_p, c_void_p, c_void_p],
    "sb_bottomup_gathered": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    "sb_gather_close": [c_void_p, c_int],
    "sb_global_configure": [c_void_p, c_int, POINTER(GlobalParams)],
    "sb_infer_global": [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "sb_global_submit": [c_void_p, c_int, c_void_p, c_int, c_int],
    "sb_global_collect": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p],
    "sb_topdown_configure": [c_void_p, POINTER(TopdownParams), c_int, c_int, c_int, c_int],
    "sb_infer_topdown": [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sb_topdown_submit": [c_void_p, c_int, c_void_p, c_int, c_int],
    "sb_topdown_collect": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sb_topdown_gt_submit": [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int],
    "sb_topdown_gt_instances_configure": [c_void_p, POINTER(TopdownParams), c_int, c_int, c_int, c_int, c_int, c_int],
    "sb_topdown_gt_instances_submit": [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int],
    "sb_topdown_gt_instances_collect": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_void_p],
    "sb_topdown_multiclass_configure": [c_void_p, POINTER(TopdownMultiClassParams), c_int, c_int, c_int, c_int],
    "sb_infer_topdown_multiclass": [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p],
    "sb_topdown_multiclass_submit": [c_void_p, c_int, c_void_p, c_int, c_int],
    "sb_topdown_multiclass_collect": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                      c_void_p, c_void_p],
    "sb_topdown_multiclass_from_features": [c_void_p, POINTER(TopdownMultiClassParams), c_void_p, c_int, c_int, c_int, c_int,
                                            c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                            c_void_p, c_void_p, c_void_p, c_void_p],
    "sb_centroid_configure": [c_void_p, c_int, POINTER(CentroidParams)],
    "sb_infer_centroids": [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                           c_void_p],
    "sb_flow_create": [c_void_p, c_int, c_int, c_float, c_int, POINTER(c_int)],
    "sb_flow_add_frame": [c_void_p, c_int, c_int64, c_void_p, c_int, c_int, c_int, c_int],
    "sb_flow_shift": [c_void_p, c_int, c_int64, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p],
    "sb_flow_fetch_level": [c_void_p, c_int, c_int64, c_int, c_void_p, c_void_p, POINTER(c_int), POINTER(c_int),
                            POINTER(c_int)],
    "sb_flow_destroy": [c_void_p, c_int],
    "sb_tracker_create": [c_void_p, POINTER(TrackerParams), POINTER(c_int)],
    "sb_tracker_reset": [c_void_p, c_int],
    "sb_bottomup_attach_tracker": [c_void_p, c_int, c_int, c_int, ctypes.c_double, ctypes.c_double],
    "sb_bottomup_tracks": [c_void_p, c_int, c_int, c_int, c_void_p],
    "sb_bottomup_device_tracks": [c_void_p, c_int, c_int, c_void_p],
    "sb_topdown_attach_tracker": [c_void_p, c_int, c_int, ctypes.c_double, ctypes.c_double],
    "sb_topdown_tracks": [c_void_p, c_int, c_int, c_int, c_void_p],
    "sb_tracker_destroy": [c_void_p, c_int],
    "sb_track_instances": [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                           c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, POINTER(c_int32), POINTER(c_int32)],
}

EXPORTED_SYMBOLS = sorted(list(_SIGS.keys()) + ["sb_last_error"])


def lib():
    """Load (once) and return the ctypes library.  Raises if the extension is not built."""
    global _lib
    with _lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise SleapB200Error(
                    f"{LIB_PATH} is missing: build it with `python -m sleap_b200.build` "
                    "(or __graft_entry__.build()).  There is no CPU fallback.")
            L = ctypes.CDLL(LIB_PATH)
            for name, args in _SIGS.items():
                fn = getattr(L, name)
                fn.argtypes = args
                fn.restype = c_int
            L.sb_last_error.argtypes = [c_void_p]
            L.sb_last_error.restype = c_char_p
            _lib = L
    return _lib


def ptr(a):
    """Host pointer of a C-contiguous numpy array (None -> NULL)."""
    if a is None:
        return None
    assert a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(c_void_p)


def f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


class Handle:
    """One libsleapb200 handle (= one GPU)."""

    def __init__(self, device_id=0):
        self._h = c_void_p()
        rc = lib().sb_create(int(device_id), ctypes.byref(self._h))
        if rc != 0:
            raise SleapB200Error(f"sb_create failed ({rc}): {lib().sb_last_error(None).decode()}")
        self.device_id = int(device_id)

    @property
    def h(self):
        return self._h

    def check(self, rc, what=""):
        if rc != 0:
            raise SleapB200Error(f"{what} failed ({rc}): {lib().sb_last_error(self._h).decode()}")

    def call(self, name, *args):
        self.check(getattr(lib(), name)(self._h, *args), name)

    def gpu_launches(self):
        return lib().sb_gpu_launches(self._h)

    def synchronize(self):
        self.call("sb_synchronize")

    def set_stream(self, stream_ptr):
        self.call("sb_set_stream", c_void_p(stream_ptr))

    def close(self):
        if self._h:
            lib().sb_destroy(self._h)
            self._h = c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


_default = {}


def default_handle(device_id=None):
    """Process-wide handle on ``device_id`` (default: LOCAL_RANK or 0)."""
    if device_id is None:
        device_id = int(os.environ.get("LOCAL_RANK", "0"))
    with _lock:
        h = _default.get(device_id)
    if h is None:
        h = Handle(device_id)
        with _lock:
            _default[device_id] = h
    return h
