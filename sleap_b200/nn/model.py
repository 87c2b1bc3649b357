"""Device model: compiled op-list + weights resident on one GPU (replaces the Keras model of
sleap/nn/model.py:312-364 and ``tf.keras.models.load_model`` at sleap/nn/inference.py:3203-3213)."""
import ctypes
import functools
import json
import os
from ctypes import c_int, c_void_p

import numpy as np

from sleap_b200 import _lib
from sleap_b200._lib import ptr
from sleap_b200.nn import architectures as arch

PRECISION_FP16 = 0   # fp16 activations, tensor-core convs, fp32 accumulate, fp32 head outputs
PRECISION_FP32 = 1   # fp32 CUDA-core path (strict parity with the fp32 reference)
PRECISION_SPLIT = 2  # fp32-grade results on the fp16 tensor cores: activations and weights as hi + lo fp16 pairs, three
                     # MMAs per product term (hi*Wh + lo*Wh + hi*Wl), fp32 accumulate; ~1e-6 of the fp32 path


class DeviceModel:
    def __init__(self, spec, weights, input_channels=1, input_scale=1.0, pad_to_stride=None,
                 precision=PRECISION_FP16, handle=None):
        self.handle = handle or _lib.default_handle()
        self.spec = spec
        self.precision = precision
        self.input_scale = float(input_scale)
        self.cm = arch.compile_model(spec, input_channels, input_scale, pad_to_stride, split=(precision == PRECISION_SPLIT))
        blob = self.cm.pack_weights(weights)
        # dense layers of "vector" heads (heads.py:431-460): run on the host by forward(), packed for the device by the
        # top-down multi-class step (pack_dense_weights)
        self.dense_weights = {k: {kk: np.asarray(vv, np.float32) for kk, vv in v.items()} for k, v in weights.items()
                              if k.startswith("pre_classification") or k in self.cm.vector_taps}
        ops = self.cm.ops_array()
        mid = c_int(-1)
        self.handle.call("sb_load_model", ptr(ops), ops.shape[0], ptr(blob), int(blob.size), int(precision),
                         ctypes.byref(mid))
        self.model_id = mid.value
        self.configured_for = None
        # (configure call, chain_key) of the post-processing chain the device model runs (None: none, or not known).
        # Any configure call drops the previous chain, the network's included (include/sleap_b200.h).
        self.chain = None
        self.peer_gather = None      # sleap_b200.parallel.PeerGather once the multi-GPU record exchange is connected

    def head_buffer(self, name):
        return self.cm.head_buffers[name]

    def configure(self, max_batch, H, W, C_in):
        key = (int(max_batch), int(H), int(W), int(C_in))
        if self.configured_for != key:
            self.handle.call("sb_model_configure", self.model_id, *key)
            self.configured_for = key
            self.chain = None
        return self

    def configure_chain(self, fn_name, params, *arrays):
        """Configures the post-processing chain with ``fn_name`` (``sb_bottomup_configure``, ``sb_multiclass_configure``,
        ``sb_global_configure`` or ``sb_centroid_configure``) unless the model already runs it with these parameters;
        ``arrays`` are the ones the pointer fields of ``params`` point to."""
        record = (fn_name, chain_key(params, *arrays))
        if self.chain != record:
            self.chain = None                     # a refused call may have dropped the previous chain
            self.handle.call(fn_name, self.model_id, ctypes.byref(params))
            self.chain = record
        return self

    def net_hw(self, H, W):
        """Network input size after resize + pad (resizing.py:71-106, :34-68)."""
        if self.input_scale != 1.0:
            W, H = int(np.float32(W) * np.float32(self.input_scale)), int(np.float32(H) * np.float32(self.input_scale))
        ms = self.cm.max_stride
        return -(-H // ms) * ms, -(-W // ms) * ms

    def forward(self, images, head_names=None):
        """images (B,H,W,C) uint8 or float32 in [0,1] -> list of head outputs (NHWC float32)."""
        images = np.ascontiguousarray(images)
        is_u8 = images.dtype == np.uint8
        if not is_u8:
            images = np.ascontiguousarray(images, dtype=np.float32)
        B, H, W, C = images.shape
        if self.configured_for is None or self.configured_for[0] < B or self.configured_for[1:] != (H, W, C):
            self.configure(B, H, W, C)
        head_names = head_names or [h["name"] for h in self.spec["heads"] if not h.get("vector")]
        nh, nw = self.net_hw(H, W)
        outs, ids = [], []
        for n in head_names:
            st = self.cm.head_strides[n]
            if n in self.cm.vector_taps:          # "vector" head: fetch the feature map it taps, dense layers on the host
                outs.append(np.zeros((B, nh // st, nw // st, self.cm.vector_taps[n]["buf_C"]), np.float32))
                ids.append(self.cm.vector_taps[n]["buf"])
                continue
            ch = next(h["channels"] for h in self.spec["heads"] if h["name"] == n)
            outs.append(np.zeros((B, nh // st, nw // st, ch), np.float32))
            ids.append(self.cm.head_buffers[n])
        ids_a = np.asarray(ids, np.int32)
        ptrs = (c_void_p * len(outs))(*[o.ctypes.data for o in outs])
        self.handle.call("sb_model_forward", self.model_id, ptr(images), int(is_u8), B, len(outs), ptr(ids_a), ptrs)
        for i, n in enumerate(head_names):
            if n in self.cm.vector_taps:
                outs[i] = self._class_vectors(outs[i], n)
        return outs

    def _class_vectors(self, buf, name):
        tap = self.cm.vector_taps[name]
        c0, Cl = tap["coff"], tap["C"]
        if tap["planes"] == 3:                    # precision 2: [lo | hi | hi] planes -> lo + hi
            feat = buf[..., c0:c0 + Cl] + buf[..., c0 + Cl:c0 + 2 * Cl]
        else:
            feat = buf[..., c0:c0 + Cl]
        head = next(h for h in self.spec["heads"] if h["name"] == name)
        return class_vectors_from_features(feat, head, self.dense_weights)


def head_spec(spec, name):
    """The entry of head ``name`` in a model spec."""
    return next(h for h in spec["heads"] if h["name"] == name)


def pack_dense_weights(head, weights):
    """The dense layers of "vector" head ``head`` in the layout the device's class-vector head reads (include/sleap_b200.h,
    sb_topdown_multiclass_params.dense_weights): float32, Keras layout, ``pre_classification{i}_fc`` kernel (n_in, units)
    then bias for each fc layer, then the head's own kernel and bias."""
    names = [f"pre_classification{i}_fc" for i in range(int(head.get("num_fc_layers", 1)))] + [head["name"]]
    return np.ascontiguousarray(np.concatenate([np.asarray(weights[n][k], np.float32).reshape(-1) for n in names
                                                for k in ("kernel", "bias")]))


def chain_key(params, *arrays):
    """Cache key of a chain's ctypes parameter struct: its bytes with the pointer fields zeroed, then the bytes of the
    ``arrays`` those fields point to -- a key of the values, whichever copy of them the pointers name.  It is computed
    on every predictor call, so a struct without pointer fields is not copied."""
    pointers = _pointer_fields(type(params))
    if pointers:
        params = type(params).from_buffer_copy(params)
        for name in pointers:
            setattr(params, name, None)
    key = bytes(params)
    for a in arrays:
        key += np.ascontiguousarray(a).tobytes()
    return key


@functools.lru_cache(maxsize=None)
def _pointer_fields(cls):
    return tuple(name for name, typ in cls._fields_ if typ is c_void_p)


def class_vectors_from_features(feat, head, weights):
    """``ClassVectorsHead.make_head`` (sleap/nn/heads.py:431-460) on a feature map ``feat`` (N, H, W, C) float32: global max
    pool (or Keras Flatten in H, W, C order), ``num_fc_layers`` x (Dense + ReLU), Dense + softmax -> (N, n_classes)."""
    x = np.asarray(feat, np.float32)
    x = x.max(axis=(1, 2)) if head.get("global_pool", True) else x.reshape(len(x), -1)
    for i in range(int(head.get("num_fc_layers", 1))):
        p = weights[f"pre_classification{i}_fc"]
        x = np.maximum(x @ np.asarray(p["kernel"], np.float32) + np.asarray(p["bias"], np.float32), np.float32(0))
    p = weights[head["name"]]
    z = x @ np.asarray(p["kernel"], np.float32) + np.asarray(p["bias"], np.float32)
    z = z - z.max(axis=1, keepdims=True)
    e = np.exp(z, dtype=np.float32)
    return (e / e.sum(axis=1, keepdims=True)).astype(np.float32)


class FrameResizer:
    """``sleap.nn.data.resizing.resize_image`` (resizing.py:71-106) for uint8 / float frame stacks on the device:
    a one-op model (PREPROCESS with ``input_scale``) runs the bilinear half-pixel resize kernel the networks use;
    integer frames are fed as float 0..255 and cast back by truncation, like ``tf.cast(tf.image.resize(...), dtype)``."""

    def __init__(self, handle=None):
        self.handle = handle or _lib.default_handle()
        self._models = {}

    def __call__(self, imgs: np.ndarray, scale: float) -> np.ndarray:
        from sleap_b200.nn import oplist as ol
        imgs = np.ascontiguousarray(imgs)
        B, H, W, C = imgs.shape
        key = (H, W, C, float(scale))
        if key not in self._models:
            ops = np.ascontiguousarray(np.stack([ol.buffer_record(0, 1, C, 1, 1), ol.preprocess_record(0, C, float(scale), 1)]).astype(np.int32))
            blob = np.zeros(1, np.float32)
            mid = c_int(-1)
            self.handle.call("sb_load_model", ptr(ops), ops.shape[0], ptr(blob), 1, int(PRECISION_FP32), ctypes.byref(mid))
            self._models[key] = [mid.value, 0]
        mid, cap = self._models[key]
        if cap < B:
            self.handle.call("sb_model_configure", mid, B, H, W, C)
            self._models[key][1] = B
        nh, nw = int(np.float32(H) * np.float32(scale)), int(np.float32(W) * np.float32(scale))
        out = np.zeros((B, nh, nw, C), np.float32)
        ids = np.asarray([0], np.int32)
        ptrs = (c_void_p * 1)(out.ctypes.data)
        src = np.ascontiguousarray(imgs, dtype=np.float32)                  # 0..255 stays 0..255 (no ensure_float scaling)
        self.handle.call("sb_model_forward", mid, ptr(src), 0, B, 1, ptr(ids), ptrs)
        if imgs.dtype == np.uint8:
            return np.clip(np.trunc(out), 0, 255).astype(np.uint8)
        return out.astype(imgs.dtype)


def load_weights_npz(path):
    """``{layer}/{param}`` arrays exported from a Keras ``best_model.h5`` (see INTEGRATION.md)."""
    z = np.load(path)
    w = {}
    for k in z.files:
        layer, param = k.rsplit("/", 1)
        w.setdefault(layer, {})[param] = z[k]
    return w


_KERAS_PARAM = {"moving_mean": "mean", "moving_variance": "var"}


def load_weights_h5(path):
    """Keras ``best_model.h5`` -> ``{layer: {param: array}}`` (sleap/nn/inference.py:3203-3213 loads the same
    file with ``tf.keras.models.load_model``).  Read with the in-tree HDF5 reader (no h5py needed).
    Output layers are named ``{HeadClass}_{i}`` by the reference (sleap/nn/model.py:351-360); the
    compiled graph uses the class name, so an index suffix ``_0`` is dropped."""
    from sleap_b200.io import h5lite
    raw = h5lite.read_keras_weights(path)
    w = {}
    for layer, params in raw.items():
        name = layer
        if "Head_" in layer and layer.rsplit("_", 1)[1].isdigit():
            base, idx = layer.rsplit("_", 1)
            name = base if idx == "0" else layer
        w[name] = {_KERAS_PARAM.get(k, k): np.asarray(v) for k, v in params.items()}
    return w


def load_weights(model_dir):
    """``best_model.npz`` (exported) if present, else the Keras ``best_model.h5``."""
    npz, h5 = os.path.join(model_dir, "best_model.npz"), os.path.join(model_dir, "best_model.h5")
    if os.path.exists(npz):
        return load_weights_npz(npz)
    if os.path.exists(h5):
        return load_weights_h5(h5)
    raise FileNotFoundError(f"neither best_model.npz nor best_model.h5 found in {model_dir}")


def save_weights_npz(path, weights):
    flat = {f"{layer}/{param}": arr for layer, p in weights.items() for param, arr in p.items()}
    np.savez(path, **flat)
