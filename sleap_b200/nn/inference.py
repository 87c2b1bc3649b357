"""Drop-in for the inference side of ``sleap.nn.inference`` (reference: sleap/nn/inference.py).

Kept surface (same names / attributes / dict contract, NumPy in and out):
  Predictor (:158-590), InferenceModel.predict / predict_on_batch (:989-1090),
  SingleInstanceInferenceLayer/Model/Predictor (:1229-1636),
  CentroidCrop (:1638-1967), FindInstancePeaks (:1969-2201), TopDownInferenceModel (:2246-2311),
  TopDownPredictor (:2314-2735), BottomUpInferenceLayer/Model (:2737-3053),
  BottomUpPredictor (:3055-3349), load_model (:4865).
All tensor work runs on the GPU through libsleapb200 (C-ABI); this file is orchestration only.
"""
import collections
import contextlib
import ctypes
import json
import os
import queue
import threading
from ctypes import c_int32, byref
from typing import Dict, List, Optional

import numpy as np

from sleap_b200 import _lib
from sleap_b200._lib import (BottomUpParams, CentroidParams, GlobalParams, MultiClassParams, TopdownMultiClassParams, TopdownParams,
                             f32, i32, ptr)
from sleap_b200.nn import architectures as arch
from sleap_b200.nn import paf_grouping, peak_finding
from sleap_b200.nn.model import (DeviceModel, PRECISION_FP16, PRECISION_FP32, chain_key, head_spec, load_weights, load_weights_npz,
                                 pack_dense_weights)

REFINE = peak_finding.REFINE


def _images_of(data):
    if isinstance(data, dict):
        return data["image"]
    return data


def _ragged_to_dense(rows: List[np.ndarray], inner_shape, dtype=np.float32):
    """RaggedTensor.to_tensor(default=NaN) to the bounding shape + row lengths (data/utils.py:118-146)."""
    n = max([len(r) for r in rows] + [0])
    out = np.full((len(rows), n) + tuple(inner_shape), np.nan, dtype)
    for i, r in enumerate(rows):
        if len(r):
            out[i, :len(r)] = r
    return out, np.asarray([len(r) for r in rows], np.int64)


class InferenceModel:
    """sleap/nn/inference.py:969-1171 (predict / predict_on_batch contract)."""

    def call(self, data):
        raise NotImplementedError

    def __call__(self, data):
        return self.call(data)

    def predict_on_batch(self, data, numpy: bool = True, **kwargs):
        """:1047-1090.  Ragged outputs come back NaN-padded with an ``n_valid`` key."""
        outs = self.call(data)
        if isinstance(data, dict):
            for k in ("video_ind", "frame_ind", "scale", "offset_x", "offset_y"):
                if k in data and k not in outs:
                    outs[k] = data[k]
        return outs

    def predict(self, data, numpy: bool = True, batch_size: int = 4, **kwargs):
        """:989-1045: iterate batches and concatenate (NaN-padding to the widest batch)."""
        return _merge_batches(list(self.predict_batches(data, batch_size)))

    def predict_batches(self, data, batch_size: int = 4):
        """Generator over per-batch result dicts (the Predictor batch loop, :377-420).  When the model's device step
        takes these frames (``_stream``), the loop is double-buffered: the upload of batch i+1 overlaps the compute of
        batch i.  Otherwise one predict_on_batch per batch."""
        imgs = _images_of(data)
        n = len(imgs)
        if n == 0:
            return
        stream = self._stream(InferenceLayer._prep(np.asarray(imgs[0:min(n, batch_size)])), batch_size)
        if stream is None:
            for i in range(0, n, batch_size):
                yield self.predict_on_batch(np.asarray(imgs[i:i + batch_size]))
            return
        batches = ((InferenceLayer._prep(np.asarray(imgs[i:i + batch_size])),) for i in range(0, n, batch_size))
        yield from _pipelined_batches(batches, *stream)

    def _stream(self, first, batch_size):
        """The streamed step for batches of up to ``batch_size`` frames like ``first`` (the first batch, prepped), set
        up for them: (device model, submit call, ``collect(slot, B)`` returning the batch dict), or None for the
        per-batch route."""
        return None

    def predict_examples(self, examples, batch_size: int, max_centroids: int):
        """Generator over (example, result dict) for batches of labels examples (dicts with the frames ``image`` and the
        ground-truth ``centroids`` and ``instances``, at most ``max_centroids`` of each per frame): the batch loop of a
        predictor fed labels.  A run of batches whose frames the model's ground-truth step takes (``_stream_ground_truth``)
        is double-buffered as predict_batches is; other batches take one predict_on_batch each."""
        it = iter(examples)
        ex = next(it, None)
        while ex is not None:
            first = InferenceLayer._prep(ex["image"])
            got = self._stream_ground_truth(first, batch_size, max_centroids, ex)
            if got is None:
                yield ex, self.predict_on_batch(ex)
                ex = next(it, None)
                continue
            stream, K = got
            order, rest = collections.deque(), []

            def run(ex=ex):                   # the examples up to the first with other frames, as submit arguments
                while ex is not None:
                    imgs = InferenceLayer._prep(ex["image"])
                    table = None
                    if imgs.shape[1:] == first.shape[1:] and imgs.dtype == first.dtype:
                        table = self._ground_truth_table(ex, K)
                    if table is None:
                        rest.append(ex)
                        return
                    order.append(ex)
                    yield (imgs,) + table
                    ex = next(it, None)

            for out in _pipelined_batches(run(), *stream):
                yield order.popleft(), out
            ex = rest[0] if rest else None

    def _stream_ground_truth(self, first, batch_size, max_centroids, ex=None):
        """The streamed ground-truth step for batches of up to ``batch_size`` labels examples like ``ex`` with frames like
        ``first`` (prepped) and up to ``max_centroids`` centroids (or labelled instances) per frame, set up for them:
        ((device model, submit call, ``collect(slot, B)``), the capacity of the tables it takes), or None for the
        per-batch route."""
        return None

    def _ground_truth_table(self, ex, K):
        """The arrays the ground-truth submit takes after the frames of labels example ``ex``, for tables of capacity K:
        the centroid table and counts; None when the streamed step cannot take the example."""
        return _centroid_table(ex["centroids"], K)


def _merge_batches(chunks):
    out = {}
    if not chunks:
        return out
    for k in chunks[0]:
        if k.startswith("gathered_"):             # per-step arrays of the multi-GPU exchange: kept as a list
            out[k] = [c[k] for c in chunks]
            continue
        arrs = [np.asarray(c[k]) for c in chunks]
        if arrs[0].ndim >= 2 and np.issubdtype(arrs[0].dtype, np.floating):
            n = max(a.shape[1] for a in arrs)
            padded = []
            for a in arrs:
                if a.shape[1] < n:
                    pad = np.full((a.shape[0], n - a.shape[1]) + a.shape[2:], np.nan, a.dtype)
                    a = np.concatenate([a, pad], axis=1)
                padded.append(a)
            out[k] = np.concatenate(padded, axis=0)
        else:
            out[k] = np.concatenate(arrs, axis=0)
    return out


class InferenceLayer:
    """sleap/nn/inference.py:897-967: owns the device model and the preprocessing parameters.
    (uint8 -> float, gray/rgb, resize by input_scale and pad_to_stride run inside the device op-list.)"""

    CHAIN = None        # configure call of the layer's post-processing chain; ``params()`` returns its parameters
    _keep = ()          # the arrays the pointer fields of those parameters point to

    def __init__(self, keras_model: DeviceModel, input_scale: float = 1.0, pad_to_stride: int = 1,
                 ensure_grayscale: Optional[bool] = None, ensure_float: bool = True):
        self.keras_model = keras_model      # attribute name kept from the reference
        self.input_scale = input_scale
        self.pad_to_stride = pad_to_stride
        if ensure_grayscale is None:
            ensure_grayscale = keras_model.cm.input_channels == 1
        self.ensure_grayscale = ensure_grayscale
        self.ensure_float = ensure_float

    @staticmethod
    def _prep(imgs):
        imgs = np.ascontiguousarray(imgs)
        if imgs.ndim == 3:
            imgs = imgs[..., None]
        if imgs.dtype != np.uint8:
            imgs = np.ascontiguousarray(imgs, dtype=np.float32)
        return imgs

    def _configure(self, B, H, W, C):
        """The device model for batches of up to B frames of (H, W, C), then the layer's chain (``CHAIN``)."""
        m = self.keras_model
        if not (m.configured_for and m.configured_for[0] >= B and m.configured_for[1:] == (H, W, C)):
            m.configure(B, H, W, C)
        m.configure_chain(self.CHAIN, self.params(), *self._keep)


def _track_fields(rec):
    """Per-frame track records ([B][2 + 3 I] doubles: n, flag, order[I], track id[I], tracking score[I]) as batch-dict
    fields: track_order / track_ids / tracking_scores (B, I) (order = index into the frame's instance list, -1 padded),
    track_n and track_flags (B)."""
    I = (rec.shape[1] - 2) // 3
    return {"track_n": rec[:, 0].astype(np.int64), "track_flags": rec[:, 1].astype(np.int64),
            "track_order": rec[:, 2:2 + I].astype(np.int64), "track_ids": rec[:, 2 + I:2 + 2 * I].astype(np.int64),
            "tracking_scores": rec[:, 2 + 2 * I:].copy()}


def _step_tracks(m, fn, tracker, slot, B):
    """The track fields of the B frames a step of model ``m`` returned, read with ``fn`` (sb_bottomup_tracks or
    sb_topdown_tracks) from slot 0 / 1 (slot 0 after the synchronous call); none without ``tracker``."""
    if tracker is None:
        return {}
    rec = np.zeros((B, 2 + 3 * tracker._device.max_instances), np.float64)
    m.handle.call(fn, m.model_id, slot, B, ptr(rec))
    return _track_fields(rec)


def _find_head(model: DeviceModel, name: str):
    if name not in model.cm.head_buffers:
        return None
    return model.cm.head_buffers[name]


def head_channels(model: DeviceModel, name: str) -> int:
    """Output channels of head ``name`` in the model's spec."""
    return next(h["channels"] for h in model.spec["heads"] if h["name"] == name)


# ------------------------------------------------------------------------------------------
class SingleInstanceInferenceLayer(InferenceLayer):
    """sleap/nn/inference.py:1229-1380."""

    HEAD = "SingleInstanceConfmapsHead"
    CHAIN = "sb_global_configure"

    def __init__(self, keras_model, input_scale=1.0, pad_to_stride=1, output_stride=None, peak_threshold=0.2,
                 refinement="local", integral_patch_size=5, return_confmaps=False, confmaps_ind=None,
                 offsets_ind=None, **kwargs):
        super().__init__(keras_model, input_scale=input_scale, pad_to_stride=pad_to_stride, **kwargs)
        self.confmaps_buffer = _find_head(keras_model, self.HEAD)
        if self.confmaps_buffer is None:
            raise ValueError(f"Index of the confidence maps output tensor must be specified if not named '{self.HEAD}'.")
        self.offsets_buffer = _find_head(keras_model, "OffsetRefinementHead")
        if output_stride is None:
            output_stride = keras_model.cm.head_strides[self.HEAD]
        self.output_stride = output_stride
        self.peak_threshold = peak_threshold
        self.refinement = refinement
        self.integral_patch_size = integral_patch_size
        self.return_confmaps = return_confmaps

    def params(self) -> GlobalParams:
        return GlobalParams(self.confmaps_buffer, -1 if self.offsets_buffer is None else self.offsets_buffer,
                            int(self.output_stride), float(self.peak_threshold), REFINE.get(self.refinement, 0),
                            int(self.integral_patch_size), float(self.input_scale))

    def call(self, data, crop_offsets=None):
        imgs = self._prep(_images_of(data))
        B, H, W, C = imgs.shape
        self._configure(B, H, W, C)
        co = None if crop_offsets is None else f32(crop_offsets).reshape(B, 2)
        out = self._run_step(B, "sb_infer_global", ptr(imgs), int(imgs.dtype == np.uint8), B, ptr(co))
        if self.return_confmaps:
            out["confmaps"] = self.keras_model.forward(imgs, [self.HEAD])[0]
        return out

    def _run_step(self, B, fn, *args):
        """One call ``fn(model id, *args, <outputs>)`` (sb_infer_global or sb_global_collect) into B frames' peaks, as a
        batch dict.  ``args`` run up to the outputs, B included: sb_infer_global takes the crop offsets after B."""
        m = self.keras_model
        n_nodes = head_channels(m, self.HEAD)
        pts = np.zeros((B, n_nodes, 2), np.float32)
        vals = np.zeros((B, n_nodes), np.float32)
        m.handle.call(fn, m.model_id, *args, ptr(pts), ptr(vals))
        return {"instance_peaks": pts[:, None], "instance_peak_vals": vals[:, None]}


class SingleInstanceInferenceModel(InferenceModel):
    """sleap/nn/inference.py:1383-1415."""

    def __init__(self, single_instance_layer: SingleInstanceInferenceLayer):
        self.single_instance_layer = single_instance_layer

    def call(self, example):
        return self.single_instance_layer.call(example)

    def _stream(self, first, batch_size):
        """sb_global_submit / sb_global_collect: uint8 frames without return_confmaps."""
        layer = self.single_instance_layer
        if first.dtype != np.uint8 or layer.return_confmaps:
            return None
        layer._configure(batch_size, *first.shape[1:])
        return layer.keras_model, "sb_global_submit", lambda slot, B: layer._run_step(B, "sb_global_collect", slot, B)


# ------------------------------------------------------------------------------------------
class CentroidCrop(InferenceLayer):
    """sleap/nn/inference.py:1638-1967: centroid net -> local peaks -> crops of the raw frames."""

    HEAD = "CentroidConfmapsHead"

    def __init__(self, keras_model, crop_size, input_scale=1.0, pad_to_stride=1, output_stride=None,
                 peak_threshold=0.2, refinement="local", integral_patch_size=5, return_confmaps=False,
                 return_crops=True, confmaps_ind=None, offsets_ind=None, max_instances=None,
                 precrop_resize=1.0, max_peaks_per_sample=256, **kwargs):
        super().__init__(keras_model, input_scale=input_scale, pad_to_stride=pad_to_stride, **kwargs)
        self.crop_size = crop_size
        self.confmaps_buffer = _find_head(keras_model, self.HEAD)
        if self.confmaps_buffer is None:
            raise ValueError(f"Index of the confidence maps output tensor must be specified if not named '{self.HEAD}'.")
        self.offsets_buffer = _find_head(keras_model, "OffsetRefinementHead")
        self.output_stride = output_stride or keras_model.cm.head_strides[self.HEAD]
        self.peak_threshold = peak_threshold
        self.refinement = refinement
        self.integral_patch_size = integral_patch_size
        self.return_confmaps = return_confmaps
        self.return_crops = return_crops
        self.max_instances = max_instances
        self.precrop_resize = precrop_resize
        self.max_peaks_per_sample = max_peaks_per_sample
        self._resizer = None

    def params(self) -> CentroidParams:
        return CentroidParams(self.confmaps_buffer, -1 if self.offsets_buffer is None else self.offsets_buffer,
                              int(self.output_stride), float(self.peak_threshold), REFINE.get(self.refinement, 0),
                              int(self.integral_patch_size), float(self.input_scale), int(self.max_peaks_per_sample))

    def call(self, inputs):
        full_imgs = self._prep(_images_of(inputs))
        B, H, W, C = full_imgs.shape
        m = self.keras_model
        m.configure(B, H, W, C).configure_chain("sb_centroid_configure", self.params())
        cap = B * self.max_peaks_per_sample
        pts = np.zeros((cap, 2), np.float32)
        vals = np.zeros((cap,), np.float32)
        sinds = np.zeros((cap,), np.int32)
        n = c_int32(0)
        flags = np.zeros((B,), np.int32)
        m.handle.call("sb_infer_centroids", m.model_id, ptr(full_imgs), int(full_imgs.dtype == np.uint8), B, ptr(pts),
                      ptr(vals), ptr(sinds), byref(n), ptr(flags))
        k = n.value
        pts, vals, sinds = pts[:k].copy(), vals[:k].copy(), sinds[:k].copy()
        if self.precrop_resize != 1.0:                       # :1836-1841 (the returned centroids stay in the resized frame, as in the reference)
            if self._resizer is None:
                from sleap_b200.nn.model import FrameResizer
                self._resizer = FrameResizer(m.handle)
            full_imgs = self._resizer(full_imgs, self.precrop_resize)
            H, W = full_imgs.shape[1:3]
            pts = (pts * np.float32(self.precrop_resize)).astype(np.float32)
        if k > 0 and self.max_instances is not None:
            keep = []
            for s in range(B):   # tf.math.top_k: descending score, ties keep the lower index (:1879-1894)
                idx = np.nonzero(sinds == s)[0]
                if self.max_instances < len(idx):
                    order = np.argsort(-vals[idx], kind="stable")[: self.max_instances]
                    idx = idx[order]
                keep.append(idx)
            keep = np.concatenate(keep) if keep else np.zeros((0,), np.int64)
            pts, vals, sinds = pts[keep], vals[keep], sinds[keep]
            k = len(keep)
        crop_offsets = (pts - np.float32(self.crop_size / 2)).astype(np.float32)
        out = dict(centroids=[pts[sinds == s] for s in range(B)], centroid_vals=[vals[sinds == s] for s in range(B)],
                   flags=flags)
        if self.return_crops:
            if k > 0:
                crops = np.zeros((k, self.crop_size, self.crop_size, C), full_imgs.dtype)
                m.handle.call("sb_crop_centered", ptr(full_imgs), int(full_imgs.dtype == np.uint8), B, H, W, C,
                              ptr(f32(pts)), ptr(i32(sinds)), k, self.crop_size, self.crop_size, ptr(crops))
            else:
                crops = np.zeros((0, self.crop_size, self.crop_size, C), full_imgs.dtype)
            out["crops"] = crops
            out["crop_offsets"] = crop_offsets
            out["crop_sample_inds"] = sinds
            out["samples"] = B
        return out


class FindInstancePeaks(SingleInstanceInferenceLayer):
    """sleap/nn/inference.py:1969-2201: centered-instance net on crops -> global peaks (+ crop offsets)."""

    HEAD = "CenteredInstanceConfmapsHead"

    def __init__(self, keras_model, max_crops_per_call=64, **kwargs):
        super().__init__(keras_model, **kwargs)
        self.max_crops_per_call = max_crops_per_call

    def call(self, inputs):
        if isinstance(inputs, dict):
            crops = inputs["crops"]
        else:
            crops, inputs = inputs, {}
        crops = self._prep(crops)
        n = crops.shape[0]
        if "crop_sample_inds" in inputs:
            samples, sinds = inputs["samples"], np.asarray(inputs["crop_sample_inds"])
        else:
            samples, sinds = n, np.arange(n)
        co = inputs.get("crop_offsets")
        m = self.keras_model
        n_nodes = head_channels(m, self.HEAD)
        pts = np.zeros((n, n_nodes, 2), np.float32)
        vals = np.zeros((n, n_nodes), np.float32)
        for i in range(0, n, self.max_crops_per_call):
            sl = slice(i, min(n, i + self.max_crops_per_call))
            sub = np.ascontiguousarray(crops[sl])
            # keep one device configuration for all chunk sizes
            self._configure(self.max_crops_per_call, *sub.shape[1:])
            o = super().call(sub, crop_offsets=None if co is None else np.asarray(co)[sl])
            pts[sl], vals[sl] = o["instance_peaks"][:, 0], o["instance_peak_vals"][:, 0]
        out = {"instance_peaks": [pts[sinds == s] for s in range(samples)],
               "instance_peak_vals": [vals[sinds == s] for s in range(samples)]}
        for k in ("centroids", "centroid_vals"):
            if k in inputs:
                out[k] = inputs[k]
        return out


class CentroidCropGroundTruth:
    """sleap/nn/inference.py:723-809: stands in for a centroid model -- crops of ``crop_size`` around the
    ground-truth centroids of a labels example (``example_gt["centroids"]``: one (n, 2) array per sample, made by
    ``LabelsReader(with_centroids=True)`` = InstanceCentroidFinder).  The crop itself is the device kernel."""

    def __init__(self, crop_size: int, input_scale: float = 1.0, handle=None):
        self.crop_size = crop_size
        self.input_scale = input_scale
        self.handle = handle
        self._resizer = None

    def call(self, example_gt):
        from sleap_b200 import _lib
        full_imgs = np.ascontiguousarray(example_gt["image"])
        cents = [f32(c).reshape(-1, 2) for c in example_gt["centroids"]]
        if self.input_scale != 1.0:                          # :768-770: resized frames, centroids scaled with them
            if self._resizer is None:
                from sleap_b200.nn.model import FrameResizer
                self._resizer = FrameResizer(self.handle or _lib.default_handle())
            full_imgs = self._resizer(full_imgs, self.input_scale)
            cents = [(c * np.float32(self.input_scale)).astype(np.float32) for c in cents]
        B, H, W, C = full_imgs.shape
        sinds = np.concatenate([np.full(len(c), s, np.int32) for s, c in enumerate(cents)]) if cents else np.zeros(0, np.int32)
        pts = np.concatenate(cents) if cents else np.zeros((0, 2), np.float32)
        k = len(pts)
        crop_offsets = (pts - np.float32(self.crop_size / 2)).astype(np.float32)          # :777
        crops = np.zeros((k, self.crop_size, self.crop_size, C), full_imgs.dtype)
        if k > 0:
            h = self.handle or _lib.default_handle()
            h.call("sb_crop_centered", ptr(full_imgs), int(full_imgs.dtype == np.uint8), B, H, W, C, ptr(f32(pts)), ptr(i32(sinds)), k,
                   self.crop_size, self.crop_size, ptr(crops))
        return dict(crops=crops, crop_offsets=crop_offsets, crop_sample_inds=sinds, samples=B, centroids=cents,
                    centroid_vals=[np.ones(len(c), np.float32) for c in cents])


class FindInstancePeaksGroundTruth:
    """sleap/nn/inference.py:812-893: stands in for a centered-instance model -- every centroid gets the
    ground-truth instance whose nearest node is closest to it (``example_gt["instances"]``: one (n, nodes, 2)
    array per sample); peak values are 1."""

    def call(self, example_gt, crop_output):
        peaks, vals = [], []
        for inst, cent in zip(example_gt["instances"], crop_output["centroids"]):
            inst, cent = f32(inst), f32(cent).reshape(-1, 2)
            n_nodes = inst.shape[1] if inst.ndim == 3 else 0
            rows = []
            if len(inst) and len(cent):
                import warnings
                with np.errstate(invalid="ignore"), warnings.catch_warnings():
                    warnings.simplefilter("ignore", RuntimeWarning)
                    d = np.sqrt(((inst[None] - cent[:, None, None, :]) ** 2).sum(-1))      # (n_centroids, n_insts, n_nodes)
                    # reduce_min over nodes (:860): Eigen's scalar min keeps the accumulator when the new value is NaN,
                    # so invisible nodes are skipped and only an all-NaN instance yields NaN
                    # (tests/nn/test_inference.py:168-209 "GT instances have NaNs")
                    d = np.nanmin(d, axis=-1)
                for c in range(len(cent)):
                    if np.all(np.isnan(d[c])):
                        continue                                                           # :866-868 all-NaN rows are dropped
                    best = 0                                                               # tf.argmin: first index; NaN never wins a "<"
                    for j in range(1, d.shape[1]):
                        if d[c, j] < d[c, best]:
                            best = j
                    rows.append(inst[best])
            peaks.append(np.stack(rows) if rows else np.zeros((0, n_nodes, 2), np.float32))
            vals.append(np.ones(peaks[-1].shape[:2], np.float32))
        return dict(centroids=crop_output["centroids"], centroid_vals=crop_output["centroid_vals"], instance_peaks=peaks,
                    instance_peak_vals=vals)


class CentroidInferenceModel(InferenceModel):
    """sleap/nn/inference.py:2203-2244: the first stage of the top-down path on its own (centroids only)."""

    def __init__(self, centroid_crop):
        self.centroid_crop = centroid_crop

    def call(self, example):
        if isinstance(example, np.ndarray):
            example = dict(image=example)
        out = self.centroid_crop.call(example)
        ce, nv = _ragged_to_dense(out["centroids"], (2,))
        cv, _ = _ragged_to_dense(out["centroid_vals"], ())
        res = {"centroids": ce, "centroid_vals": cv, "n_valid": nv}
        for k in ("crops", "crop_offsets", "crop_sample_inds", "flags"):
            if k in out:
                res[k] = out[k]
        return res


def _topdown_params(cc, fp):
    """TopdownParams of the fused pipeline over centroid layer ``cc`` and instance layer ``fp``, and its K (centroids kept
    per frame)."""
    K = int(cc.max_instances) if cc.max_instances else int(cc.max_peaks_per_sample)
    return TopdownParams(cc.keras_model.model_id, fp.keras_model.model_id, cc.params(), fp.params(), int(cc.crop_size),
                         int(cc.max_instances or 0), K, int(fp.max_crops_per_call), float(cc.precrop_resize)), K


def _centroid_table(centroids, K):
    """The ragged ground-truth centroids of a batch (one (n, 2) array per frame) as sb_topdown_gt_submit takes them: the
    (B, K, 2) float32 table, NaN past each frame's count, and the (B,) int32 counts.  A frame with more than K centroids
    keeps its count, so the submit refuses the batch rather than dropping centroids."""
    cents = [f32(c).reshape(-1, 2) for c in centroids]
    counts = np.asarray([len(c) for c in cents], np.int32)
    table = np.full((len(cents), K, 2), np.nan, np.float32)
    for b, c in enumerate(cents):
        table[b, :len(c)] = c[:K]
    return table, counts


def _ground_truth_params(cc, fp, K):
    """TopdownParams of the ground-truth pipeline of layer ``cc`` on instance layer ``fp`` with K centroids per frame."""
    return TopdownParams(-1, fp.keras_model.model_id, CentroidParams(), fp.params(), int(cc.crop_size), 0, int(K),
                         int(fp.max_crops_per_call), float(cc.input_scale))


def _instance_nodes(instances):
    """The node count of a batch's ground-truth instances (one (n, nodes, 2) array per frame) as the host route's batch
    dict has it (the most nodes of any frame's array), or None when the fused step cannot take them: no nodes, or a
    frame with instances of another shape."""
    arrs = [np.asarray(a) for a in instances]
    nodes = max([a.shape[1] for a in arrs if a.ndim == 3] + [0])
    if nodes == 0 or any(len(a) and (a.ndim != 3 or a.shape[1:] != (nodes, 2)) for a in arrs):
        return None
    return nodes


def _instance_table(instances, N, nodes):
    """The ground-truth instances of a batch (one (n, nodes, 2) array per frame) as sb_topdown_gt_instances_submit takes
    them: the (B, N, nodes, 2) float32 table, NaN past each frame's count, and the (B,) int32 counts.  A frame with more
    than N instances keeps its count, so the submit refuses the batch rather than dropping instances."""
    arrs = [f32(a) for a in instances]
    counts = np.asarray([len(a) for a in arrs], np.int32)
    table = np.full((len(arrs), N, nodes, 2), np.nan, np.float32)
    for b, a in enumerate(arrs):
        if len(a):
            table[b, :len(a)] = a[:N]
    return table, counts


def _gt_instances_params(cc):
    """TopdownParams of the ground-truth instances pipeline of centroid layer ``cc`` (no instance model), and its K."""
    K = int(cc.max_instances) if cc.max_instances else int(cc.max_peaks_per_sample)
    return TopdownParams(cc.keras_model.model_id, -1, cc.params(), GlobalParams(), int(cc.crop_size), int(cc.max_instances or 0), K, 1,
                         float(cc.precrop_resize)), K


# The last configure of a top-down pipeline (TopDownInferenceModel._configure_pipeline): its call at capacities 0 (the
# call's name, the chain key of its parameters, the arguments after them), its capacities (B, then K or N), the chain
# record it set and the device models it set it on.
_Configured = collections.namedtuple("_Configured", "key caps chain models")


class TopDownInferenceModel(InferenceModel):
    """sleap/nn/inference.py:2246-2311.  The fused pipeline takes one of three centroid sources: a centroid model, the
    ground-truth centroids of labels (CentroidCropGroundTruth), or a centroid model matched against ground-truth instances
    (FindInstancePeaksGroundTruth).  TopDownMultiClassInferenceModel shares the configure, the streams and the dispatch,
    and supplies its own parameters (``_params``), calls and result builder (``_run_fused``)."""

    CONFIGURE, INFER, SUBMIT, COLLECT = "sb_topdown_configure", "sb_infer_topdown", "sb_topdown_submit", "sb_topdown_collect"
    _keep = ()          # the arrays the pointer fields of ``_params`` point to

    def __init__(self, centroid_crop, instance_peaks):
        self.centroid_crop = centroid_crop
        self.instance_peaks = instance_peaks
        self.fused = True            # one device pipeline (sb_infer_topdown) when both stages are device models
        # a Tracker with track_device, run by k_track inside each fused step (TopDownPredictor.predict sets it for its span)
        self.tracker = None
        self._pipeline = None        # the _Configured of the last pipeline configure

    def detach_tracker(self):
        mc = self.centroid_crop.keras_model
        if getattr(self.tracker, "_device", None) is not None and mc.chain and mc.chain[0] == "sb_topdown_configure":
            mc.handle.call("sb_topdown_attach_tracker", mc.model_id, -1, 1.0, 1.0)

    def _can_fuse(self):
        cc, fp = self.centroid_crop, self.instance_peaks
        if not (self.fused and type(fp) is FindInstancePeaks and not fp.return_confmaps and fp.keras_model.input_scale == 1.0):
            return False
        if type(cc) is CentroidCropGroundTruth:
            return cc.handle is fp.keras_model.handle
        return (type(cc) is CentroidCrop and cc.return_crops and not cc.return_confmaps
                and cc.keras_model.handle is fp.keras_model.handle)

    @property
    def ground_truth(self):
        """Centroids come from the labels (CentroidCropGroundTruth), not from a centroid model."""
        return isinstance(self.centroid_crop, CentroidCropGroundTruth)

    def _fuses_instances(self):
        """A centroid model with ground-truth instances (FindInstancePeaksGroundTruth) runs as one device step
        (sb_topdown_gt_instances_submit) on uint8 labels examples."""
        cc = self.centroid_crop
        return (self.fused and type(self.instance_peaks) is FindInstancePeaksGroundTruth and type(cc) is CentroidCrop
                and not cc.return_confmaps and (cc.max_instances is None or cc.max_instances > 0))

    def _params(self, td):
        """The parameters of ``CONFIGURE`` over TopdownParams ``td``."""
        return td

    def _configure_pipeline(self, fn, args, caps, plans, arrays=()):
        """Configures a form of the pipeline with ``fn(byref(p), *rest)``, where (p, *rest) = ``args(*caps)``.  When the
        last configure made the same call at capacities 0 and every model it configured still runs the chain it set, the
        capacities ``caps`` (B, then K or N) grow to the larger of asked and held, and nothing is called while the held ones
        suffice; otherwise the call is made at the asked ones.  ``plans(*caps)``: (device model, its configured_for) of each
        model the pipeline uses, the one that holds it first; ``arrays``: the ones the pointer fields of p point to.
        Returns the pipeline's capacities."""
        p0, *rest0 = args(*(0,) * len(caps))
        key = (fn, chain_key(p0, *arrays), tuple(rest0))
        have = self._pipeline
        if have is not None and have.key == key and all(m.chain is have.chain for m in have.models):
            if all(c <= h for c, h in zip(caps, have.caps)):
                return have.caps
            caps = tuple(max(c, h) for c, h in zip(caps, have.caps))
        p, *rest = args(*caps)
        plan = plans(*caps)
        for m, _ in plan:
            m.chain = None                       # a refused call may have dropped the previous chain
        plan[0][0].handle.call(fn, byref(p), *rest)
        chain = (fn, chain_key(p, *arrays))
        for m, configured_for in plan:
            m.configured_for, m.chain = configured_for, chain
        self._pipeline = _Configured(key, tuple(caps), chain, [m for m, _ in plan])
        return self._pipeline.caps

    def _configure_fused(self, B, H, W, C):
        """The pipeline with a centroid model for batches of up to B frames of (H, W, C), with ``self.tracker`` attached
        (the raw frame size, as the predictor's image_hw; default capacity, not K).  Returns K."""
        cc, fp = self.centroid_crop, self.instance_peaks
        mc = cc.keras_model
        td, K = _topdown_params(cc, fp)
        p = self._params(td)
        self._configure_pipeline(self.CONFIGURE, lambda b: (p, b, H, W, C), (B,),
                                 lambda b: [(mc, (b, H, W, C)), (fp.keras_model, (fp.max_crops_per_call, cc.crop_size, cc.crop_size, C))],
                                 self._keep)
        if self.tracker is not None:
            dev = self.tracker._device_tracker(head_channels(fp.keras_model, fp.HEAD), handle=mc.handle)
            mc.handle.call("sb_topdown_attach_tracker", mc.model_id, dev.id, float(H), float(W))
        return K

    def _configure_ground_truth(self, B, K, shape):
        """The ground-truth centroids pipeline of the instance model (sb_topdown_gt_submit) for batches of up to B frames
        of ``shape`` (H, W, C) with up to K centroids each: B and K grow only when a batch exceeds them, and K is at least
        1.  Returns the pipeline's K."""
        cc, fp = self.centroid_crop, self.instance_peaks
        shape = tuple(shape)
        _, K = self._configure_pipeline(
            self.CONFIGURE, lambda b, k: (self._params(_ground_truth_params(cc, fp, k)), b) + shape, (B, max(K, 1)),
            # the instance network's plan: chunks of max_crops_per_call crops, but no more than a batch's B x K
            # (include/sleap_b200.h)
            lambda b, k: [(fp.keras_model, (min(fp.max_crops_per_call, b * k), cc.crop_size, cc.crop_size, shape[2]))],
            self._keep)
        return K

    def _configure_gt_instances(self, B, N, nodes, shape):
        """The ground-truth instances pipeline of the centroid model (sb_topdown_gt_instances_submit) for batches of up
        to B frames of ``shape`` (H, W, C) with tables of up to N instances of ``nodes`` nodes: B and N grow only when a
        batch exceeds them, and N is at least 1.  Returns (K, N) of the pipeline."""
        cc = self.centroid_crop
        shape = tuple(shape)
        p, K = _gt_instances_params(cc)
        _, N = self._configure_pipeline("sb_topdown_gt_instances_configure", lambda b, n: (p, int(nodes), n, b) + shape,
                                        (B, max(N, 1)), lambda b, n: [(cc.keras_model, (b,) + shape)])
        return K, N

    def _run_gt_instances(self, B, K, nodes, slot):
        """sb_topdown_gt_instances_collect of ``slot`` into the batch dict of the host route: the centroids padded to the
        batch's most centroids, the matched instances to its most rows (``n_valid``)."""
        mc = self.centroid_crop.keras_model
        ce = np.zeros((B, K, 2), np.float32); cv = np.zeros((B, K), np.float32)
        ip = np.zeros((B, K, nodes, 2), np.float32); iv = np.zeros((B, K, nodes), np.float32)
        nc = np.zeros((B,), np.int32); nr = np.zeros((B,), np.int32); fl = np.zeros((B,), np.int32)
        mc.handle.call("sb_topdown_gt_instances_collect", mc.model_id, slot, B, ptr(ce), ptr(cv), ptr(nc), ptr(ip), ptr(iv), ptr(nr),
                       ptr(fl))
        c, r = int(nc.max()), int(nr.max())
        return {"centroids": ce[:, :c].copy(), "centroid_vals": cv[:, :c].copy(), "instance_peaks": ip[:, :r].copy(),
                "instance_peak_vals": iv[:, :r].copy(), "n_valid": nr.astype(np.int64), "flags": fl}

    def _owner(self):
        """The device model that holds the fused pipeline: the centroid model, or with ground-truth centroids the
        instance model."""
        return self.instance_peaks.keras_model if self.ground_truth else self.centroid_crop.keras_model

    def _run_fused(self, B, K, fn, *args, slot=0):
        """One fused call ``fn(model id, *args, B, <outputs>)`` (sb_infer_topdown or sb_topdown_collect) into dense arrays
        of B frames, as a batch dict; with a tracker, the track records of ``slot`` (0 after sb_infer_topdown)."""
        mc, n_nodes = self._owner(), head_channels(self.instance_peaks.keras_model, self.instance_peaks.HEAD)
        ce = np.zeros((B, K, 2), np.float32); cv = np.zeros((B, K), np.float32)
        ip = np.zeros((B, K, n_nodes, 2), np.float32); iv = np.zeros((B, K, n_nodes), np.float32)
        nv = np.zeros((B,), np.int32); fl = np.zeros((B,), np.int32)
        mc.handle.call(fn, mc.model_id, *args, B, ptr(ce), ptr(cv), ptr(ip), ptr(iv), ptr(nv), ptr(fl))
        n = int(nv.max()) if B else 0
        out = {"centroids": ce[:, :n].copy(), "centroid_vals": cv[:, :n].copy(), "instance_peaks": ip[:, :n].copy(),
               "instance_peak_vals": iv[:, :n].copy(), "n_valid": nv.astype(np.int64), "flags": fl}
        out.update(_step_tracks(mc, "sb_topdown_tracks", self.tracker, slot, B))
        return out

    def _call_fused(self, imgs):
        """``INFER``: frames up once, the whole step on the device, one dense record per frame back (include/sleap_b200.h)."""
        imgs = self.centroid_crop._prep(imgs)
        B, H, W, C = imgs.shape
        K = self._configure_fused(B, H, W, C)
        return self._run_fused(B, K, self.INFER, ptr(imgs), int(imgs.dtype == np.uint8))

    def _stream(self, first, batch_size):
        """``SUBMIT`` / ``COLLECT`` (the upload of batch i+1 and its centroid stage are queued before batch i is
        collected): uint8 frames and a model that can run the fused step with a centroid model."""
        if not self._can_fuse() or self.ground_truth or first.dtype != np.uint8:
            return None
        K = self._configure_fused(batch_size, *first.shape[1:])
        return (self.centroid_crop.keras_model, self.SUBMIT, lambda slot, B: self._run_fused(B, K, self.COLLECT, slot, slot=slot))

    def _stream_ground_truth(self, first, batch_size, max_centroids, ex=None):
        """sb_topdown_gt_submit / ``COLLECT``: uint8 frames and a model that can run the fused step with ground-truth
        centroids; or sb_topdown_gt_instances_submit / _collect: uint8 frames and ground-truth instances (``ex``) for a
        centroid model, tables of ``max_centroids`` instances.  The whole step is queued at the submit."""
        if first.dtype != np.uint8:
            return None
        if self._fuses_instances():
            nodes = _instance_nodes(ex["instances"]) if ex is not None and "instances" in ex else None
            if nodes is None:
                return None
            K, N = self._configure_gt_instances(batch_size, max_centroids, nodes, first.shape[1:])
            return (self.centroid_crop.keras_model, "sb_topdown_gt_instances_submit",
                    lambda slot, B: self._run_gt_instances(B, K, nodes, slot)), N
        if not (self._can_fuse() and self.ground_truth):
            return None
        K = self._configure_ground_truth(batch_size, max_centroids, first.shape[1:])
        return (self.instance_peaks.keras_model, "sb_topdown_gt_submit", lambda slot, B: self._run_ground_truth(B, K, slot)), K

    def _ground_truth_table(self, ex, K):
        if not self._fuses_instances():
            return super()._ground_truth_table(ex, K)
        nodes = self._pipeline.key[2][0]         # the node count: the first argument after the parameters
        return _instance_table(ex["instances"], K, nodes) if _instance_nodes(ex["instances"]) == nodes else None

    def _run_ground_truth(self, B, K, slot):
        return self._run_fused(B, K, self.COLLECT, slot, slot=slot)

    def call(self, example):
        if isinstance(example, np.ndarray):
            example = dict(image=example)
        if self._can_fuse() and not self.ground_truth:
            return self._call_fused(_images_of(example))
        rows = "instances" if self._fuses_instances() else "centroids"
        if rows in example and np.asarray(example["image"]).dtype == np.uint8:
            # one batch through the ground-truth step: its submit into slot 0, then the collect
            imgs = InferenceLayer._prep(example["image"])
            B = imgs.shape[0]
            got = self._stream_ground_truth(imgs, B, max([len(a) for a in example[rows]] + [0]), example)
            if got is not None:
                (m, fn, collect), cap = got
                m.handle.call(fn, m.model_id, ptr(imgs), *map(ptr, self._ground_truth_table(example, cap)), B, 0)
                return collect(0, B)
        return self._call_staged(example)

    def _call_staged(self, example):
        crop_out = self.centroid_crop.call(example)
        if isinstance(self.instance_peaks, FindInstancePeaksGroundTruth):                 # :2300-2304
            peaks_out = self.instance_peaks.call(example, crop_out)
        else:
            peaks_out = self.instance_peaks.call(crop_out)
        if isinstance(self.instance_peaks, FindInstancePeaksGroundTruth):
            n_nodes = max([p.shape[1] for p in peaks_out["instance_peaks"] if p.ndim == 3] + [0])
        else:
            n_nodes = head_channels(self.instance_peaks.keras_model, self.instance_peaks.HEAD)
        ip, nv = _ragged_to_dense(peaks_out["instance_peaks"], (n_nodes, 2))
        iv, _ = _ragged_to_dense(peaks_out["instance_peak_vals"], (n_nodes,))
        ce, _ = _ragged_to_dense(peaks_out["centroids"], (2,))
        cv, _ = _ragged_to_dense(peaks_out["centroid_vals"], ())
        out = {"centroids": ce, "centroid_vals": cv, "instance_peaks": ip, "instance_peak_vals": iv, "n_valid": nv}
        if "flags" in crop_out:
            out["flags"] = crop_out["flags"]
        return out


# ------------------------------------------------------------------------------------------
class BottomUpInferenceLayer(InferenceLayer):
    """sleap/nn/inference.py:2737-3003: net -> local peaks -> PAF scoring -> matching -> grouping,
    executed as one device pipeline (``sb_infer_bottomup``)."""

    CHAIN = "sb_bottomup_configure"

    def __init__(self, keras_model, paf_scorer, input_scale=1.0, pad_to_stride=1, cm_output_stride=None,
                 paf_output_stride=None, peak_threshold=0.2, refinement="local", integral_patch_size=5,
                 return_confmaps=False, return_pafs=False, return_paf_graph=False, confmaps_ind=None,
                 pafs_ind=None, offsets_ind=None, max_peaks_per_sample=1024, max_node_peaks=32,
                 max_instances=64, **kwargs):
        super().__init__(keras_model, input_scale=input_scale, pad_to_stride=pad_to_stride, **kwargs)
        self.paf_scorer = paf_scorer
        self.confmaps_buffer = _find_head(keras_model, "MultiInstanceConfmapsHead")
        self.pafs_buffer = _find_head(keras_model, "PartAffinityFieldsHead")
        self.offsets_buffer = _find_head(keras_model, "OffsetRefinementHead")
        if self.confmaps_buffer is None:
            raise ValueError("Index of the confidence maps output tensor must be specified if not named 'MultiInstanceConfmapsHead'.")
        if self.pafs_buffer is None:
            raise ValueError("Index of the part affinity fields output tensor must be specified if not named 'PartAffinityFieldsHead'.")
        self.cm_output_stride = cm_output_stride or keras_model.cm.head_strides["MultiInstanceConfmapsHead"]
        self.paf_output_stride = paf_output_stride or keras_model.cm.head_strides["PartAffinityFieldsHead"]
        self.peak_threshold = peak_threshold
        self.refinement = refinement
        self.integral_patch_size = integral_patch_size
        self.return_confmaps = return_confmaps
        self.return_pafs = return_pafs
        self.return_paf_graph = return_paf_graph
        self.max_peaks_per_sample = max_peaks_per_sample
        self.max_node_peaks = max_node_peaks
        self.max_instances = max_instances
        # a Tracker with track_device, run by k_track inside each step (BottomUpPredictor.predict sets it for its span),
        # and the predictor's max_instances cut of the instance list (-1: none)
        self.tracker = None
        self.tracker_cut = -1

    def attach_tracker(self, image_hw):
        """Attach ``self.tracker`` to the configured model for the frames of size ``image_hw`` (sb_bottomup_attach_tracker)."""
        if self.tracker is None:
            return
        m = self.keras_model
        dev = self.tracker._device_tracker(self.paf_scorer.n_nodes, handle=m.handle, max_instances=self.max_instances)
        m.handle.call("sb_bottomup_attach_tracker", m.model_id, dev.id, int(self.tracker_cut), float(image_hw[0]),
                      float(image_hw[1]))

    def detach_tracker(self):
        m = self.keras_model
        if getattr(self.tracker, "_device", None) is not None and m.chain and m.chain[0] == "sb_bottomup_configure":
            m.handle.call("sb_bottomup_attach_tracker", m.model_id, -1, -1, 1.0, 1.0)

    def track_fields(self, slot, B):
        """The track records of the batch just collected (slot 0 / 1; 0 after sb_infer_bottomup) as batch-dict fields."""
        return _step_tracks(self.keras_model, "sb_bottomup_tracks", self.tracker, slot, B)

    def params(self) -> BottomUpParams:
        """The chain's parameters; their edge arrays stay alive in ``self._keep``."""
        p, self._keep = paf_params(
            self.paf_scorer, (self.confmaps_buffer, self.pafs_buffer, -1 if self.offsets_buffer is None else self.offsets_buffer),
            self.cm_output_stride, self.paf_output_stride, self.peak_threshold, self.refinement, self.integral_patch_size,
            self.input_scale, self.max_peaks_per_sample, self.max_node_peaks, self.max_instances)
        return p

    def call(self, data):
        imgs = self._prep(_images_of(data))
        if imgs.dtype != np.uint8:
            raise ValueError("BottomUpInferenceLayer expects uint8 frames (the fused path reads raw frames).")
        B, H, W, C = imgs.shape
        self._configure(B, H, W, C)
        self.attach_tracker((H, W))
        m = self.keras_model
        out = self._run_step(B, "sb_infer_bottomup", ptr(imgs))
        if self.return_confmaps or self.return_pafs:
            cms, pafs = m.forward(imgs, ["MultiInstanceConfmapsHead", "PartAffinityFieldsHead"])
            if self.return_confmaps:
                out["confmaps"] = cms
            if self.return_pafs:
                out["part_affinity_fields"] = pafs
        if self.return_paf_graph:
            out.update(self.fetch_graph(B))
        return out

    def _run_step(self, B, fn, *args, slot=0):
        """One call ``fn(model id, *args, B, <outputs>)`` (sb_infer_bottomup or sb_bottomup_collect) into B frames'
        instances, as a batch dict; the track records and, with the multi-GPU exchange, every rank's records of this step
        (they came over with the result copy) from ``slot`` (0 after sb_infer_bottomup)."""
        m = self.keras_model
        I, N = self.max_instances, self.paf_scorer.n_nodes
        ip = np.zeros((B, I, N, 2), np.float32); iv = np.zeros((B, I, N), np.float32)
        isc = np.zeros((B, I), np.float32); nv = np.zeros((B,), np.int32); fl = np.zeros((B,), np.int32)
        m.handle.call(fn, m.model_id, *args, B, ptr(ip), ptr(iv), ptr(isc), ptr(nv), ptr(fl))
        n = int(nv.max()) if B else 0
        out = {"instance_peaks": ip[:, :n], "instance_peak_vals": iv[:, :n], "instance_scores": isc[:, :n],
               "n_valid": nv.astype(np.int64), "flags": fl}
        out.update(self.track_fields(slot, B))
        pg = getattr(m, "peer_gather", None)
        if pg is not None:
            out["gathered_records"], out["gathered_counts"] = pg.gathered(slot, B, I, N)
        return out

    def fetch_graph(self, B):
        m = self.keras_model
        pks, cands = _paf_graph_arrays(B, self.max_peaks_per_sample, self.paf_scorer.n_edges, self.max_node_peaks)
        m.handle.call("sb_bottomup_fetch_graph", m.model_id, B, len(pks[0]), *map(ptr, pks), len(cands[0]), *map(ptr, cands))
        return _paf_graph_rows(pks, cands)


def _paf_graph_arrays(B, max_peaks_per_sample, n_edges, max_node_peaks):
    """Host arrays of B frames' PAF graph: (peaks, values, channels, offsets), (edges, edge peaks, line scores, offsets)."""
    cp, cc = B * max_peaks_per_sample, B * n_edges * max_node_peaks ** 2
    return ((np.zeros((cp, 2), np.float32), np.zeros((cp,), np.float32), np.zeros((cp,), np.int32), np.zeros((B + 1,), np.int32)),
            (np.zeros((cc,), np.int32), np.zeros((cc, 2), np.int32), np.zeros((cc,), np.float32), np.zeros((B + 1,), np.int32)))


def _paf_graph_rows(pks, cands):
    """The PAF-graph arrays split into one row per frame at their offsets."""
    (peaks, pv, pc, po), (ei, epi, ls, co) = pks, cands
    rows = lambda a, o: [a[o[b]:o[b + 1]].copy() for b in range(len(o) - 1)]
    return {"peaks": rows(peaks, po), "peak_vals": rows(pv, po), "peak_channel_inds": rows(pc, po),
            "edge_inds": rows(ei, co), "edge_peak_inds": rows(epi, co), "line_scores": rows(ls, co)}


def paf_params(ps, buffers, cm_output_stride, paf_output_stride, peak_threshold, refinement, integral_patch_size, input_scale,
               max_peaks_per_sample, max_node_peaks, max_instances):
    """BottomUpParams of the PAF chain of PAFScorer ``ps`` reading head ``buffers`` (cms, pafs, offsets), and the
    (edges, sorted edges) arrays its pointers point to, to keep alive while it is used."""
    edges = i32(ps.edge_inds).reshape(-1, 2)
    sorted_e = i32(list(ps.sorted_edge_inds))
    mip = ps.min_instance_peaks
    if isinstance(mip, float):
        mip = int(mip * ps.n_nodes)
    p = BottomUpParams(*buffers, int(cm_output_stride), int(paf_output_stride), float(peak_threshold), REFINE.get(refinement, 0),
                       int(integral_patch_size), ps.n_nodes, ps.n_edges, edges.ctypes.data, sorted_e.ctypes.data, len(sorted_e),
                       int(ps.n_points), float(ps.max_edge_length_ratio), float(ps.dist_penalty_weight), float(ps.min_line_scores),
                       int(mip), float(input_scale), int(max_peaks_per_sample), int(max_node_peaks), int(max_instances))
    return p, (edges, sorted_e)


def bottomup_from_maps(cms, pafs, paf_scorer, cm_output_stride, peak_threshold=0.2, refinement="integral",
                       integral_patch_size=5, offsets=None, input_scale=1.0, max_peaks_per_sample=1024,
                       max_node_peaks=32, max_instances=64, return_paf_graph=True, handle=None):
    """The BottomUpInferenceLayer post-processing chain (inference.py:2892-3003) on caller-supplied
    confidence maps / PAFs -- the parity entry point (identical maps in, bit-exact instances out)."""
    h = handle or _lib.default_handle()
    cms, pafs = f32(cms), f32(pafs)
    B, H, W, C = cms.shape
    _, Hp, Wp, C2 = pafs.shape
    ps = paf_scorer
    p, keep = paf_params(ps, (-1, -1, -1), cm_output_stride, ps.pafs_stride, peak_threshold, refinement, integral_patch_size,
                         input_scale, max_peaks_per_sample, max_node_peaks, max_instances)
    I, N = max_instances, ps.n_nodes
    ip = np.zeros((B, I, N, 2), np.float32); iv = np.zeros((B, I, N), np.float32); isc = np.zeros((B, I), np.float32)
    nv = np.zeros((B,), np.int32); fl = np.zeros((B,), np.int32)
    pks, cands = _paf_graph_arrays(B, max_peaks_per_sample, ps.n_edges, max_node_peaks)
    off = None if offsets is None else f32(offsets)
    h.call("sb_bottomup_from_maps", byref(p), ptr(cms), B, H, W, ptr(pafs), Hp, Wp, ptr(off), ptr(ip), ptr(iv), ptr(isc),
           ptr(nv), ptr(fl), len(pks[0]), ptr(pks[0]) if return_paf_graph else None, *map(ptr, pks[1:]), len(cands[0]),
           *map(ptr, cands))
    out = {"instance_peaks": [ip[b, :nv[b]].copy() for b in range(B)],
           "instance_peak_vals": [iv[b, :nv[b]].copy() for b in range(B)],
           "instance_scores": [isc[b, :nv[b]].copy() for b in range(B)], "n_valid": nv, "flags": fl}
    if return_paf_graph:
        out.update(_paf_graph_rows(pks, cands))
    return out


def _pipelined_batches(batches, m, submit_fn, collect):
    """The double-buffered batch loop of the streaming models (uint8 frames, chain configured): batch i+1 is submitted
    (``submit_fn`` of device model ``m``: its upload on the copy stream, network and post-processing queued) into slot
    (i+1) % 2 before ``collect(slot, B)`` waits for batch i and returns its result dict.  ``batches`` yields each batch's
    arrays the submit takes before B: its prepped frames and, for sb_topdown_gt_submit, its centroid table and counts;
    they are kept alive until the batch is collected.  A batch is drawn from ``batches`` only when it is submitted.  A
    consumer that stops early (an exception, a closed generator) leaves no batch submitted: the rest are collected and
    dropped."""
    it = iter(batches)
    keep, sizes = {}, {}

    def submit(k):
        arrays = next(it, None)
        if arrays is None:
            return
        keep[k % 2] = arrays                      # the async copies read these host buffers until collect()
        B = arrays[0].shape[0]
        m.handle.call(submit_fn, m.model_id, *[ptr(a) for a in arrays], B, k % 2)
        sizes[k] = B

    try:
        submit(0)
        k = 0
        while k in sizes:
            submit(k + 1)
            yield collect(k % 2, sizes.pop(k))
            k += 1
    finally:
        for k in sorted(sizes):
            try:
                collect(k % 2, sizes[k])
            except _lib.SleapB200Error:
                pass                                  # already failed: the error that stopped the loop is the one to see


class BottomUpInferenceModel(InferenceModel):
    """sleap/nn/inference.py:3006-3052."""

    def __init__(self, bottomup_layer: BottomUpInferenceLayer):
        self.bottomup_layer = bottomup_layer

    def call(self, example):
        return self.bottomup_layer.call(example)

    def _stream(self, first, batch_size):
        """sb_bottomup_submit / sb_bottomup_collect: uint8 frames without return_confmaps, return_pafs or
        return_paf_graph."""
        layer = self.bottomup_layer
        if first.dtype != np.uint8 or layer.return_confmaps or layer.return_pafs or layer.return_paf_graph:
            return None
        layer._configure(batch_size, *first.shape[1:])
        layer.attach_tracker(first.shape[1:3])
        return (layer.keras_model, "sb_bottomup_submit",
                lambda slot, B: layer._run_step(B, "sb_bottomup_collect", slot, slot=slot))


# ------------------------------------------------------------------------------------------
class BottomUpMultiClassInferenceLayer(InferenceLayer):
    """sleap/nn/inference.py:3351-3589: network (confidence maps + class maps) -> local peaks -> identity grouping by the
    class-map probability at each peak, executed as one device step (``sb_infer_multiclass``): k_class_group samples
    the class-map logits at the rounded peak cells, applies the sigmoid (``identity.class_probabilities``) and solves
    each (frame, node) assignment of peaks to classes, as ``identity.classify_peaks_from_maps`` does on the host."""

    CMS, CLASS_MAPS, OFFSETS = "MultiInstanceConfmapsHead", "ClassMapsHead", "OffsetRefinementHead"
    CHAIN = "sb_multiclass_configure"

    def __init__(self, keras_model, input_scale=1.0, pad_to_stride=1, cm_output_stride=None, class_maps_output_stride=None,
                 peak_threshold=0.2, refinement="integral", integral_patch_size=5, return_confmaps=False,
                 return_class_maps=False, max_peaks_per_sample=1024, max_node_peaks=32, **kwargs):
        super().__init__(keras_model, input_scale=input_scale, pad_to_stride=pad_to_stride, **kwargs)
        heads = keras_model.cm.head_buffers
        if self.CMS not in heads:
            raise ValueError("Index of the confidence maps output tensor must be specified if not named 'MultiInstanceConfmapsHead'.")
        if self.CLASS_MAPS not in heads:
            raise ValueError("Index of the class maps output tensor must be specified if not named 'ClassMapsHead'.")
        self.has_offsets = self.OFFSETS in heads
        self.cm_output_stride = cm_output_stride or keras_model.cm.head_strides[self.CMS]
        self.class_maps_output_stride = class_maps_output_stride or keras_model.cm.head_strides[self.CLASS_MAPS]
        self.peak_threshold = peak_threshold
        self.refinement = refinement
        self.integral_patch_size = integral_patch_size
        self.return_confmaps = return_confmaps
        self.return_class_maps = return_class_maps
        self.max_peaks_per_sample = max_peaks_per_sample
        self.max_node_peaks = max_node_peaks
        self.n_nodes, self.n_classes = int(head_channels(keras_model, self.CMS)), int(head_channels(keras_model, self.CLASS_MAPS))

    def params(self) -> MultiClassParams:
        heads = self.keras_model.cm.head_buffers
        return class_params((heads[self.CMS], heads[self.CLASS_MAPS], heads[self.OFFSETS] if self.has_offsets else -1),
                            self.cm_output_stride, self.class_maps_output_stride, self.peak_threshold, self.refinement,
                            self.integral_patch_size, self.n_nodes, self.n_classes, self.input_scale, self.max_peaks_per_sample,
                            self.max_node_peaks)

    def _outputs(self, B):
        K, N = self.n_classes, self.n_nodes
        return (np.zeros((B, K, N, 2), np.float32), np.zeros((B, K, N), np.float32), np.zeros((B, K, N), np.float32),
                np.zeros((B,), np.int32))

    def _run_step(self, B, fn, *args):
        """One call ``fn(model id, *args, B, <outputs>)`` (sb_infer_multiclass or sb_multiclass_collect) into B frames'
        instances, one per class, as a batch dict."""
        m = self.keras_model
        pts, vals, probs, fl = self._outputs(B)
        m.handle.call(fn, m.model_id, *args, B, ptr(pts), ptr(vals), ptr(probs), ptr(fl))
        return {"instance_peaks": pts, "instance_peak_vals": vals, "instance_scores": probs, "flags": fl}

    def call(self, data):
        """:3530-3589."""
        from sleap_b200.nn import identity
        imgs = self._prep(_images_of(data))
        B, H, W, C = imgs.shape
        self._configure(B, H, W, C)
        out = self._run_step(B, "sb_infer_multiclass", ptr(imgs), int(imgs.dtype == np.uint8))
        if self.return_confmaps or self.return_class_maps:
            cms, logits = self.keras_model.forward(imgs, [self.CMS, self.CLASS_MAPS])
            if self.return_confmaps:
                out["confmaps"] = cms
            if self.return_class_maps:
                out["class_maps"] = identity.class_probabilities(logits)
        return out


def class_params(buffers, cm_output_stride, class_maps_output_stride, peak_threshold, refinement, integral_patch_size, n_nodes,
                 n_classes, input_scale, max_peaks_per_sample, max_node_peaks):
    """MultiClassParams of the identity chain reading head ``buffers`` (cms, class maps, offsets)."""
    return MultiClassParams(*buffers, int(cm_output_stride), int(class_maps_output_stride), float(peak_threshold),
                            REFINE.get(refinement, 0), int(integral_patch_size), int(n_nodes), int(n_classes), float(input_scale),
                            int(max_peaks_per_sample), int(max_node_peaks))


def bottomup_multiclass_from_maps(cms, class_logits, cm_output_stride, class_maps_output_stride, peak_threshold=0.2,
                                  refinement="integral", integral_patch_size=5, offsets=None, input_scale=1.0,
                                  max_peaks_per_sample=1024, max_node_peaks=32, handle=None):
    """The BottomUpMultiClassInferenceLayer post-processing (local peaks + k_class_group) on caller-supplied confidence
    maps (B,H,W,n_nodes) and class-map logits (B,Hc,Wc,n_classes), before the sigmoid -- the parity entry point.  Returns
    the layer's keys: instance_peaks (B,n_classes,n_nodes,2), instance_peak_vals, instance_scores, flags."""
    h = handle or _lib.default_handle()
    cms, class_logits = f32(cms), f32(class_logits)
    B, H, W, N = cms.shape
    _, Hc, Wc, K = class_logits.shape
    p = class_params((-1, -1, -1), cm_output_stride, class_maps_output_stride, peak_threshold, refinement, integral_patch_size,
                     N, K, input_scale, max_peaks_per_sample, max_node_peaks)
    pts = np.zeros((B, K, N, 2), np.float32); vals = np.zeros((B, K, N), np.float32); probs = np.zeros((B, K, N), np.float32)
    fl = np.zeros((B,), np.int32)
    off = None if offsets is None else f32(offsets)
    h.call("sb_multiclass_from_maps", byref(p), ptr(cms), B, H, W, ptr(class_logits), Hc, Wc, ptr(off), ptr(pts), ptr(vals),
           ptr(probs), ptr(fl))
    return {"instance_peaks": pts, "instance_peak_vals": vals, "instance_scores": probs, "flags": fl}


class BottomUpMultiClassInferenceModel(InferenceModel):
    """sleap/nn/inference.py:3592-3635."""

    def __init__(self, inference_layer: BottomUpMultiClassInferenceLayer):
        self.inference_layer = inference_layer

    def call(self, example):
        return self.inference_layer.call(example)

    def _stream(self, first, batch_size):
        """sb_multiclass_submit / sb_multiclass_collect: uint8 frames without return_confmaps or return_class_maps."""
        layer = self.inference_layer
        if first.dtype != np.uint8 or layer.return_confmaps or layer.return_class_maps:
            return None
        layer._configure(batch_size, *first.shape[1:])
        return layer.keras_model, "sb_multiclass_submit", lambda slot, B: layer._run_step(B, "sb_multiclass_collect", slot)


class TopDownMultiClassFindPeaks(InferenceLayer):
    """sleap/nn/inference.py:3863-4136: centered-instance confidence maps + class vectors on crops -> global peaks ->
    one instance per class and sample (``identity.classify_peaks_from_vectors``).  Confidence maps and the class-vector
    head's feature map come from one device pass; the head's dense layers and the grouping run on the host.  (Inside a
    fused TopDownMultiClassInferenceModel both run on the device instead.)"""

    HEAD, CLASS_VECTORS = "CenteredInstanceConfmapsHead", "ClassVectorsHead"

    def __init__(self, keras_model, input_scale=1.0, output_stride=None, peak_threshold=0.2, refinement="local",
                 integral_patch_size=5, return_confmaps=False, return_class_vectors=False, optimal_grouping=True,
                 max_crops_per_call=64, **kwargs):
        super().__init__(keras_model, input_scale=input_scale, pad_to_stride=1, **kwargs)
        if self.HEAD not in keras_model.cm.head_buffers:
            raise ValueError(f"Index of the confidence maps output tensor must be specified if not named '{self.HEAD}'.")
        if "ClassVectorsHead" not in keras_model.cm.vector_taps:
            raise ValueError("Index of the classifier output tensor must be specified if not named 'ClassVectorsHead'.")
        self.has_offsets = "OffsetRefinementHead" in keras_model.cm.head_buffers
        self.output_stride = output_stride or keras_model.cm.head_strides[self.HEAD]
        self.peak_threshold = peak_threshold
        self.refinement = refinement
        self.integral_patch_size = integral_patch_size
        self.return_confmaps = return_confmaps
        self.return_class_vectors = return_class_vectors
        self.optimal_grouping = optimal_grouping
        self.max_crops_per_call = max_crops_per_call
        self.class_head = head_spec(keras_model.spec, self.CLASS_VECTORS)
        self.dense = pack_dense_weights(self.class_head, keras_model.dense_weights)     # what the fused step uploads

    def params(self) -> GlobalParams:
        """The global-peak chain of the fused top-down step (find_global_peaks, or with offsets, x output_stride)."""
        heads = self.keras_model.cm.head_buffers
        return GlobalParams(heads[self.HEAD], heads["OffsetRefinementHead"] if self.has_offsets else -1, int(self.output_stride),
                            float(self.peak_threshold), REFINE.get(self.refinement, 0), int(self.integral_patch_size),
                            float(self.input_scale))

    def call(self, inputs):
        from sleap_b200.nn import identity
        if isinstance(inputs, dict):
            crops = inputs["crops"]
        else:
            crops, inputs = inputs, {}
        crops = self._prep(crops)
        n = crops.shape[0]
        if "crop_sample_inds" in inputs:
            samples, sinds = int(inputs["samples"]), np.asarray(inputs["crop_sample_inds"], np.int32)
        else:
            samples, sinds = n, np.arange(n, dtype=np.int32)
        m = self.keras_model
        n_nodes, n_classes = head_channels(m, self.HEAD), head_channels(m, "ClassVectorsHead")
        pts = np.zeros((n, n_nodes, 2), np.float32)
        vals = np.zeros((n, n_nodes), np.float32)
        probs = np.zeros((n, n_classes), np.float32)
        names = [self.HEAD, "ClassVectorsHead"] + (["OffsetRefinementHead"] if self.has_offsets else [])
        all_cms = []
        for i in range(0, n, self.max_crops_per_call):
            sl = slice(i, min(n, i + self.max_crops_per_call))
            outs = m.forward(np.ascontiguousarray(crops[sl]), names)
            cms, probs[sl] = outs[0], outs[1]
            if self.has_offsets:
                pts[sl], vals[sl] = peak_finding.find_global_peaks_with_offsets(cms, outs[2], threshold=self.peak_threshold, handle=m.handle)
            else:
                pts[sl], vals[sl] = peak_finding.find_global_peaks(cms, threshold=self.peak_threshold, refinement=self.refinement,
                                                                   integral_patch_size=self.integral_patch_size, handle=m.handle)
            if self.return_confmaps:
                all_cms.append(cms)
        pts = (pts * np.float32(self.output_stride)).astype(np.float32)                      # :4076-4082
        if self.input_scale != 1.0:
            pts = (pts / np.float32(self.input_scale) + np.float32(0.5)).astype(np.float32)
        if inputs.get("crop_offsets") is not None:
            pts = (pts + f32(inputs["crop_offsets"]).reshape(n, 1, 2)).astype(np.float32)     # :4084-4088
        if self.optimal_grouping:
            points, point_vals, class_probs = identity.classify_peaks_from_vectors(pts, vals, probs, sinds, samples)
            out = {"instance_peaks": points, "instance_peak_vals": point_vals, "instance_scores": class_probs}
        else:
            out = {"instance_peaks": pts, "instance_peak_vals": vals, "instance_scores": probs}
        for k in ("centroids", "centroid_vals"):
            if k in inputs:
                out[k] = inputs[k]
        if self.return_confmaps:
            cms = np.concatenate(all_cms) if all_cms else np.zeros((0,), np.float32)
            out["instance_confmaps"] = [cms[sinds == s_] for s_ in range(samples)]
        if self.return_class_vectors and self.optimal_grouping:
            out["class_vectors"] = probs
        return out


def topdown_multiclass_params(topdown, tap, head, dense):
    """TopdownMultiClassParams over ``topdown`` (TopdownParams) for the class-vector head ``head`` (its spec entry) reading
    ``tap`` (an entry of ``CompiledModel.vector_taps``; None: no tap) with the packed weights ``dense``, which must outlive
    the call that takes the parameters."""
    tap = tap or dict(buf=-1, coff=0, C=0, planes=1)
    return TopdownMultiClassParams(topdown, int(tap["buf"]), int(tap["coff"]), int(tap["C"]), int(tap["planes"]), int(head["channels"]),
                                   int(head.get("num_fc_layers", 1)), int(head.get("num_fc_units", 64)),
                                   int(bool(head.get("global_pool", True))), dense.ctypes.data, int(dense.size))


def topdown_multiclass_from_features(cms, features, crop_sample_inds, n_samples, head, dense_weights, output_stride,
                                     peak_threshold=0.2, refinement="local", integral_patch_size=5, offsets=None, crop_offsets=None,
                                     input_scale=1.0, handle=None):
    """The post-processing of the fused top-down multi-class step (global peaks x output_stride + crop offsets,
    k_class_vectors, k_td_class_assign) on caller-supplied crops: confidence maps (n_crops,H,W,n_nodes), feature maps
    (n_crops,Hf,Wf,Cf) as the class-vector head ``head`` taps them, the head's dense weights (``{layer: {kernel, bias}}``)
    and the crops' frames (non-decreasing) -- the parity entry point.  Returns the fused keys instance_peaks
    (n_samples,n_classes,n_nodes,2), instance_peak_vals, instance_scores (n_samples,n_classes), plus class_vectors
    (n_crops,n_classes) and features (n_crops, the first dense layer's input)."""
    h = handle or _lib.default_handle()
    cms, features = f32(cms), f32(features)
    n, H, W, N = cms.shape
    _, Hf, Wf, Cf = features.shape
    dense = pack_dense_weights(head, dense_weights)
    gp = GlobalParams(-1, -1, int(output_stride), float(peak_threshold), REFINE.get(refinement, 0), int(integral_patch_size),
                      float(input_scale))
    p = topdown_multiclass_params(TopdownParams(-1, -1, CentroidParams(), gp, 0, 0, 0, 0), None, head, dense)
    B, NC = int(n_samples), p.n_classes
    pts = np.zeros((B, NC, N, 2), np.float32); vals = np.zeros((B, NC, N), np.float32); probs = np.zeros((B, NC), np.float32)
    cvec = np.zeros((n, NC), np.float32)
    feats = np.zeros((n, Cf if p.global_pool else Hf * Wf * Cf), np.float32)
    off = None if offsets is None else f32(offsets)
    co = None if crop_offsets is None else f32(crop_offsets).reshape(n, 2)
    h.call("sb_topdown_multiclass_from_features", byref(p), ptr(cms), n, H, W, N, ptr(off), ptr(features), Hf, Wf, Cf, ptr(co),
           ptr(i32(crop_sample_inds)), B, ptr(pts), ptr(vals), ptr(probs), ptr(cvec), ptr(feats))
    return {"instance_peaks": pts, "instance_peak_vals": vals, "instance_scores": probs, "class_vectors": cvec, "features": feats}


class TopDownMultiClassInferenceModel(TopDownInferenceModel):
    """sleap/nn/inference.py:4139-4210: centroid stage (model or ground truth) -> TopDownMultiClassFindPeaks.

    The whole chain runs as one device step (``sb_infer_topdown_multiclass``): centroids, top-k, crops, instance network,
    global peaks, the class-vector head (k_class_vectors) and the per-frame assignment of crops to classes
    (k_td_class_assign); with ground-truth centroids, the same step from the crops on.  ``fused = False`` keeps the staged
    path."""

    CONFIGURE, INFER = "sb_topdown_multiclass_configure", "sb_infer_topdown_multiclass"
    SUBMIT, COLLECT = "sb_topdown_multiclass_submit", "sb_topdown_multiclass_collect"

    def _can_fuse(self):
        cc, fp = self.centroid_crop, self.instance_peaks
        if not (self.fused and type(fp) is TopDownMultiClassFindPeaks and not fp.return_confmaps and fp.optimal_grouping and
                fp.input_scale == 1.0 and fp.keras_model.input_scale == 1.0):
            return False
        if type(cc) is CentroidCropGroundTruth:
            return cc.input_scale == 1.0 and cc.handle is fp.keras_model.handle
        return (type(cc) is CentroidCrop and cc.precrop_resize == 1.0 and cc.return_crops and not cc.return_confmaps
                and cc.keras_model.handle is fp.keras_model.handle)

    @property
    def _keep(self):
        return (self.instance_peaks.dense,)

    def _params(self, td):
        fp = self.instance_peaks
        return topdown_multiclass_params(td, fp.keras_model.cm.vector_taps[fp.CLASS_VECTORS], fp.class_head, fp.dense)

    def _run_fused(self, B, K, fn, *args, slot=0):
        """One fused call ``fn(model id, *args, B, <outputs>)`` (sb_infer_topdown_multiclass or
        sb_topdown_multiclass_collect) into dense arrays of B frames, as a batch dict (no tracker: ``slot`` is unused)."""
        fp, mc = self.instance_peaks, self._owner()
        N, NC = head_channels(fp.keras_model, fp.HEAD), int(fp.class_head["channels"])
        ce = np.zeros((B, K, 2), np.float32); cv = np.zeros((B, K), np.float32)
        pts = np.zeros((B, NC, N, 2), np.float32); vals = np.zeros((B, NC, N), np.float32); probs = np.zeros((B, NC), np.float32)
        nv = np.zeros((B,), np.int32); fl = np.zeros((B,), np.int32)
        cvec = np.zeros((B, K, NC), np.float32) if fp.return_class_vectors else None
        mc.handle.call(fn, mc.model_id, *args, B, ptr(ce), ptr(cv), ptr(pts), ptr(vals), ptr(probs), ptr(nv), ptr(fl), ptr(cvec))
        n = int(nv.max()) if B else 0
        out = {"instance_peaks": pts, "instance_peak_vals": vals, "instance_scores": probs, "centroids": ce[:, :n].copy(),
               "centroid_vals": cv[:, :n].copy(), "flags": fl}
        if cvec is not None:
            out["class_vectors"] = np.concatenate([cvec[b, :nv[b]] for b in range(B)])
        return out

    def _call_staged(self, example):
        crop_out = self.centroid_crop.call(example)
        out = self.instance_peaks.call(crop_out)
        res = {k: out[k] for k in ("instance_peaks", "instance_peak_vals", "instance_scores")}
        if "centroids" in out:
            res["centroids"], _ = _ragged_to_dense(out["centroids"], (2,))
            res["centroid_vals"], _ = _ragged_to_dense(out["centroid_vals"], ())
        return res


class PredictedInstance:
    """Array contract of ``sleap.PredictedInstance.from_numpy`` (sleap/instance.py:1164)."""

    def __init__(self, points, point_confidences, instance_score, skeleton=None, track=None, tracking_score=0.0):
        self.points = np.asarray(points)
        self.point_confidences = np.asarray(point_confidences)
        self.score = float(instance_score)
        self.skeleton = skeleton
        self.track = track
        self.tracking_score = float(tracking_score)

    @classmethod
    def from_numpy(cls, points, point_confidences, instance_score, skeleton=None, track=None, tracking_score=0.0):
        return cls(points, point_confidences, instance_score, skeleton, track, tracking_score)

    def numpy(self):
        return self.points

    @property
    def n_visible_points(self):
        return int(np.sum(~np.isnan(self.points).any(axis=1)))


class LabeledFrame:
    def __init__(self, video, frame_idx, instances):
        self.video, self.frame_idx, self.instances = video, frame_idx, instances


class Predictor:
    """sleap/nn/inference.py:158-590."""

    verbosity = "none"
    report_rate = 2.0
    model_paths: List[str] = []
    tracker = None          # optional sleap_b200.nn.tracking.Tracker applied frame by frame (:3306-3313)

    def __init__(self, batch_size=4):
        self.batch_size = batch_size
        self.inference_model = None

    @classmethod
    def from_model_paths(cls, model_paths, peak_threshold=0.2, integral_refinement=True, integral_patch_size=5,
                         batch_size=4, resize_input_layer=True, max_instances=None, precision=PRECISION_FP16,
                         handle=None, **caps):
        """:176-311: dispatch on the head type found in each model's training_config.json."""
        if isinstance(model_paths, str):
            model_paths = [model_paths]
        if not model_paths:
            raise ValueError("Must specify at least one model path.")   # :2479
        cfgs = {}
        for p in model_paths:
            cfg, d = cls._read_config(p)
            heads = {k: v for k, v in cfg["model"]["heads"].items() if v is not None}
            cfgs[next(iter(heads))] = (cfg, d)
        kw = dict(peak_threshold=peak_threshold, integral_refinement=integral_refinement,
                  integral_patch_size=integral_patch_size, batch_size=batch_size, precision=precision, handle=handle)
        kw.update(caps)
        if "single_instance" in cfgs:
            return SingleInstancePredictor.from_trained_models(cfgs["single_instance"], **kw)
        if "multi_class_topdown" in cfgs:
            mk = {k: kw[k] for k in ("peak_threshold", "integral_refinement", "integral_patch_size", "batch_size", "precision", "handle")}
            return TopDownMultiClassPredictor.from_trained_models(centroid_model_path=cfgs.get("centroid"),
                                                                  confmap_model_path=cfgs["multi_class_topdown"], **mk)
        if "centroid" in cfgs or "centered_instance" in cfgs:
            return TopDownPredictor.from_trained_models(centroid_model_path=cfgs.get("centroid"),
                                                        confmap_model_path=cfgs.get("centered_instance"),
                                                        max_instances=max_instances, **kw)
        if "multi_instance" in cfgs:
            return BottomUpPredictor.from_trained_models(cfgs["multi_instance"], max_instances=max_instances, **kw)
        if "multi_class_bottomup" in cfgs:
            mk = {k: kw[k] for k in ("peak_threshold", "integral_refinement", "integral_patch_size", "batch_size", "precision", "handle",
                                     "max_peaks_per_sample", "max_node_peaks") if k in kw}
            return BottomUpMultiClassPredictor.from_trained_models(cfgs["multi_class_bottomup"], **mk)
        raise ValueError("Could not create predictor from model paths:" + "\n".join(model_paths))

    # -- shared helpers ---------------------------------------------------------------------
    @staticmethod
    def _read_config(model_path):
        """``TrainingJobConfig.load_json`` (config/training_job.py:93-124) on a model folder or a json inside it."""
        cfg_path = model_path if model_path.endswith(".json") else os.path.join(model_path, "training_config.json")
        with open(cfg_path) as f:
            return json.load(f), os.path.dirname(cfg_path)

    @staticmethod
    def _load(cfg_and_dir, precision, handle, resize_in_graph=True):
        """``resize_in_graph=False``: the network graph gets no resize op (top-down instance models: their crops come
        from frames that were already resized, FindInstancePeaks(resize_input_image=False), :2405-2413); the
        configured ``input_scaling`` is still returned through ``model.input_scale``."""
        if isinstance(cfg_and_dir, (str, os.PathLike)):        # the reference passes model paths here
            cfg_and_dir = Predictor._read_config(os.fspath(cfg_and_dir))
        cfg, d = cfg_and_dir
        spec = arch.spec_from_config(cfg["model"], *_skeleton_from_cfg(cfg))
        pre = cfg["data"]["preprocessing"]
        weights = load_weights(d)
        # The reference reads the channel count off the loaded Keras model's input (:905-911,
        # ``is_grayscale``); here it is the C_in of the first convolution's kernel.
        first = arch.compile_model(spec, 1).layers[0]["name"]
        in_ch = int(np.asarray(weights[first]["kernel"]).shape[2])
        if arch.resnet_pretrained(spec):
            # conv1_conv always sees 3 channels after tile_channels; the model's own input has 1 channel when it was
            # trained on grayscale frames (colour frames are then converted to gray before the tile, :1477, :3149)
            in_ch = 1 if pre.get("ensure_grayscale") else 3
        scale = float(pre.get("input_scaling", 1.0) or 1.0)
        model = DeviceModel(spec, weights, input_channels=in_ch, input_scale=scale if resize_in_graph else 1.0,
                            pad_to_stride=pre.get("pad_to_stride"), precision=precision, handle=handle)
        model.config_input_scale = scale
        return cfg, spec, model

    def _as_frames(self, data):
        """``predict`` accepts a video path, ``Video`` or ``VideoReader`` provider (:496-531, make_pipeline :329-371):
        those are read through the threaded ``FrameFeeder`` (decode ahead into pinned batch buffers)."""
        from sleap_b200.io.video import FrameFeeder, Video, VideoReader
        if isinstance(data, (str, os.PathLike, Video, VideoReader)):
            return FrameFeeder(data, batch_size=self.batch_size)
        return data

    def _label_examples(self, reader):
        """Batches of labels examples (make_pipeline with a LabelsReader, :329-371): stacked frames plus the
        per-sample ground-truth ``instances`` / ``centroids`` the stand-in layers read."""
        idx = reader.indices()
        for i in range(0, len(idx), self.batch_size):
            exs = [reader.example(j) for j in idx[i:i + self.batch_size]]
            batch = {"image": np.stack([e["image"] for e in exs]), "instances": [e["instances"] for e in exs],
                     "frame_ind": np.asarray([e["frame_ind"] for e in exs]), "video_ind": np.asarray([e["video_ind"] for e in exs])}
            if "centroids" in exs[0]:
                batch["centroids"] = [e["centroids"] for e in exs]
            yield batch

    def _predict_generator(self, data):
        """:377-420: the inference model's batch loop (+ frame indices)."""
        from sleap_b200.io.labels import Labels, LabelsReader
        from sleap_b200.io.video import FrameFeeder
        if isinstance(data, Labels):
            data = LabelsReader(data, with_centroids=True, center_on_part=getattr(self, "anchor_part", None))
        if isinstance(data, LabelsReader):
            batches = self._label_examples(data)
            if getattr(self, "uses_ground_truth", False):     # streamed where the model's ground-truth step takes them
                results = self.inference_model.predict_examples(batches, self.batch_size, data.max_instance_count())
            else:
                results = ((b, self.inference_model.predict_on_batch(b["image"])) for b in batches)
            with contextlib.closing(results):
                for batch, ex in results:
                    ex["frame_ind"], ex["video_ind"] = batch["frame_ind"], batch["video_ind"]
                    ex["image_hw"] = tuple(batch["image"].shape[1:3])
                    if self.tracker is not None and getattr(self.tracker, "uses_image", False):
                        ex["image"] = batch["image"]
                    self._check_flags(ex)
                    yield ex
            return
        data = self._as_frames(data)
        feeder = data if isinstance(data, FrameFeeder) else None
        frame_inds = (lambda a, b: np.asarray(feeder.inds[a:b])) if feeder is not None else (lambda a, b: np.arange(a, b))
        try:
            i0 = 0
            want_img = self.tracker is not None and getattr(self.tracker, "uses_image", False)   # flow trackers (:2664-2671)
            imgs_all = _images_of(data)
            hw = tuple(np.asarray(imgs_all[0]).shape[:2]) if len(imgs_all) else (1, 1)
            for ex in self.inference_model.predict_batches(imgs_all, self.batch_size):
                n = len(ex["instance_peaks"])
                ex["frame_ind"] = frame_inds(i0, i0 + n)
                ex["video_ind"] = np.zeros(n, np.int64)
                ex["image_hw"] = hw
                if want_img:
                    ex["image"] = np.stack([np.asarray(imgs_all[j]) for j in range(i0, i0 + n)])
                i0 += n
                self._check_flags(ex)
                yield ex
        finally:
            if feeder is not None:
                feeder.close()

    # Device workspaces are capacity bounded (the reference's ragged tensors are not): a frame that hits a cap comes
    # back truncated with SB_FLAG_* bits set.  ``on_overflow``: "warn" (default), "raise" or "ignore".
    on_overflow = "warn"
    _FLAG_NAMES = {1: "max_peaks_per_sample", 2: "max_node_peaks", 4: "max_instances_per_frame"}   # SB_FLAG_* (include/sleap_b200.h)

    def _check_flags(self, ex):
        fl = ex.get("flags")
        if fl is None or self.on_overflow == "ignore":
            return
        fl = np.asarray(fl)
        if not fl.any():
            return
        bits = int(np.bitwise_or.reduce(fl.astype(np.int64)))
        names = [n for b, n in self._FLAG_NAMES.items() if bits & b] or [f"flags=0x{bits:x}"]
        frames = np.asarray(ex.get("frame_ind", np.arange(len(fl))))[fl != 0].tolist()
        msg = (f"device capacity reached ({', '.join(names)}) on frame(s) {frames[:8]}{'...' if len(frames) > 8 else ''}: "
               "detections were truncated; raise the corresponding cap (max_peaks_per_sample / max_node_peaks / "
               "max_instances_per_frame) when constructing the predictor")
        if self.on_overflow == "raise":
            raise OverflowError(msg)
        import warnings
        warnings.warn(msg, RuntimeWarning, stacklevel=3)

    def _with_progress(self, gen, n_total):
        """:422-491: ``verbosity`` = "none" | "json" (one JSON line per ``report_period`` seconds: n_processed, n_total, elapsed,
        rate over the last 30 batches, eta) | "rich" (a rich progress bar with the same rate estimate)."""
        import time
        from collections import deque
        if self.verbosity not in ("json", "rich"):
            yield from gen
            return
        n_processed, n_recent, el_recent = 0, deque(maxlen=30), deque(maxlen=30)
        t0_all = t0_batch = last_report = time.time()
        period = 1.0 / self.report_rate
        progress = task = None
        if self.verbosity == "rich":
            import rich.progress
            progress = rich.progress.Progress("{task.description}", rich.progress.BarColumn(), "[progress.percentage]{task.percentage:>3.0f}%",
                                              "ETA:", rich.progress.TimeRemainingColumn(), auto_refresh=False, speed_estimate_period=5)
            progress.start()
            task = progress.add_task("Predicting...", total=n_total)
        try:
            for ex in gen:
                now = time.time()
                n_batch = len(ex["frame_ind"])
                n_processed += n_batch
                n_recent.append(n_batch); el_recent.append(now - t0_batch)
                t0_batch = now
                rate = sum(n_recent) / max(sum(el_recent), 1e-9)
                if progress is not None:
                    progress.update(task, advance=n_batch)
                if now - last_report > period:
                    if progress is not None:
                        progress.refresh()
                    else:
                        print(json.dumps({"n_processed": n_processed, "n_total": n_total, "elapsed": now - t0_all, "rate": rate,
                                          "eta": (n_total - n_processed) / rate if n_total else None}), flush=True)
                    last_report = now
                yield ex
        finally:
            if progress is not None:
                progress.refresh()
                progress.stop()

    @staticmethod
    def _n_total(data):
        try:
            return len(_images_of(data))
        except TypeError:
            return len(getattr(data, "inds", [])) or None

    def predict(self, data, make_labels: bool = True):
        """:496-531."""
        gen = self._with_progress(self._predict_generator(data), self._n_total(data))
        try:
            if make_labels:
                return self._make_labeled_frames_from_generator(gen, data)
            return list(gen)
        finally:
            gen.close()           # a streamed batch loop stopped by an error collects what it submitted before this returns

    def skeleton(self):
        """Skeleton of the loaded model(s): node names (+ edges for bottom-up models), as the reference takes them
        from the training config (:1547-1560, :2562-2580, :3230-3240)."""
        from sleap_b200.io.labels import Skeleton
        for m in (getattr(self, "bottomup_model", None), getattr(self, "confmap_model", None), getattr(self, "centroid_model", None),
                  getattr(self, "model", None)):
            if m is not None and m.spec.get("part_names"):
                return Skeleton(m.spec["part_names"], m.spec.get("edges") or [])
        raise ValueError("the loaded model carries no part names")

    def to_labels(self, frames, video_filename: str = "", video_spec=None):
        """``predict(..., make_labels=True)`` output -> ``sleap_b200.io.labels.Labels`` (``.save("out.slp")`` writes the
        reference's HDF5 labels container, sleap/io/format/hdf5.py:265-575)."""
        from sleap_b200.io.labels import labels_from_predictions
        return labels_from_predictions(frames, self.skeleton(), video_spec, video_filename)

    def _make_labeled_frames_from_generator(self, generator, data):
        """:3230-3343 pattern: a consumer thread builds the objects while the batch loop runs."""
        q: "queue.Queue" = queue.Queue()
        frames: List[LabeledFrame] = []
        errors: list = []

        def worker():
            while True:
                ex = q.get()
                if ex is None:
                    return
                new = self._frames_from_example(ex)
                if "track_ids" in ex:                            # tracked on the device inside the step: map ids to Tracks
                    try:
                        self._apply_device_tracks(ex, new)
                    except Exception as e:                       # raised on the calling thread after the join
                        errors.append(e)
                        return
                elif self.tracker is not None:                   # sequential by nature; runs on the consumer thread
                    hw = tuple(ex.get("image_hw") or (1, 1))
                    for k, lf in enumerate(new):
                        img = ex["image"][k] if "image" in ex else None
                        lf.instances = self.tracker.track(lf.instances, img_hw=hw, img=img, t=lf.frame_idx)
                frames.extend(new)

        t = threading.Thread(target=worker)
        t.start()
        try:
            for ex in generator:
                q.put(ex)
        finally:
            q.put(None)
            t.join()
        if errors:
            raise errors[0]
        if self.tracker is not None:                                 # :2702-2703, :3345-3346
            self.tracker.final_pass(frames)
        return frames

    def _step_tracker(self, model, make_labels):
        """The tracker to run inside the device step of ``model`` (a Tracker with ``track_device``), or None when the
        step runs without one.  The tracker's GPU must be the model's, and the run must be on one rank."""
        tr = self.tracker
        if tr is None or getattr(tr, "track_device", None) is None or tr.candidate_maker is None:
            return None
        if int(str(tr.track_device).split(":")[-1]) != model.handle.device_id:
            raise ValueError(f"the tracker's track_device {tr.track_device!r} is not the model's GPU ({model.handle.device_id})")
        if getattr(model, "peer_gather", None) is not None or int(os.environ.get("WORLD_SIZE", "1")) > 1:
            raise ValueError("a device tracker tracks one rank's frames: run the multi-rank prediction without track_device")
        if not make_labels:                          # no labeled frames, nothing to track (as with the host tracker)
            return None
        return tr

    @contextlib.contextmanager
    def _tracking_in_step(self, owner, model, make_labels):
        """For the span of the block, the step tracker (``_step_tracker``) set as ``owner.tracker`` (the layer or model
        whose device step of ``model`` runs it), detached from the step after."""
        tr = self._step_tracker(model, make_labels)
        if tr is None:
            yield
            return
        owner.tracker = tr
        try:
            yield
        finally:
            owner.detach_tracker()
            owner.tracker = None

    def _apply_device_tracks(self, ex, new):
        """The frames' tracked lists from the track records of their step (a predictor with a device tracker)."""
        for k, lf in enumerate(new):
            flag = int(ex["track_flags"][k])
            if flag == 1:
                raise ValueError("cost matrix is infeasible")
            if flag == 3:                                # SB_TRACK_OVER_CAPACITY
                raise _lib.SleapB200Error(f"frame {lf.frame_idx} has {len(lf.instances)} instances, more than the device tracker's "
                                          f"capacity of {self.tracker._device.max_instances} (Tracker.device_max_instances)")
            if flag:
                raise _lib.SleapB200Error(f"the device tracker's track queue table is full (frame {lf.frame_idx})")
            n = int(ex["track_n"][k])
            lf.instances = self.tracker.apply_device_tracks(lf.instances, lf.frame_idx, ex["track_order"][k, :n],
                                                            ex["track_ids"][k, :n], ex["tracking_scores"][k, :n])

    def _frames_from_example(self, ex):
        out = []
        scores = ex.get("instance_scores")
        topdown = scores is None and "centroid_vals" in ex
        if topdown:                       # top-down: the instance score is the centroid confidence (:2640-2660)
            scores = ex["centroid_vals"]
        for i in range(len(ex["instance_peaks"])):
            insts = []
            for j in range(ex["instance_peaks"].shape[1]):
                pts = ex["instance_peaks"][i, j]
                if np.all(np.isnan(pts)):
                    continue   # :3285
                sc = float(scores[i, j]) if scores is not None else float(np.nansum(ex["instance_peak_vals"][i, j]))
                insts.append(PredictedInstance.from_numpy(pts, ex["instance_peak_vals"][i, j], sc))
            mi = None if topdown else getattr(self, "max_instances", None)   # top-down caps centroids (:1879-1894) only
            if mi is not None and len(insts) > mi:   # :3297
                insts = sorted(insts, key=lambda x: x.score, reverse=True)[:mi]
            out.append(LabeledFrame(int(ex["video_ind"][i]), int(ex["frame_ind"][i]), insts))
        return out


def _skeleton_from_cfg(cfg):
    sk = (cfg.get("data", {}).get("labels", {}).get("skeletons") or [None])[0]
    if not sk or "nodes" not in sk:
        return None, None
    try:
        names = [n["id"]["py/state"]["py/tuple"][0] if "py/state" in n["id"] else None for n in sk["nodes"]]
        if all(names):
            return names, None
    except Exception:
        pass
    return None, None


class SingleInstancePredictor(Predictor):
    """sleap/nn/inference.py:1418-1636."""

    def __init__(self, confmap_model, peak_threshold=0.2, integral_refinement=True, integral_patch_size=5,
                 batch_size=4):
        super().__init__(batch_size)
        self.confmap_model = confmap_model
        self.peak_threshold = peak_threshold
        self.integral_refinement = integral_refinement
        self.integral_patch_size = integral_patch_size
        self._initialize_inference_model()

    def _initialize_inference_model(self):
        """:1456-1478."""
        m = self.confmap_model
        self.inference_model = SingleInstanceInferenceModel(SingleInstanceInferenceLayer(
            keras_model=m, input_scale=m.input_scale, pad_to_stride=m.cm.max_stride,
            peak_threshold=self.peak_threshold, refinement="integral" if self.integral_refinement else "local",
            integral_patch_size=self.integral_patch_size))

    @classmethod
    def from_trained_models(cls, model_path, inference_object=None, peak_threshold=0.2, integral_refinement=True,
                            integral_patch_size=5, batch_size=4, resize_input_layer=True, precision=PRECISION_FP16,
                            handle=None, **_):
        """:1480-1545 (same argument names; ``model_path`` may also be a loaded (config, folder) pair)."""
        _, _, model = cls._load(model_path, precision, handle)
        return cls(model, peak_threshold, integral_refinement, integral_patch_size, batch_size)


class TopDownPredictor(Predictor):
    """sleap/nn/inference.py:2314-2735."""

    def __init__(self, centroid_model=None, confmap_model=None, crop_size=160, peak_threshold=0.2,
                 integral_refinement=True, integral_patch_size=5, batch_size=4, max_instances=None,
                 max_peaks_per_sample=256):
        super().__init__(batch_size)
        self.max_peaks_per_sample = max_peaks_per_sample
        if centroid_model is None and confmap_model is None:
            raise ValueError("Either the centroid or topdown confidence map model must be provided.")   # :2479
        self.centroid_model, self.confmap_model = centroid_model, confmap_model
        self.anchor_part = None          # instance_cropping.center_on_part of the model config (ground-truth centroids)
        self.crop_size = crop_size
        self.peak_threshold = peak_threshold
        self.integral_refinement = integral_refinement
        self.integral_patch_size = integral_patch_size
        self.max_instances = max_instances
        self._initialize_inference_model()

    def _initialize_inference_model(self):
        """:2373-2433."""
        ref = "integral" if self.integral_refinement else "local"
        cm, im = self.centroid_model, self.confmap_model
        if cm is None:                                   # ground-truth centroids stand in for the centroid model
            cc = CentroidCropGroundTruth(crop_size=self.crop_size, handle=im.handle)
        else:
            cc = CentroidCrop(keras_model=cm, crop_size=self.crop_size if im is not None else 1, input_scale=cm.input_scale,
                              pad_to_stride=cm.cm.max_stride, peak_threshold=self.peak_threshold, refinement=ref,
                              integral_patch_size=self.integral_patch_size, max_instances=self.max_instances,
                              return_crops=im is not None, max_peaks_per_sample=self.max_peaks_per_sample)
        if im is None:                                   # ground-truth instances stand in for the instance model
            fp = FindInstancePeaksGroundTruth()
        else:
            iscale = float(getattr(im, "config_input_scale", im.input_scale))
            if im.input_scale != 1.0:
                raise ValueError("top-down instance models must be built without a resize op (resize_input_image=False)")
            fp = FindInstancePeaks(keras_model=im, input_scale=iscale, peak_threshold=self.peak_threshold,
                                   refinement=ref, integral_patch_size=self.integral_patch_size)
            if cm is None:
                cc.input_scale = iscale                  # :2414-2415
            else:
                cc.precrop_resize = iscale               # :2416-2419
        self.inference_model = TopDownInferenceModel(cc, fp)

    @property
    def uses_ground_truth(self):
        return self.centroid_model is None or self.confmap_model is None

    def predict(self, data, make_labels: bool = True):
        """As Predictor.predict.  On the fused step (frames in, not ``Labels``), a tracker with ``track_device`` runs
        inside each step (k_track after the record kernel, on the model's GPU); the consumer thread only maps its track
        ids to ``Track`` objects before ``final_pass``.  The tracker's GPU must be the model's, and the run must be on
        one rank.  Other inputs, and ground-truth centroids, track on the consumer thread."""
        from sleap_b200.io.labels import Labels, LabelsReader
        im = self.inference_model
        if not im._can_fuse() or im.ground_truth or isinstance(data, (Labels, LabelsReader)):
            return super().predict(data, make_labels)
        with self._tracking_in_step(im, im.centroid_crop.keras_model, make_labels):
            return super().predict(data, make_labels)

    @classmethod
    def from_trained_models(cls, centroid_model_path=None, confmap_model_path=None, batch_size=4, peak_threshold=0.2,
                            integral_refinement=True, integral_patch_size=5, resize_input_layer=True,
                            max_instances=None, precision=PRECISION_FP16, handle=None, max_peaks_per_sample=256, **_):
        """:2435-2560 (same argument names; paths may also be loaded (config, folder) pairs)."""
        centroid_cfg, confmap_cfg = centroid_model_path, confmap_model_path
        if centroid_cfg is None and confmap_cfg is None:
            raise ValueError("Either the centroid or topdown confidence map model must be provided.")  # :2479
        cmodel = imodel = None
        crop, anchor = 1, None
        if centroid_cfg is not None:
            ccfg, _, cmodel = cls._load(centroid_cfg, precision, handle)
            anchor = ccfg["data"]["instance_cropping"].get("center_on_part")
        if confmap_cfg is not None:
            icfg, _, imodel = cls._load(confmap_cfg, precision, handle, resize_in_graph=False)
            crop = icfg["data"]["instance_cropping"]["crop_size"]
            anchor = icfg["data"]["instance_cropping"].get("center_on_part") if anchor is None else anchor
        obj = cls(cmodel, imodel, crop, peak_threshold, integral_refinement, integral_patch_size, batch_size, max_instances,
                  max_peaks_per_sample)
        obj.anchor_part = anchor
        return obj


class BottomUpPredictor(Predictor):
    """sleap/nn/inference.py:3055-3349 (attrs :3104-3117)."""

    def __init__(self, bottomup_model, part_names, edges, peak_threshold=0.2, batch_size=4, max_edge_length_ratio=0.25,
                 dist_penalty_weight=1.0, paf_line_points=10, min_line_scores=0.25, integral_refinement=True,
                 integral_patch_size=5, max_instances=None, max_peaks_per_sample=1024, max_node_peaks=32,
                 max_instances_per_frame=64):
        super().__init__(batch_size)
        self.bottomup_model = bottomup_model
        self.part_names, self.edges = list(part_names), [tuple(e) for e in edges]
        self.peak_threshold = peak_threshold
        self.max_edge_length_ratio = max_edge_length_ratio
        self.dist_penalty_weight = dist_penalty_weight
        self.paf_line_points = paf_line_points
        self.min_line_scores = min_line_scores
        self.integral_refinement = integral_refinement
        self.integral_patch_size = integral_patch_size
        self.max_instances = max_instances
        self._caps = (max_peaks_per_sample, max_node_peaks, max_instances_per_frame)
        self._initialize_inference_model()

    def predict(self, data, make_labels: bool = True):
        """As Predictor.predict.  A tracker with ``track_device`` runs inside each bottom-up step (k_track after the
        grouping kernel, on the model's GPU); the consumer thread only maps its track ids to ``Track`` objects before
        ``final_pass``.  The tracker's GPU must be the model's, and the run must be on one rank."""
        layer = self.inference_model.bottomup_layer
        layer.tracker_cut = -1 if self.max_instances is None else int(self.max_instances)
        with self._tracking_in_step(layer, layer.keras_model, make_labels):
            return super().predict(data, make_labels)

    def _initialize_inference_model(self):
        """:3119-3150."""
        m = self.bottomup_model
        scorer = paf_grouping.PAFScorer(
            part_names=self.part_names, edges=self.edges, pafs_stride=m.cm.head_strides["PartAffinityFieldsHead"],
            max_edge_length_ratio=self.max_edge_length_ratio, dist_penalty_weight=self.dist_penalty_weight,
            n_points=self.paf_line_points, min_instance_peaks=0, min_line_scores=self.min_line_scores)
        self.inference_model = BottomUpInferenceModel(BottomUpInferenceLayer(
            keras_model=m, paf_scorer=scorer, input_scale=m.input_scale, pad_to_stride=m.cm.max_stride,
            peak_threshold=self.peak_threshold, refinement="integral" if self.integral_refinement else "local",
            integral_patch_size=self.integral_patch_size, max_peaks_per_sample=self._caps[0],
            max_node_peaks=self._caps[1], max_instances=self._caps[2]))

    @classmethod
    def from_trained_models(cls, model_path, batch_size=4, peak_threshold=0.2, integral_refinement=True,
                            integral_patch_size=5, max_edge_length_ratio=0.25, dist_penalty_weight=1.0,
                            paf_line_points=10, min_line_scores=0.25, resize_input_layer=True, max_instances=None,
                            precision=PRECISION_FP16, handle=None, max_peaks_per_sample=1024, max_node_peaks=32,
                            max_instances_per_frame=64, **_):
        """:3150-3228 (same argument names; ``model_path`` may also be an already loaded (config, folder) pair).
        ``max_peaks_per_sample`` / ``max_node_peaks`` / ``max_instances_per_frame`` size the device workspaces (the
        reference's ragged tensors are unbounded); a frame that reaches one is reported through ``on_overflow``."""
        _, spec, model = cls._load(model_path, precision, handle)
        return cls(model, spec["part_names"], spec["edges"], peak_threshold=peak_threshold, batch_size=batch_size,
                   max_edge_length_ratio=max_edge_length_ratio, dist_penalty_weight=dist_penalty_weight,
                   paf_line_points=paf_line_points, min_line_scores=min_line_scores,
                   integral_refinement=integral_refinement, integral_patch_size=integral_patch_size,
                   max_instances=max_instances, max_peaks_per_sample=max_peaks_per_sample, max_node_peaks=max_node_peaks,
                   max_instances_per_frame=max_instances_per_frame)


class BottomUpMultiClassPredictor(Predictor):
    """sleap/nn/inference.py:3638-3860: bottom-up identity models (confidence maps + class maps).  Instances come out one per
    class, in class order; each gets the ``Track`` named after its class (:3781-3790), ``score`` = mean point confidence and
    ``tracking_score`` = mean class probability (:3818-3826)."""

    def __init__(self, model, classes, peak_threshold=0.2, batch_size=4, integral_refinement=True, integral_patch_size=5, tracks=None,
                 max_peaks_per_sample=1024, max_node_peaks=32):
        super().__init__(batch_size)
        self.model = model
        self.classes = list(classes)
        self.peak_threshold = peak_threshold
        self.integral_refinement = integral_refinement
        self.integral_patch_size = integral_patch_size
        self.tracks = tracks
        self._caps = (max_peaks_per_sample, max_node_peaks)
        self._initialize_inference_model()

    def _initialize_inference_model(self):
        """:3682-3697."""
        m = self.model
        self.inference_model = BottomUpMultiClassInferenceModel(BottomUpMultiClassInferenceLayer(
            keras_model=m, input_scale=m.input_scale, pad_to_stride=m.cm.max_stride, peak_threshold=self.peak_threshold,
            refinement="integral" if self.integral_refinement else "local", integral_patch_size=self.integral_patch_size,
            cm_output_stride=m.cm.head_strides["MultiInstanceConfmapsHead"],
            class_maps_output_stride=m.cm.head_strides["ClassMapsHead"], max_peaks_per_sample=self._caps[0],
            max_node_peaks=self._caps[1]))

    @classmethod
    def from_trained_models(cls, model_path, batch_size=4, peak_threshold=0.2, integral_refinement=True, integral_patch_size=5,
                            resize_input_layer=True, precision=PRECISION_FP16, handle=None, max_peaks_per_sample=1024,
                            max_node_peaks=32, **_):
        """:3699-3745.  ``max_peaks_per_sample`` / ``max_node_peaks`` size the device workspace (the reference's ragged
        tensors are unbounded); a frame that reaches one is reported through ``on_overflow``."""
        _, spec, model = cls._load(model_path, precision, handle)
        return cls(model, spec["classes"], peak_threshold=peak_threshold, batch_size=batch_size,
                   integral_refinement=integral_refinement, integral_patch_size=integral_patch_size,
                   max_peaks_per_sample=max_peaks_per_sample, max_node_peaks=max_node_peaks)

    def _frames_from_example(self, ex):
        """:3781-3838."""
        return _multiclass_frames(self, ex)


def _multiclass_frames(predictor, ex):
    """Shared by the two identity predictors (:3781-3838, :4506-4566): instance j of a frame belongs to class j and gets
    the ``Track`` named after it; ``score`` = mean point confidence, ``tracking_score`` = mean class probability."""
    from sleap_b200.nn.tracking import Track
    tracks = predictor.tracks
    if tracks is None:
        tracks = predictor.tracks = [Track(spawned_on=0, name=n) for n in predictor.classes]
    out = []
    for i in range(len(ex["instance_peaks"])):
        insts = []
        for j in range(ex["instance_peaks"].shape[1]):
            pts, confs = ex["instance_peaks"][i, j], ex["instance_peak_vals"][i, j]
            if np.all(np.isnan(pts)):
                continue
            insts.append(PredictedInstance.from_numpy(pts, confs, float(np.nanmean(confs)), track=tracks[j] if j < len(tracks) else None,
                                                      tracking_score=float(np.nanmean(ex["instance_scores"][i, j]))))
        out.append(LabeledFrame(int(ex["video_ind"][i]), int(ex["frame_ind"][i]), insts))
    return out


class TopDownMultiClassPredictor(Predictor):
    """sleap/nn/inference.py:4213-4605: top-down identity models -- a centroid model (or ground-truth centroids from a
    labels provider) and a centered-instance model with a class-vector head; one instance per class and frame."""

    def __init__(self, centroid_model=None, confmap_model=None, crop_size=160, peak_threshold=0.2, integral_refinement=True,
                 integral_patch_size=5, batch_size=4, max_instances=None, max_peaks_per_sample=256, tracks=None):
        super().__init__(batch_size)
        if confmap_model is None:
            raise ValueError("The topdown multi-class confidence map model must be provided.")
        self.centroid_model, self.confmap_model = centroid_model, confmap_model
        self.classes = list(confmap_model.spec["classes"])
        self.anchor_part = None
        self.crop_size = crop_size
        self.peak_threshold = peak_threshold
        self.integral_refinement = integral_refinement
        self.integral_patch_size = integral_patch_size
        self.max_instances = max_instances
        self.max_peaks_per_sample = max_peaks_per_sample
        self.tracks = tracks
        self._initialize_inference_model()

    def _initialize_inference_model(self):
        """:4263-4318."""
        ref = "integral" if self.integral_refinement else "local"
        cm, im = self.centroid_model, self.confmap_model
        iscale = float(getattr(im, "config_input_scale", im.input_scale))
        if im.input_scale != 1.0:
            raise ValueError("top-down instance models must be built without a resize op (resize_input_image=False)")
        if cm is None:
            cc = CentroidCropGroundTruth(crop_size=self.crop_size, handle=im.handle)
            cc.input_scale = iscale
        else:
            cc = CentroidCrop(keras_model=cm, crop_size=self.crop_size, input_scale=cm.input_scale, pad_to_stride=cm.cm.max_stride,
                              peak_threshold=self.peak_threshold, refinement=ref, integral_patch_size=self.integral_patch_size,
                              max_instances=self.max_instances, return_crops=True, max_peaks_per_sample=self.max_peaks_per_sample)
            cc.precrop_resize = iscale
        fp = TopDownMultiClassFindPeaks(keras_model=im, input_scale=iscale, peak_threshold=self.peak_threshold, refinement=ref,
                                        integral_patch_size=self.integral_patch_size)
        self.inference_model = TopDownMultiClassInferenceModel(cc, fp)

    @property
    def uses_ground_truth(self):
        return self.centroid_model is None

    @classmethod
    def from_trained_models(cls, centroid_model_path=None, confmap_model_path=None, batch_size=4, peak_threshold=0.2,
                            integral_refinement=True, integral_patch_size=5, resize_input_layer=True, max_instances=None,
                            precision=PRECISION_FP16, handle=None, max_peaks_per_sample=256, **_):
        """:4320-4401."""
        if confmap_model_path is None:
            raise ValueError("The topdown multi-class confidence map model must be provided.")
        cmodel, anchor = None, None
        if centroid_model_path is not None:
            ccfg, _, cmodel = cls._load(centroid_model_path, precision, handle)
            anchor = ccfg["data"]["instance_cropping"].get("center_on_part")
        icfg, _, imodel = cls._load(confmap_model_path, precision, handle, resize_in_graph=False)
        crop = icfg["data"]["instance_cropping"]["crop_size"]
        anchor = icfg["data"]["instance_cropping"].get("center_on_part") if anchor is None else anchor
        obj = cls(cmodel, imodel, crop, peak_threshold, integral_refinement, integral_patch_size, batch_size, max_instances,
                  max_peaks_per_sample)
        obj.anchor_part = anchor
        return obj

    def _frames_from_example(self, ex):
        """:4506-4566."""
        return _multiclass_frames(self, ex)


def load_model(model_path, batch_size=4, peak_threshold=0.2, refinement="integral", **kwargs):
    """sleap/nn/inference.py:4865-5005 (``sleap.load_model``)."""
    return Predictor.from_model_paths(model_path, peak_threshold=peak_threshold,
                                      integral_refinement=(refinement == "integral"), batch_size=batch_size, **kwargs)
