"""Grouping of peaks into identity classes (multi-class models): host-side logic, as in the reference, where these
functions run as TensorFlow ops around a SciPy ``numpy_function`` (sleap/nn/identity.py, sleap/nn/utils.py:79-98).

  class_probabilities          the class maps' sigmoid (float64, rounded once to float32)
  group_class_peaks            sleap/nn/identity.py:13-94
  classify_peaks_from_maps     sleap/nn/identity.py:97-179
  classify_peaks_from_vectors  sleap/nn/identity.py:182-254

Inputs / outputs are NumPy arrays with the reference's shapes and NaN conventions.
"""
from typing import Tuple

import numpy as np
from scipy.optimize import linear_sum_assignment


def class_probabilities(logits) -> np.ndarray:
    """The class maps' sigmoid (heads.py:336-338 of the reference applies it in the graph), evaluated in float64 and
    rounded once to float32: the one definition the device's multi-class step uses for the logits it samples."""
    with np.errstate(over="ignore"):         # exp(+large) = inf -> 1 / inf = 0: the limit the sigmoid has there
        return (1.0 / (1.0 + np.exp(-np.asarray(logits).astype(np.float64)))).astype(np.float32)


def group_class_peaks(peak_class_probs, peak_sample_inds, peak_channel_inds, n_samples: int,
                      n_channels: int) -> Tuple[np.ndarray, np.ndarray]:
    """Per (sample, channel): assign peaks to classes by the Hungarian algorithm on -probability, then keep only the
    matches whose class is the most probable one for that peak.  Returns ``(peak_inds, class_inds)`` (int32)."""
    probs = np.asarray(peak_class_probs, np.float32)
    if probs.ndim != 2:
        probs = probs.reshape(len(probs), -1) if probs.size else np.zeros((0, 0), np.float32)
    s_inds = np.asarray(peak_sample_inds).astype(np.int32).reshape(-1)
    c_inds = np.asarray(peak_channel_inds).astype(np.int32).reshape(-1)
    peak_inds, class_inds = [], []
    for sample in range(int(n_samples)):
        for channel in range(int(n_channels)):
            where = np.flatnonzero((s_inds == sample) & (c_inds == channel))
            if where.size == 0 or probs.shape[1] == 0:
                continue
            rows, cols = linear_sum_assignment(-probs[where])
            peak_inds.append(where[rows])
            class_inds.append(cols)
    if not peak_inds:
        return np.zeros((0,), np.int32), np.zeros((0,), np.int32)
    peak_inds = np.concatenate(peak_inds).astype(np.int32)
    class_inds = np.concatenate(class_inds).astype(np.int32)
    matched = probs[peak_inds, class_inds]
    best = probs[peak_inds].max(axis=1)
    keep = matched == best
    return peak_inds[keep], class_inds[keep]


def classify_peaks_from_maps(class_maps, peak_points, peak_vals, peak_sample_inds, peak_channel_inds,
                             n_channels: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Class probabilities are read off the class maps at the rounded peak locations (``tf.round`` = half to even,
    peak coordinates in class-map pixels).  Returns ``points (S, n_classes, n_channels, 2)``, ``point_vals`` and
    ``class_probs (S, n_classes, n_channels)``, NaN where nothing was assigned."""
    class_maps = np.asarray(class_maps, np.float32)
    n_samples, H, W, n_classes = class_maps.shape
    pts = np.asarray(peak_points, np.float32).reshape(-1, 2)
    vals = np.asarray(peak_vals, np.float32).reshape(-1)
    s_inds = np.asarray(peak_sample_inds).astype(np.int32).reshape(-1)
    c_inds = np.asarray(peak_channel_inds).astype(np.int32).reshape(-1)
    xy = np.rint(pts).astype(np.int64)                      # np.rint rounds half to even, like tf.round
    rows, cols = xy[:, 1], xy[:, 0]
    inside = (rows >= 0) & (rows < H) & (cols >= 0) & (cols < W)     # gather_nd out of range = 0 (TF-GPU semantics)
    probs = np.zeros((len(pts), n_classes), np.float32)
    probs[inside] = class_maps[s_inds[inside], rows[inside], cols[inside]]
    peak_inds, class_inds = group_class_peaks(probs, s_inds, c_inds, n_samples, n_channels)
    points = np.full((n_samples, n_classes, int(n_channels), 2), np.nan, np.float32)
    point_vals = np.full((n_samples, n_classes, int(n_channels)), np.nan, np.float32)
    class_probs = np.full((n_samples, n_classes, int(n_channels)), np.nan, np.float32)
    sub = (s_inds[peak_inds], class_inds, c_inds[peak_inds])
    points[sub] = pts[peak_inds]
    point_vals[sub] = vals[peak_inds]
    class_probs[sub] = probs[peak_inds, class_inds]
    return points, point_vals, class_probs


def classify_peaks_from_vectors(peak_points, peak_vals, peak_class_probs, crop_sample_inds,
                                n_samples: int) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """Top-down variant: one class-probability vector per crop.  ``peak_points (n_crops, n_channels, 2)``; returns
    ``points (S, n_classes, n_channels, 2)``, ``point_vals (S, n_classes, n_channels)``, ``class_probs (S, n_classes)``."""
    pts = np.asarray(peak_points, np.float32)
    vals = np.asarray(peak_vals, np.float32)
    probs = np.asarray(peak_class_probs, np.float32)
    s_inds = np.asarray(crop_sample_inds).astype(np.int32).reshape(-1)
    n_channels, n_classes = pts.shape[1], probs.shape[1]
    peak_inds, class_inds = group_class_peaks(probs, s_inds, np.zeros_like(s_inds), n_samples, 1)
    points = np.full((int(n_samples), n_classes, n_channels, 2), np.nan, np.float32)
    point_vals = np.full((int(n_samples), n_classes, n_channels), np.nan, np.float32)
    class_probs = np.full((int(n_samples), n_classes), np.nan, np.float32)
    sub = (s_inds[peak_inds], class_inds)
    points[sub] = pts[peak_inds]
    point_vals[sub] = vals[peak_inds]
    class_probs[sub] = probs[peak_inds, class_inds]
    return points, point_vals, class_probs
