"""compute-sanitizer target for the streamed (submit / collect) steps: short predict_batches streams of small synthetic
networks -- single-instance (sb_global_submit / _collect), bottom-up (sb_bottomup_*) plain and with an attached device
tracker, bottom-up identity (sb_multiclass_*), top-down (sb_topdown_submit / _collect) plain, with an attached device
tracker and with several instance chunks per batch, top-down identity (sb_topdown_multiclass_*, class vectors
returned), ground-truth top-down (sb_topdown_gt_submit) plain and identity, and a centroid model with ground-truth
instances (sb_topdown_gt_instances_*) -- each checked against the per-batch route, so that the copy stream, the
deferred instance stage and the per-slot staging run under memcheck / racecheck in minutes.
Usage: compute-sanitizer --tool memcheck python tools/sanitize_stream.py"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sleap_b200.nn import architectures as A
from sleap_b200.nn import tracking as T
from sleap_b200.nn.inference import (BottomUpMultiClassPredictor, BottomUpPredictor, SingleInstancePredictor,
                                     TopDownMultiClassPredictor, TopDownPredictor)
from sleap_b200.nn.model import DeviceModel

NODES = list("abcd")
EDGES = [("a", "b"), ("b", "c"), ("c", "d")]
B = 2


def unet(output_stride, up_interpolate=True):
    return dict(filters=8, filters_rate=2, max_stride=16, output_stride=output_stride, middle_block=True, up_interpolate=up_interpolate)


def same(im, frames, tracker=None, holder=None):
    """predict_batches against the per-batch route; `tracker`: kwargs of a device tracker, a fresh one for each route, set
    on `holder` (default: im)."""
    def fresh():
        if tracker:
            (holder or im).tracker = T.Tracker.make_tracker_by_name(track_device=0, **tracker)

    fresh()
    streamed = list(im.predict_batches(frames, B))
    fresh()
    per_batch = [im.predict_on_batch(frames[i:i + B]) for i in range(0, len(frames), B)]
    assert len(streamed) == len(per_batch)
    for a, b in zip(streamed, per_batch):
        assert sorted(a) == sorted(b) and all(np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes() for k in a)
    return sum(len(x["instance_peaks"]) for x in streamed)


def same_ground_truth(im, frames, seed, nodes=0):
    """predict_examples (sb_topdown_gt_submit / collect) against predict_on_batch on labels of 0-3 random centroids; with
    `nodes`, (sb_topdown_gt_instances_submit / _collect) on labels of 0-3 random instances of that many nodes, some NaN."""
    rng = np.random.default_rng(seed)
    rows = [rng.uniform(0, [frames.shape[2], frames.shape[1]], (int(rng.integers(0, 4)),) + ((nodes, 2) if nodes else (2,)))
            .astype(np.float32) for _ in frames]
    for r in rows if nodes else ():
        r[rng.random(r.shape[:2]) < 0.3] = np.nan
    key = "instances" if nodes else "centroids"
    examples = [{"image": frames[i:i + B], key: rows[i:i + B]} for i in range(0, len(frames), B)]
    n = 0
    for ex, a in list(im.predict_examples(iter(examples), B, 3)):      # streamed first: predict_on_batch uses slot 0
        b = im.predict_on_batch(ex)
        assert sorted(a) == sorted(b) and all(np.asarray(a[k]).tobytes() == np.asarray(b[k]).tobytes() for k in a)
        n += len(a["instance_peaks"])
    return n


def centroid_model(frames):
    spec = dict(backbone="unet", backbone_cfg=unet(2), head_type="centroid", part_names=None, edges=None,
                heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
    m = DeviceModel(spec, A.make_synthetic_weights(A.compile_model(spec, 1), 61), input_channels=1, precision=0)
    return m, max(float(np.quantile(m.forward(frames[:B])[0], 0.99)), 1e-3)


def main():
    frames = np.random.default_rng(9).integers(0, 256, size=(5, 192, 224, 1), dtype=np.uint8)
    frames[2] = 0                                                        # a frame without a centroid
    sspec = dict(backbone="unet", backbone_cfg=unet(2), head_type="single_instance", part_names=NODES, edges=None,
                 heads=[dict(name="SingleInstanceConfmapsHead", channels=len(NODES), output_stride=2)])
    sm = DeviceModel(sspec, A.make_synthetic_weights(A.compile_model(sspec, 1), 59), input_channels=1, precision=0)
    print("single-instance", same(SingleInstancePredictor(sm, batch_size=B).inference_model, frames), flush=True)

    bspec = dict(backbone="unet", backbone_cfg=unet(2), head_type="multi_instance", part_names=NODES, edges=EDGES,
                 heads=[dict(name="MultiInstanceConfmapsHead", channels=len(NODES), output_stride=2),
                        dict(name="PartAffinityFieldsHead", channels=2 * len(EDGES), output_stride=4)])
    bm = DeviceModel(bspec, A.make_synthetic_weights(A.compile_model(bspec, 1), 69), input_channels=1, precision=0)
    thr = max(float(np.quantile(bm.forward(frames[:B])[0], 0.99)), 1e-3)
    bu = BottomUpPredictor(bm, NODES, EDGES, peak_threshold=thr, batch_size=B, max_instances_per_frame=8).inference_model
    print("bottom-up", same(bu, frames), flush=True)
    simple = dict(tracker="simple", similarity="instance", match="greedy")
    print("bottom-up, device tracker", same(bu, frames, simple, bu.bottomup_layer), flush=True)
    bu.bottomup_layer.detach_tracker()
    bu.bottomup_layer.tracker = None

    cspec = dict(backbone="unet", backbone_cfg=unet(2), head_type="multi_class_bottomup", part_names=NODES, edges=None,
                 classes=["c0", "c1", "c2"],
                 heads=[dict(name="MultiInstanceConfmapsHead", channels=len(NODES), output_stride=2),
                        dict(name="ClassMapsHead", channels=3, output_stride=2, activation="sigmoid")])
    cmod = DeviceModel(cspec, A.make_synthetic_weights(A.compile_model(cspec, 1), 71), input_channels=1, precision=0)
    thr = max(float(np.quantile(cmod.forward(frames[:B], ["MultiInstanceConfmapsHead"])[0], 0.99)), 1e-3)
    bmc = BottomUpMultiClassPredictor(cmod, cspec["classes"], peak_threshold=thr, batch_size=B).inference_model
    print("bottom-up identity", same(bmc, frames), flush=True)

    ispec = dict(backbone="unet", backbone_cfg=unet(4, False), head_type="centered_instance", part_names=NODES, edges=None,
                 heads=[dict(name="CenteredInstanceConfmapsHead", channels=len(NODES), output_stride=4)])
    im_model = DeviceModel(ispec, A.make_synthetic_weights(A.compile_model(ispec, 1), 63), input_channels=1, precision=0)
    cm, thr = centroid_model(frames)
    pred = TopDownPredictor(cm, im_model, crop_size=64, peak_threshold=thr, batch_size=B, max_instances=4)
    im = pred.inference_model
    im.instance_peaks.peak_threshold = 0.0
    print("top-down", same(im, frames), flush=True)
    im.instance_peaks.max_crops_per_call = 3
    print("top-down, 3 crops per chunk", same(im, frames), flush=True)
    print("top-down, device tracker", same(im, frames, simple), flush=True)
    im.detach_tracker()
    im.tracker = None
    gt = TopDownPredictor(None, im_model, crop_size=64, peak_threshold=0.0, batch_size=B).inference_model
    print("ground-truth top-down", same_ground_truth(gt, frames, 73), flush=True)
    gti = TopDownPredictor(cm, None, peak_threshold=thr, batch_size=B, max_instances=4).inference_model
    print("ground-truth instances top-down", same_ground_truth(gti, frames, 77, len(NODES)), flush=True)

    classes = ["c0", "c1", "c2"]
    mspec = dict(ispec, head_type="multi_class_topdown", classes=classes,
                 heads=ispec["heads"] + [dict(name="ClassVectorsHead", channels=len(classes), output_stride=16, vector=True,
                                              num_fc_layers=1, num_fc_units=16, global_pool=True)])
    icm = A.compile_model(mspec, 1)
    iw = A.make_synthetic_weights(icm, 65)
    rng = np.random.default_rng(67)
    dims = [icm.vector_taps["ClassVectorsHead"]["C"], 16, len(classes)]
    for i, name in enumerate(["pre_classification0_fc", "ClassVectorsHead"]):
        iw[name] = dict(kernel=(rng.normal(0, 1, dims[i:i + 2]) * np.sqrt(2.0 / dims[i])).astype(np.float32),
                        bias=rng.normal(0, 0.1, dims[i + 1]).astype(np.float32))
    cm, thr = centroid_model(frames)
    pred = TopDownMultiClassPredictor(cm, DeviceModel(mspec, iw, input_channels=1, precision=0), crop_size=64, peak_threshold=thr,
                                      batch_size=B, max_instances=4)
    im = pred.inference_model
    im.instance_peaks.peak_threshold = 0.0
    im.instance_peaks.max_crops_per_call = 3
    im.instance_peaks.return_class_vectors = True
    print("top-down identity", same(im, frames), flush=True)
    gt = TopDownMultiClassPredictor(None, pred.inference_model.instance_peaks.keras_model, crop_size=64, batch_size=B).inference_model
    print("ground-truth top-down identity", same_ground_truth(gt, frames, 75), flush=True)
    print("ok")


if __name__ == "__main__":
    main()
