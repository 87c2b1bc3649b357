"""Secondary configurations of BASELINE.json (C1, C2, C3, C5) through the public predictors, one
JSON line each (frames/s end to end with host frames, CUDA-event timed device loop where available).
Secondary to bench.py (C4).

  python tools/bench_configs.py [c1] [c2] [c3 | topdown] [c5] [r50] [track] [multiclass] [topdown_multiclass] [topdown_scaled]
                               [topdown_gt] [topdown_track] [pipeline] [--steps K]
                               [--c5-batch B]
  (C5 default: 16 frames per GPU and step)

r50: ResNet50 bottom-up (ImageNet-preprocessed "frozen" weights, upsampling stack to stride 4 with k4 transposed convs,
BN, two refine convs, concat skips), 1024x1024x1, flies13, B=8 per GPU; it also reports the fp16 maps against the fp32
path as a fraction of the map maximum.

track: the flow trackers with the cv2 flow shift and with the device flow shift (one JSON line).  Tracker only: the
first 500 frames of the tracking clip (tests/golden/tracks, 1024x1024, two flies x two nodes, window 5) for flow, flow
with save_shifted_instances and flowmaxtracks (max_tracks 2).  End to end: BottomUpPredictor.predict (labels made) of
the C4 network on 256 clip frames with no tracker, the cv2 flow tracker and the device flow tracker; the heads are
calibrated as bench.py does (~5 detections per channel), so the tracker shifts ~65 points per reference frame.
The device tracker (track_device=0) against the host tracker: tracker only (run_tracker, 256 frames per kernel call)
for simple / instance / greedy and simplemaxtracks / centroid / hungarian on the clip predictions (300 frames) and on a
seeded synthetic set of up to 6 instances x 13 nodes (300 frames); end to end, the same predict with no tracker, the
host simple tracker and the device simple tracker (k_track inside the step).

multiclass: the bottom-up multi-class (identity) predictor, three arms on the same frames, alternating in one process:
the host chain composed from public calls (forward -> identity.class_probabilities -> find_local_peaks ->
classify_peaks_from_maps), the fused step (predict_on_batch) and the pipelined submit/collect loop (predict).  Workloads:
the trained fixture model (min_tracks_2node, 1024x1024 at input scale 0.5, 2 nodes, 2 classes) on 256 clip frames, and a
C4-sized UNet with 13 nodes and 4 classes at stride 4 (synthetic weights, confidence head calibrated to ~5 detections
per node as bench.py does), 1024x1024, B=8.  The line reports frames/s per arm and whether the arms agree (assignments
identical, points, values and class probabilities bit for bit).

topdown_multiclass: the top-down multi-class (identity) predictor, two arms alternating on the same frames in one process:
the staged path (TopDownMultiClassInferenceModel with fused = False: centroid stage, crops to the host, instance network
with the class-vector head's dense layers and the grouping on the host) and the fused step (sb_infer_topdown_multiclass),
both through predict_on_batch.  Workload: the C3 pair (centroid UNet at input scale 0.5, centered-instance UNet on 160x160
crops, max 5 animals, B=16) with a ClassVectorsHead of 4 classes and 3 x 64 fc units on the stride-16 features.  The line
reports frames/s per arm and whether they agree (centroids and points bit for bit, identical assignments, the largest
class-probability difference).

topdown_scaled: the C3 pair with the centered-instance UNet trained at input scale 0.5 (96x96 crops of the frame resized
to 512x512 before cropping), three arms alternating in one process on the same 128 pinned frames, B=16: the staged route
(fused = False: centroids to the host, the frames resized by FrameResizer, crops through host memory), the fused step
(predict_on_batch: resize and crop inside the step) and the double-buffered loop (predict_batches).  The line reports
frames/s per arm (median and range over the repetitions) and whether all arms agree bit for bit.

topdown_gt: a top-down predictor with ground-truth centroids (no centroid model: CentroidCropGroundTruth) on synthetic
labels of 128 frames of 1024x1024 uint8, 5 instances of 13 nodes each, B=16; the instance UNet of the C3 pair at input
scale 1 (160x160 crops) and at 0.5 (96x96 crops of the half-size frame).  Three arms alternate in one process on the same
decoded label batches: the staged route (fused = False: FrameResizer, crops through host memory, one synchronous
sb_infer_global per chunk), the fused step per batch (predict_on_batch: sb_topdown_gt_submit + collect) and the
double-buffered loop predict runs on labels (predict_examples).  The line reports the card and its power limit, frames/s
per arm (median and range over the repetitions) and whether all arms agree bit for bit.

topdown_gt_instances: a top-down predictor built from the C3 centroid UNet (input scale 0.5) alone, ground-truth
instances standing in for the instance model (FindInstancePeaksGroundTruth), on labels of 128 gray tracking-clip frames
with 5 synthetic instances of 13 nodes each (some nodes invisible), B=16, the centroid threshold calibrated to about 5
animals per frame.  Three arms alternate in one process on the same decoded label batches: the host route (fused = False:
the centroid list to the host, the match in numpy), the fused step per batch (predict_on_batch:
sb_topdown_gt_instances_submit + collect) and the double-buffered loop predict runs on labels (predict_examples).  The
line reports the card and its power limit, frames/s per arm (median and range over the repetitions) and whether all arms
agree bit for bit.

topdown_track: the top-down predictor with a tracker, four arms alternating in one process: TopDownPredictor.predict
(labels made) of the C3 pair on 256 gray tracking-clip frames, B=16, the centroid threshold calibrated on clip frames to
about 5 animals per frame; no tracker, the host simple tracker, the device simple tracker inside the fused step
(sb_topdown_attach_tracker) and the device simple tracker on the per-frame route (fused = False).  The line reports
frames/s and instances per frame per arm, and whether the device tracks equal the host's, with numpy's greedy ties and
with the device's stable ones.

pipeline: the per-batch loop (predict_on_batch) against the double-buffered loop (predict_batches: submit / collect) of
the same inference model, alternating in one process on the same 128 pinned gray tracking-clip frames (1024x1024), B=16,
outputs compared batch by batch, bit for bit.  Workloads: a single-instance UNet as single() builds it (13 nodes); the C3
top-down pair of topdown_track (about 5 animals per frame) without a tracker and with the device simple tracker; the C3
identity pair of topdown_multiclass.  The line reports per workload the median frames/s of each loop over the
repetitions, their spread, and the agreement.
"""
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sleap_b200.nn import architectures as A
from sleap_b200.nn.inference import (BottomUpPredictor, SingleInstancePredictor, TopDownPredictor)
from sleap_b200.nn.model import DeviceModel

FLIES13 = ["head", "thorax", "abdomen", "wingL", "wingR", "forelegL", "forelegR", "midlegL", "midlegR", "hindlegL",
           "hindlegR", "eyeL", "eyeR"]


def frames(n, h, w, c, seed):
    """Page-locked frame stack (what FrameFeeder hands the predictors): the upload is a true asynchronous DMA."""
    import torch
    a = np.random.default_rng(seed).integers(0, 256, size=(n, h, w, c), dtype=np.uint8)
    return torch.from_numpy(a).pin_memory().numpy()


def model_for(spec, in_ch, seed, input_scale=1.0):
    cm = A.compile_model(spec, in_ch, input_scale)
    w = A.make_synthetic_weights(cm, seed)
    return DeviceModel(spec, w, input_channels=in_ch, input_scale=input_scale, precision=0), cm, w


def timed(fn, steps, warmup=3):
    """Seconds per call (wall clock, the call returns host results) + nvidia-smi clock samples taken meanwhile."""
    global LAST_CLOCKS
    import bench
    for _ in range(warmup):
        fn()
    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.25)
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    dt = (time.perf_counter() - t0) / steps
    LAST_CLOCKS = sampler.stop()
    return dt


LAST_CLOCKS = None


def roofline(gflop_per_frame, fps):
    """Tensor roofline of a whole config: algorithmic conv FLOPs per second / measured cuBLAS bf16 burst peak."""
    import bench
    peaks, src = bench.peaks_file()
    tf = gflop_per_frame * fps / 1e3
    return {"bound": "tensor", "achieved": tf, "peak": float(peaks["bf16_tflops"]), "unit": "TFLOP/s",
            "frac": tf / float(peaks["bf16_tflops"]), "peak_source": f"{src} bf16_tflops", "note": "end-to-end time incl. H2D / post-processing / D2H"}


def unet(filters, max_stride, output_stride):
    return dict(filters=filters, filters_rate=2, max_stride=max_stride, output_stride=output_stride, middle_block=True,
                up_interpolate=True, stacks=1)


def single(name, size, nodes, B, steps):
    spec = dict(backbone="unet", backbone_cfg=unet(16, 16, 2), head_type="single_instance", part_names=nodes, edges=None,
                heads=[dict(name="SingleInstanceConfmapsHead", channels=len(nodes), output_stride=2)])
    m, cm, _ = model_for(spec, 1, 1001)
    pred = SingleInstancePredictor(m, peak_threshold=0.2, integral_refinement=True, batch_size=B)
    fr = frames(B, size, size, 1, 1)
    dt = timed(lambda: pred.inference_model.predict_on_batch(fr), steps)
    return {"config": name, "metric": "frames/s (predict_on_batch, host frames)", "value": B / dt, "ms_per_step": dt * 1e3,
            "batch": B, "gflop_per_frame": cm.flops_per_pixel * size * size / 1e9, "dtype": "f16", "clocks": LAST_CLOCKS,
            "roofline": roofline(cm.flops_per_pixel * size * size / 1e9, B / dt)}


def topdown(steps):
    cspec = dict(backbone="unet", backbone_cfg=unet(16, 16, 2), head_type="centroid", part_names=None, edges=None,
                 heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
    ispec = dict(backbone="unet", backbone_cfg=dict(unet(24, 16, 4), up_interpolate=False), head_type="centered_instance",
                 part_names=FLIES13, edges=None, heads=[dict(name="CenteredInstanceConfmapsHead", channels=13, output_stride=4)])
    cm_model, ccm, cw = model_for(cspec, 1, 1003, input_scale=0.5)
    B = 16
    fr = frames(B, 1024, 1024, 1, 3)
    # calibrate the centroid head so that ~5 animals per frame pass the threshold (random weights otherwise give thousands)
    cms = cm_model.forward(fr[:2])[0]
    thr = float(np.sort(cms.reshape(-1))[-(5 * 2 * 6)])
    im_model, icm, _ = model_for(ispec, 1, 1004)
    pred = TopDownPredictor(cm_model, im_model, crop_size=160, peak_threshold=thr, integral_refinement=True, batch_size=B,
                            max_instances=5)
    pred.inference_model.instance_peaks.peak_threshold = 0.0
    out = pred.inference_model.predict_on_batch(fr)
    dt = timed(lambda: pred.inference_model.predict_on_batch(fr), steps)
    return {"config": "C3 top-down centroid(512^2 after 0.5 scale)+centered-instance(160^2 crops), 1024x1024, max 5 animals, B=16",
            "metric": "frames/s (predict_on_batch, host frames)", "value": B / dt, "ms_per_step": dt * 1e3, "batch": B,
            "mean_instances_per_frame": float(np.mean(out.get("n_valid", [0]))), "dtype": "f16", "clocks": LAST_CLOCKS,
            "gflop_per_frame": ccm.flops_per_pixel * 512 * 512 / 1e9 + 5 * icm.flops_per_pixel * 160 * 160 / 1e9,
            "roofline": roofline(ccm.flops_per_pixel * 512 * 512 / 1e9 + 5 * icm.flops_per_pixel * 160 * 160 / 1e9, B / dt)}


def hourglass(steps, B=16):
    nodes = [f"n{i}" for i in range(24)]
    edges = [(f"n{i}", f"n{i + 1}") for i in range(23)]
    spec = dict(backbone="hourglass", backbone_cfg=dict(stem_stride=4, max_stride=64, output_stride=4, stem_filters=128,
                                                         filters=256, filter_increase=128, stacks=3),
                head_type="multi_instance", part_names=nodes, edges=edges,
                heads=[dict(name="MultiInstanceConfmapsHead", channels=24, output_stride=4),
                       dict(name="PartAffinityFieldsHead", channels=46, output_stride=4)])
    m, cm, w = model_for(spec, 3, 1005)
    fr = frames(B, 1536, 1536, 3, 5)
    cms, pafs = m.forward(fr[:1])
    thr = float(np.quantile(cms, 1 - 5.0 / (384 * 384)))   # ~5 peaks per channel
    pred = BottomUpPredictor(m, nodes, edges, peak_threshold=thr, batch_size=B, max_peaks_per_sample=4096,
                             max_node_peaks=64, max_instances_per_frame=64)
    out = pred.inference_model.predict_on_batch(fr)
    dt = timed(lambda: pred.inference_model.predict_on_batch(fr), steps, warmup=2)
    gf = cm.flops_per_pixel * 1536 * 1536 / 1e9
    return {"config": f"C5 stacked hourglass x3 bottom-up 1536x1536x3, 24 nodes / 23 edges, B={B} per GPU and step",
            "metric": "frames/s (predict_on_batch, host frames)", "value": B / dt, "ms_per_step": dt * 1e3, "batch": B,
            "gflop_per_frame": gf, "tflops": gf * B / dt / 1e3, "flags": [int(f) for f in out.get("flags", [])], "dtype": "f16",
            "clocks": LAST_CLOCKS, "roofline": roofline(gf, B / dt)}


def gpu_identity():
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip()


def resnet50(steps, B=8):
    edges = [("head", "thorax"), ("thorax", "abdomen"), ("thorax", "wingL"), ("thorax", "wingR"), ("thorax", "forelegL"),
             ("thorax", "forelegR"), ("thorax", "midlegL"), ("thorax", "midlegR"), ("thorax", "hindlegL"), ("thorax", "hindlegR"),
             ("head", "eyeL"), ("head", "eyeR")]
    up = dict(method="transposed_conv", skip_connections="concatenate", block_stride=2, filters=64, filters_rate=1, refine_convs=2,
              batch_norm=True, transposed_conv_kernel_size=4)
    spec = dict(backbone="resnet", backbone_cfg=dict(version="ResNet50", weights="frozen", max_stride=32, output_stride=4, upsampling=up),
                head_type="multi_instance", part_names=FLIES13, edges=edges,
                heads=[dict(name="MultiInstanceConfmapsHead", channels=13, output_stride=4),
                       dict(name="PartAffinityFieldsHead", channels=24, output_stride=8)])
    cm = A.compile_model(spec, 1)
    w = A.make_synthetic_weights(cm, 1006)
    for L in cm.layers:        # keep 16 residual blocks of He-normal weights in a sane range
        if L["name"].endswith("_3_bn"):
            w[L["name"]]["gamma"] = np.full(L["c"], 0.3, np.float32)
    m = DeviceModel(spec, w, input_channels=1, precision=0)
    fr = frames(B, 1024, 1024, 1, 7)
    cms, pafs = m.forward(fr[:2])
    ref = DeviceModel(spec, w, input_channels=1, precision=1).forward(fr[:2])
    err = [float(np.abs(a - b).max() / np.abs(b).max()) for a, b in zip((cms, pafs), ref)]
    thr = float(np.quantile(cms, 1 - 5.0 / (256 * 256)))
    pred = BottomUpPredictor(m, FLIES13, edges, peak_threshold=thr, batch_size=B, max_peaks_per_sample=4096,
                             max_node_peaks=64, max_instances_per_frame=64)
    pred.inference_model.predict_on_batch(fr)
    dt = timed(lambda: pred.inference_model.predict_on_batch(fr), steps, warmup=2)
    gf = cm.flops_per_pixel * 1024 * 1024 / 1e9
    tf = gf * B / dt / 1e3
    return {"config": f"R50 ResNet50 bottom-up 1024x1024x1, flies13, upsampling to stride 4 (k4 tconv + BN + 2 refine, concat skips), B={B}",
            "metric": "frames/s (predict_on_batch, host frames)", "value": B / dt, "ms_per_step": dt * 1e3, "batch": B,
            "gflop_per_frame": gf, "tflops": tf, "frac_of_989_dense_fp16_tflops": tf / 989.0, "gpu": gpu_identity(),
            "fp16_vs_fp32_maps_max_err_frac": err, "dtype": "f16", "clocks": LAST_CLOCKS}


def track_bench():
    import cv2
    import torch
    import bench
    from sleap_b200.nn import tracking as T
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from flow_clip import clip_frames, clip_labeled_frames
    n_track, n_e2e = 500, 256
    clip = clip_frames(n_track)
    out = {"config": "track: flow trackers, cv2 vs device flow shift, 1024x1024 clip", "gpu": gpu_identity(),
           "cv2_threads": cv2.getNumThreads(), "cpu_count": os.cpu_count(), "tracker_only_frames_per_s": {}}

    def make(tracker, save, of_device):
        tr = T.Tracker.make_tracker_by_name(tracker=tracker, similarity="instance", match="greedy", track_window=5, max_tracks=2,
                                            max_tracking=tracker == "flowmaxtracks", save_shifted_instances=save, of_device=of_device)
        if of_device is not None:
            tr.candidate_maker.device_flow()             # handle creation is set-up, not tracking
        return tr

    variants = [("flow", False), ("flow", True), ("flowmaxtracks", False)]
    for tracker, save in variants:
        for dev in (None, 0):
            T.run_tracker(clip_labeled_frames(20), make(tracker, save, dev), images=lambda t: clip[t])    # warm-up
            tr, frames = make(tracker, save, dev), clip_labeled_frames(n_track)
            t0 = time.perf_counter()
            T.run_tracker(frames, tr, images=lambda t: clip[t])
            fps = n_track / (time.perf_counter() - t0)
            out["tracker_only_frames_per_s"][f"{tracker}{'+save' if save else ''} {'device' if dev is not None else 'cv2'}"] = fps

    # end to end: C4 network (bench.py) + post-processing + labels + tracker on the consumer thread
    spec = bench.c4_spec()
    cm = A.compile_model(spec, 1)
    w = A.make_synthetic_weights(cm, bench.SEED)
    gray = np.ascontiguousarray(clip[:n_e2e, :, :, :1])
    m0 = DeviceModel(spec, w, input_channels=1, precision=0)
    cms0, pafs0 = m0.forward(gray[:2])
    w = bench.calibrate_heads(w, cms0, pafs0, 2)
    del m0
    model = DeviceModel(spec, w, input_channels=1, precision=0)
    frames_e2e = torch.from_numpy(gray).pin_memory().numpy()
    e2e = {}
    for name, tracker, dev in (("no tracker", None, None), ("flow cv2", "flow", None), ("flow device", "flow", 0)):
        pred = BottomUpPredictor(model, bench.NODES, bench.EDGES, peak_threshold=0.2, batch_size=8, integral_refinement=True,
                                 max_peaks_per_sample=1024, max_node_peaks=32, max_instances_per_frame=32)
        pred.tracker = make(tracker, False, dev) if tracker else None
        pred.predict(frames_e2e[:32])                                    # warm-up
        pred.tracker = make(tracker, False, dev) if tracker else None
        t0 = time.perf_counter()
        labeled = pred.predict(frames_e2e)
        e2e[name] = n_e2e / (time.perf_counter() - t0)
        e2e[f"{name} instances/frame"] = float(np.mean([len(lf.instances) for lf in labeled]))
    out["predict_c4_frames_per_s"] = e2e

    # device tracker vs host tracker
    from track_cases import synthetic_frames
    sets = {"clip": lambda: clip_labeled_frames(300), "synthetic 6x13": lambda: synthetic_frames(7, 300, 6, 13, all_nan=0.0)}
    configs = {"simple/instance/greedy": dict(tracker="simple", similarity="instance", match="greedy"),
               "simplemaxtracks/centroid/hungarian": dict(tracker="simplemaxtracks", similarity="centroid", match="hungarian",
                                                          max_tracks=6, max_tracking=True)}
    only = {}
    for sname, make_set in sets.items():
        for cname, kw in configs.items():
            for where in ("host", "device"):
                dev = 0 if where == "device" else None
                T.run_tracker(make_set()[:20], T.Tracker.make_tracker_by_name(track_device=dev, **kw))     # warm-up
                frames = make_set()
                tr = T.Tracker.make_tracker_by_name(track_device=dev, **kw)
                t0 = time.perf_counter()
                T.run_tracker(frames, tr)
                only[f"{sname} {cname} {where}"] = len(frames) / (time.perf_counter() - t0)
    out["device_tracker_only_frames_per_s"] = only
    e2e = {}
    for name, dev in (("no tracker", None), ("simple host", None), ("simple device", 0)):
        pred = BottomUpPredictor(model, bench.NODES, bench.EDGES, peak_threshold=0.2, batch_size=8, integral_refinement=True,
                                 max_peaks_per_sample=1024, max_node_peaks=32, max_instances_per_frame=32)
        mk = (lambda: None) if name == "no tracker" else \
            (lambda: T.Tracker.make_tracker_by_name(tracker="simple", similarity="instance", match="greedy", track_device=dev))
        pred.tracker = mk()
        pred.predict(frames_e2e[:32])                                    # warm-up
        pred.tracker = mk()
        t0 = time.perf_counter()
        labeled = pred.predict(frames_e2e)
        e2e[name] = n_e2e / (time.perf_counter() - t0)
        e2e[f"{name} tracks"] = len({id(i.track) for lf in labeled for i in lf.instances if i.track is not None})
    out["predict_c4_simple_tracker_frames_per_s"] = e2e
    return out


def _mc_host_arm(layer, batch):
    """The parent commit's host chain for one batch, from public calls."""
    from sleap_b200.nn import identity, peak_finding
    m = layer.keras_model
    names = [layer.CMS, layer.CLASS_MAPS] + ([layer.OFFSETS] if layer.has_offsets else [])
    outs = m.forward(batch, names)
    probs = identity.class_probabilities(outs[1])
    if layer.has_offsets:
        pk, pv, si, ci = peak_finding.find_local_peaks_with_offsets(outs[0], outs[2], threshold=layer.peak_threshold, handle=m.handle)
    else:
        pk, pv, si, ci = peak_finding.find_local_peaks(outs[0], threshold=layer.peak_threshold, refinement=layer.refinement,
                                                       integral_patch_size=layer.integral_patch_size, handle=m.handle)
    cs = np.float32(layer.class_maps_output_stride)
    pk = ((pk * np.float32(layer.cm_output_stride)).astype(np.float32) / cs).astype(np.float32)
    pts, vals, cp = identity.classify_peaks_from_maps(probs, pk, pv, si, ci, n_channels=outs[0].shape[3])
    pts = (pts * cs).astype(np.float32)
    if layer.input_scale != 1.0:
        pts = (pts / np.float32(layer.input_scale) + np.float32(0.5)).astype(np.float32)
    return {"instance_peaks": pts, "instance_peak_vals": vals, "instance_scores": cp}


def _mc_agree(a, b, keys=("instance_peaks", "instance_peak_vals", "instance_scores")):
    """Assignments identical (NaN pattern) and every value bit for bit."""
    for k in keys:
        x, y = np.asarray(a[k], np.float32), np.asarray(b[k], np.float32)
        if x.shape != y.shape or not np.array_equal(np.isnan(x), np.isnan(y)):
            return False
        if not np.array_equal(x[~np.isnan(x)].view(np.uint32), y[~np.isnan(y)].view(np.uint32)):
            return False
    return True


def _mc_workload(pred, fr, B, reps):
    layer = pred.inference_model.inference_layer
    im = pred.inference_model
    arms = {
        "host chain (forward, class_probabilities, find_local_peaks, classify_peaks_from_maps)":
            lambda: _merge([_mc_host_arm(layer, fr[i:i + B]) for i in range(0, len(fr), B)]),
        "fused predict_on_batch": lambda: _merge([im.predict_on_batch(fr[i:i + B]) for i in range(0, len(fr), B)]),
        "fused predict (pipelined submit/collect loop)": lambda: im.predict(fr, batch_size=B),
    }
    outs = {k: f() for k, f in arms.items()}                             # warm-up, and the outputs compared
    times = {k: [] for k in arms}
    for _ in range(reps):                                                # arms alternate
        for k, f in arms.items():
            t0 = time.perf_counter()
            f()
            times[k].append(time.perf_counter() - t0)
    names = list(arms)
    res = {"frames": len(fr), "batch": B, "frames_per_s": {k: len(fr) / float(np.median(v)) for k, v in times.items()},
           "frames_per_s_spread": {k: [len(fr) / max(v), len(fr) / min(v)] for k, v in times.items()},
           "agree_fused_vs_host": _mc_agree(outs[names[1]], outs[names[0]]),
           "agree_pipelined_vs_host": _mc_agree(outs[names[2]], outs[names[0]]),
           "assigned_points_per_frame": float(np.isfinite(outs[names[1]]["instance_scores"]).sum() / len(fr))}
    return res


def _merge(chunks):
    return {k: np.concatenate([c[k] for c in chunks]) for k in ("instance_peaks", "instance_peak_vals", "instance_scores")}


def multiclass_bench(steps):
    import torch
    import bench
    from sleap_b200.nn.inference import BottomUpMultiClassPredictor, Predictor
    tests = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests")
    sys.path.insert(0, tests)
    from flow_clip import clip_frames
    reps = max(3, steps // 2)
    out = {"config": "multiclass: bottom-up identity predictor, host chain vs fused step vs pipelined loop", "gpu": gpu_identity(),
           "metric": "frames/s (median of alternating repetitions; host frames in, results on the host)", "repetitions": reps}
    clip = torch.from_numpy(np.ascontiguousarray(clip_frames(256))).pin_memory().numpy()
    fx = os.path.join(tests, "golden", "models", "min_tracks_2node.bottomup_multiclass", "fixture_config.json")
    pred = Predictor.from_model_paths([fx], batch_size=8)
    out["fixture min_tracks_2node (1024x1024 at scale 0.5, 2 nodes, 2 classes, maps at stride 2), 256 clip frames"] = \
        _mc_workload(pred, clip, 8, reps)
    # C4-sized identity network: the C4 UNet, 13 confidence maps and 4 class maps at stride 4
    spec = dict(backbone="unet", backbone_cfg=dict(bench.UNET_CFG), head_type="multi_class_bottomup",
                heads=[dict(name="MultiInstanceConfmapsHead", channels=13, output_stride=4),
                       dict(name="ClassMapsHead", channels=4, output_stride=4, activation="sigmoid")],
                part_names=bench.NODES, edges=None, classes=["c0", "c1", "c2", "c3"])
    cm = A.compile_model(spec, 1)
    w = A.make_synthetic_weights(cm, bench.SEED)
    fr = frames(8, 1024, 1024, 1, 11)
    m0 = DeviceModel(spec, w, input_channels=1, precision=0)
    cms = m0.forward(fr[:2], ["MultiInstanceConfmapsHead"])[0]
    del m0
    k = np.asarray(w["MultiInstanceConfmapsHead"]["kernel"]).copy()
    b = np.asarray(w["MultiInstanceConfmapsHead"]["bias"]).copy()
    for c in range(cms.shape[-1]):                                       # bench.calibrate_heads on the confidence head
        vals = np.sort(np.concatenate([bench.local_max_values(cms[i, :, :, c]) for i in range(cms.shape[0])]))[::-1]
        kth = min(len(vals) - 1, bench.TARGET_PEAKS_PER_CHANNEL * cms.shape[0])
        t, top = float(vals[kth]), float(vals[0])
        g = 0.8 / max(top - t, 1e-6)
        k[..., c] *= g
        b[c] = (b[c] - t) * g + 0.2
    w["MultiInstanceConfmapsHead"] = dict(kernel=k, bias=b)
    model = DeviceModel(spec, w, input_channels=1, precision=0)
    pred = BottomUpMultiClassPredictor(model, spec["classes"], peak_threshold=0.2, batch_size=8)
    out["C4-sized UNet (13 nodes, 4 classes at stride 4, synthetic weights), 1024x1024, B=8"] = \
        _mc_workload(pred, np.concatenate([fr] * 4), 8, reps)
    return out


def topdown_multiclass_bench(steps):
    """The C3 pair of topdown() with the instance model given a ClassVectorsHead (4 classes, 3 x 64 fc units, global max
    pool of the stride-16 features): the staged TopDownMultiClassInferenceModel (fused = False) and the fused step, both
    through predict_on_batch, alternating on the same frames."""
    from sleap_b200.nn.inference import TopDownMultiClassPredictor
    classes = ["c0", "c1", "c2", "c3"]
    cspec = dict(backbone="unet", backbone_cfg=unet(16, 16, 2), head_type="centroid", part_names=None, edges=None,
                 heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
    ispec = dict(backbone="unet", backbone_cfg=dict(unet(24, 16, 4), up_interpolate=False), head_type="multi_class_topdown",
                 part_names=FLIES13, edges=None, classes=classes,
                 heads=[dict(name="CenteredInstanceConfmapsHead", channels=13, output_stride=4),
                        dict(name="ClassVectorsHead", channels=len(classes), output_stride=16, vector=True, num_fc_layers=3,
                             num_fc_units=64, global_pool=True)])
    B = 16
    fr = frames(B, 1024, 1024, 1, 3)
    icm = A.compile_model(ispec, 1)
    iw = A.make_synthetic_weights(icm, 1004)
    rng = np.random.default_rng(1005)
    dims = [icm.vector_taps["ClassVectorsHead"]["C"], 64, 64, 64, len(classes)]
    for i in range(4):                                                    # He-normal dense layers, small biases
        iw["ClassVectorsHead" if i == 3 else f"pre_classification{i}_fc"] = dict(
            kernel=(rng.normal(0, 1, dims[i:i + 2]) * np.sqrt(2.0 / dims[i])).astype(np.float32),
            bias=rng.normal(0, 0.1, dims[i + 1]).astype(np.float32))

    def arm(fused):
        # each arm owns its two device models: a staged call reconfigures the chains the fused pipeline needs
        cm_model, _, _ = model_for(cspec, 1, 1003, input_scale=0.5)
        cms = cm_model.forward(fr[:2])[0]                                # ~5 animals per frame, as topdown() calibrates
        thr = float(np.sort(cms.reshape(-1))[-(5 * 2 * 6)])
        pred = TopDownMultiClassPredictor(cm_model, DeviceModel(ispec, iw, input_channels=1, precision=0), crop_size=160,
                                          peak_threshold=thr, integral_refinement=True, batch_size=B, max_instances=5)
        pred.inference_model.instance_peaks.peak_threshold = 0.0
        pred.inference_model.fused = fused
        return lambda: pred.inference_model.predict_on_batch(fr)

    arms = {"staged predict_on_batch (fused = False)": arm(False), "fused predict_on_batch": arm(True)}
    outs = {k: f() for k, f in arms.items()}                             # warm-up, and the outputs compared
    reps = max(3, steps)
    times = {k: [] for k in arms}
    for _ in range(reps):                                                # arms alternate
        for k, f in arms.items():
            t0 = time.perf_counter()
            f()
            times[k].append(time.perf_counter() - t0)
    a, b = (outs[k] for k in arms)
    same_assignments = np.array_equal(np.isnan(a["instance_scores"]), np.isnan(b["instance_scores"]))
    return {"config": "topdown_multiclass: C3 top-down pair, instance model with a ClassVectorsHead (4 classes, 3 x 64 fc units, "
                      "stride-16 tap), 1024x1024, max 5 animals, B=16", "gpu": gpu_identity(),
            "metric": "frames/s (median of alternating repetitions; host frames in, results on the host)", "repetitions": reps,
            "frames_per_s": {k: B / float(np.median(v)) for k, v in times.items()},
            "frames_per_s_spread": {k: [B / max(v), B / min(v)] for k, v in times.items()},
            "mean_crops_per_frame": float(np.isfinite(b["centroid_vals"]).sum() / B),
            "agree_centroids_bitwise": _mc_agree(a, b, ("centroids", "centroid_vals")), "agree_assignments": bool(same_assignments),
            "agree_points_bitwise": _mc_agree(a, b, ("instance_peaks", "instance_peak_vals")),
            "class_probability_max_abs_diff": float(np.nanmax(np.abs(a["instance_scores"] - b["instance_scores"])))
            if np.isfinite(a["instance_scores"]).any() else 0.0}


def topdown_scaled_bench(steps):
    """The C3 pair of topdown() with the instance UNet trained at input scale 0.5 (96x96 crops of the half-size frame, as
    a model with input_scaling 0.5 loads): three arms alternating on the same 128 pinned frames, B = 16 -- the staged route
    (fused = False: centroids to the host, FrameResizer, crops through host memory), the fused step per batch
    (predict_on_batch) and the double-buffered loop (predict_batches)."""
    n, B = 128, 16
    fr = frames(n, 1024, 1024, 1, 3)
    cspec = dict(backbone="unet", backbone_cfg=unet(16, 16, 2), head_type="centroid", part_names=None, edges=None,
                 heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
    ispec = dict(backbone="unet", backbone_cfg=dict(unet(24, 16, 4), up_interpolate=False), head_type="centered_instance",
                 part_names=FLIES13, edges=None, heads=[dict(name="CenteredInstanceConfmapsHead", channels=13, output_stride=4)])

    def inference_model(fused):
        # the staged arm owns its two device models: its calls reconfigure the chains the fused pipeline needs
        cm_model, _, _ = model_for(cspec, 1, 1003, input_scale=0.5)
        cms = cm_model.forward(fr[:2])[0]                                # ~5 animals per frame, as topdown() calibrates
        thr = float(np.sort(cms.reshape(-1))[-(5 * 2 * 6)])
        im_model = model_for(ispec, 1, 1004)[0]
        im_model.config_input_scale = 0.5                                # what Predictor._load(..., resize_in_graph=False) sets
        pred = TopDownPredictor(cm_model, im_model, crop_size=96, peak_threshold=thr, integral_refinement=True, batch_size=B,
                                max_instances=5)
        pred.inference_model.instance_peaks.peak_threshold = 0.0
        pred.inference_model.fused = fused
        return pred.inference_model

    staged, fused = inference_model(False), inference_model(True)
    assert not staged._can_fuse() and fused._can_fuse()
    arms = {"staged predict_on_batch (fused = False)": lambda: [staged.predict_on_batch(fr[i:i + B]) for i in range(0, n, B)],
            "fused predict_on_batch": lambda: [fused.predict_on_batch(fr[i:i + B]) for i in range(0, n, B)],
            "streamed predict_batches": lambda: list(fused.predict_batches(fr, B))}
    outs = {k: f() for k, f in arms.items()}                             # warm-up, and the outputs compared
    reps = max(5, steps)
    times = {k: [] for k in arms}
    for _ in range(reps):                                                # arms alternate
        for k, f in arms.items():
            t0 = time.perf_counter()
            f()
            times[k].append(time.perf_counter() - t0)
    keys = ("n_valid", "centroids", "centroid_vals", "instance_peaks", "instance_peak_vals")
    ref = outs["staged predict_on_batch (fused = False)"]
    agree = all(len(o) == len(ref) and all(np.asarray(x[k]).shape == np.asarray(y[k]).shape and
                                           np.asarray(x[k]).tobytes() == np.asarray(y[k]).tobytes() for x, y in zip(o, ref) for k in keys)
                for o in outs.values())
    return {"config": "topdown_scaled: C3 top-down pair, instance UNet at input scale 0.5 (96x96 crops of the 512x512 resized frame), "
                      "1024x1024, max 5 animals, B=16, 128 pinned frames", "gpu": gpu_identity(),
            "metric": "frames/s (median of alternating repetitions; host frames in, result dicts out)", "repetitions": reps,
            "frames_per_s": {k: n / float(np.median(v)) for k, v in times.items()},
            "frames_per_s_range": {k: [n / max(v), n / min(v)] for k, v in times.items()},
            "mean_instances_per_frame": float(np.mean(np.concatenate([o["n_valid"] for o in ref]))),
            "arms_agree_bitwise": bool(agree)}


def topdown_gt_bench(steps):
    """Ground-truth centroids through the three routes of a TopDownPredictor built from an instance model only (see the
    module docstring), at input scales 1 and 0.5."""
    from sleap_b200.io.labels import Instance, LabeledFrame, Labels, LabelsReader, Skeleton
    from sleap_b200.io.video import Video
    n, B, animals = 128, 16, 5
    fr = frames(n, 1024, 1024, 1, 5)
    rng = np.random.default_rng(7)
    sk = Skeleton(FLIES13, [])
    lfs = [LabeledFrame(0, i, [Instance((rng.uniform(80, 944, 2) + rng.normal(0, 20, (13, 2))).astype(np.float32), sk)
                                for _ in range(animals)]) for i in range(n)]
    labels = Labels(lfs, [{}], [sk])
    labels.set_video(0, Video.from_numpy(fr))
    ispec = dict(backbone="unet", backbone_cfg=dict(unet(24, 16, 4), up_interpolate=False), head_type="centered_instance",
                 part_names=FLIES13, edges=None, heads=[dict(name="CenteredInstanceConfmapsHead", channels=13, output_stride=4)])
    keys = ("n_valid", "centroids", "centroid_vals", "instance_peaks", "instance_peak_vals")
    res = {}
    for scale, crop in ((1.0, 160), (0.5, 96)):
        def inference_model(fused):
            # each arm owns its device model: the staged calls reconfigure the chain the fused pipeline needs
            im_model = model_for(ispec, 1, 1004)[0]
            im_model.config_input_scale = scale                          # what Predictor._load(..., resize_in_graph=False) sets
            pred = TopDownPredictor(None, im_model, crop_size=crop, batch_size=B)
            pred.inference_model.instance_peaks.peak_threshold = 0.0
            pred.inference_model.fused = fused
            return pred

        staged, fused = inference_model(False), inference_model(True)
        assert not staged.inference_model._can_fuse() and fused.inference_model._can_fuse()
        reader = LabelsReader(labels, with_centroids=True)
        batches = list(fused._label_examples(reader))
        K = reader.max_instance_count()
        sim, fim = staged.inference_model, fused.inference_model
        arms = {"staged predict_on_batch (fused = False)": lambda: [sim.predict_on_batch(b) for b in batches],
                "fused predict_on_batch": lambda: [fim.predict_on_batch(b) for b in batches],
                "streamed predict_examples": lambda: [o for _, o in fim.predict_examples(batches, B, K)]}
        outs = {k: f() for k, f in arms.items()}                         # warm-up, and the outputs compared
        reps = max(5, steps)
        times = {k: [] for k in arms}
        for _ in range(reps):                                            # arms alternate
            for k, f in arms.items():
                t0 = time.perf_counter()
                f()
                times[k].append(time.perf_counter() - t0)
        ref = outs["staged predict_on_batch (fused = False)"]
        agree = all(len(o) == len(ref) and all(np.asarray(x[k]).shape == np.asarray(y[k]).shape and
                                               np.asarray(x[k]).tobytes() == np.asarray(y[k]).tobytes() for x, y in zip(o, ref) for k in keys)
                    for o in outs.values())
        assert agree, f"the routes disagree at input scale {scale}"
        res[f"s={scale:g}, {crop}x{crop} crops"] = {
            "repetitions": reps, "frames_per_s": {k: n / float(np.median(v)) for k, v in times.items()},
            "frames_per_s_range": {k: [n / max(v), n / min(v)] for k, v in times.items()},
            "mean_instances_per_frame": float(np.mean(np.concatenate([o["n_valid"] for o in ref]))), "arms_agree_bitwise": agree}
    return {"config": "topdown_gt: ground-truth centroids + C3 instance UNet, synthetic labels of 128 1024x1024 uint8 frames, "
                      "5 instances each, B=16", "gpu": gpu_identity(),
            "metric": "frames/s (median of alternating repetitions; decoded label batches in, result dicts out)", "workloads": res}


def topdown_gt_instances_bench(steps):
    """A centroid model with ground-truth instances (FindInstancePeaksGroundTruth, no instance model) through its three
    routes (see the module docstring): the C3 centroid UNet at input scale 0.5 on 128 gray tracking-clip frames, B = 16,
    the threshold calibrated to about 5 animals per frame, and 5 synthetic labelled instances of 13 nodes per frame."""
    import torch
    from scipy.ndimage import maximum_filter
    from sleap_b200.io.labels import Instance, LabeledFrame, Labels, LabelsReader, Skeleton
    from sleap_b200.io.video import Video
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from flow_clip import clip_frames
    n, B, animals = 128, 16, 5
    gray = torch.from_numpy(np.ascontiguousarray(clip_frames(n)[:, :, :, :1])).pin_memory().numpy()
    H, W = gray.shape[1:3]
    rng = np.random.default_rng(7)
    sk = Skeleton(FLIES13, [])
    lfs = []
    for i in range(n):
        pts = [(rng.uniform(80, [W - 80, H - 80]) + rng.normal(0, 20, (13, 2))).astype(np.float32) for _ in range(animals)]
        for p in pts:
            p[rng.random(13) < 0.1] = np.nan                                # some invisible nodes
        lfs.append(LabeledFrame(0, i, [Instance(p, sk) for p in pts]))
    labels = Labels(lfs, [{}], [sk])
    labels.set_video(0, Video.from_numpy(gray))
    cspec = dict(backbone="unet", backbone_cfg=unet(16, 16, 2), head_type="centroid", part_names=None, edges=None,
                 heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])

    def predictor(fused):
        # each arm owns its device model: the host route's centroid calls reconfigure the chain the fused pipeline needs
        cm_model, _, _ = model_for(cspec, 1, 1003, input_scale=0.5)
        cms = np.concatenate([cm_model.forward(gray[i:i + B])[0][..., 0] for i in range(0, 4 * B, B)])
        fifth = [np.sort(c[c == maximum_filter(c, size=3, mode="constant", cval=-np.inf)])[-5] for c in cms]
        pred = TopDownPredictor(cm_model, None, peak_threshold=float(np.median(fifth)), integral_refinement=True, batch_size=B)
        pred.inference_model.fused = fused
        return pred

    host, fused = predictor(False), predictor(True)
    reader = LabelsReader(labels, with_centroids=True)
    batches = list(fused._label_examples(reader))
    N = reader.max_instance_count()
    him, fim = host.inference_model, fused.inference_model
    arms = {"host route (fused = False)": lambda: [him.predict_on_batch(b) for b in batches],
            "fused predict_on_batch": lambda: [fim.predict_on_batch(b) for b in batches],
            "streamed predict_examples": lambda: [o for _, o in fim.predict_examples(batches, B, N)]}
    outs = {k: f() for k, f in arms.items()}                             # warm-up, and the outputs compared
    reps = max(5, steps)
    times = {k: [] for k in arms}
    for _ in range(reps):                                                # arms alternate
        for k, f in arms.items():
            t0 = time.perf_counter()
            f()
            times[k].append(time.perf_counter() - t0)
    keys = ("n_valid", "flags", "centroids", "centroid_vals", "instance_peaks", "instance_peak_vals")
    ref = outs["host route (fused = False)"]

    def same(x, y):                                                      # NaN positions, not NaN payloads
        x, y = np.asarray(x), np.asarray(y)
        return x.dtype == y.dtype and x.shape == y.shape and bool(np.array_equal(x, y, equal_nan=x.dtype.kind == "f"))

    agree = all(len(o) == len(ref) and all(same(x[k], y[k]) for x, y in zip(o, ref) for k in keys) for o in outs.values())
    assert agree, "the routes disagree"
    return {"config": "topdown_gt_instances: C3 centroid UNet (input scale 0.5) + ground-truth instances, 128 tracking-clip "
                      "frames (1024x1024 gray), about 5 animals, 5 labelled instances of 13 nodes per frame, B=16",
            "gpu": gpu_identity(),
            "metric": "frames/s (median of alternating repetitions; decoded label batches in, result dicts out)", "repetitions": reps,
            "frames_per_s": {k: n / float(np.median(v)) for k, v in times.items()},
            "frames_per_s_range": {k: [n / max(v), n / min(v)] for k, v in times.items()},
            "mean_centroids_per_frame": float(np.mean(np.concatenate([np.isfinite(o["centroid_vals"]).sum(1) for o in ref]))),
            "mean_rows_per_frame": float(np.mean(np.concatenate([o["n_valid"] for o in ref]))), "arms_agree": agree}


def topdown_track_bench(steps):
    """TopDownPredictor.predict (labels made) of the C3 pair of topdown() on 256 tracking-clip frames (gray), B = 16, the
    centroid threshold calibrated on clip frames to about 5 animals per frame.  Four arms alternate in one process: no
    tracker, the host simple tracker, the device simple tracker inside the fused step, and the device simple tracker on
    the per-frame route (fused = False, one sb_track_instances call per frame)."""
    import torch
    from scipy.ndimage import maximum_filter
    from sleap_b200.nn import tracking as T
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from flow_clip import clip_frames
    n, B = 256, 16
    gray = torch.from_numpy(np.ascontiguousarray(clip_frames(n)[:, :, :, :1])).pin_memory().numpy()
    cspec = dict(backbone="unet", backbone_cfg=unet(16, 16, 2), head_type="centroid", part_names=None, edges=None,
                 heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
    ispec = dict(backbone="unet", backbone_cfg=dict(unet(24, 16, 4), up_interpolate=False), head_type="centered_instance",
                 part_names=FLIES13, edges=None, heads=[dict(name="CenteredInstanceConfmapsHead", channels=13, output_stride=4)])

    def predictor(fused):
        # the per-frame arm owns its two device models: its staged calls reconfigure the chains the fused pipeline needs
        cm_model, _, _ = model_for(cspec, 1, 1003, input_scale=0.5)
        cms = np.concatenate([cm_model.forward(gray[i:i + B])[0][..., 0] for i in range(0, 4 * B, B)])
        fifth = [np.sort(c[c == maximum_filter(c, size=3, mode="constant", cval=-np.inf)])[-5] for c in cms]
        pred = TopDownPredictor(cm_model, model_for(ispec, 1, 1004)[0], crop_size=160, peak_threshold=float(np.median(fifth)),
                                integral_refinement=True, batch_size=B, max_instances=5)
        pred.inference_model.instance_peaks.peak_threshold = 0.0
        pred.inference_model.fused = fused
        return pred

    fused_pred, frame_pred = predictor(True), predictor(False)
    simple = dict(tracker="simple", similarity="instance", match="greedy")
    arms = {"no tracker": (fused_pred, lambda: None),
            "simple host": (fused_pred, lambda: T.Tracker.make_tracker_by_name(**simple)),
            "simple device, fused step": (fused_pred, lambda: T.Tracker.make_tracker_by_name(track_device=0, **simple)),
            "simple device, per-frame route (fused = False)": (frame_pred, lambda: T.Tracker.make_tracker_by_name(track_device=0, **simple))}

    def run(name, frames):
        pred, mk = arms[name]
        pred.tracker = mk()
        return pred.predict(frames)

    outs = {k: run(k, gray) for k in arms}                              # warm-up, and the outputs compared
    from track_cases import host_twin                                   # the host tracker with the device's greedy tie rule
    fused_pred.tracker = host_twin(**simple)
    stable = fused_pred.predict(gray)
    reps = max(3, steps)
    times = {k: [] for k in arms}
    for _ in range(reps):                                                # arms alternate
        for k in arms:
            t0 = time.perf_counter()
            run(k, gray)
            times[k].append(time.perf_counter() - t0)
    names = lambda frames: [[x.track.name if x.track else None for x in lf.instances] for lf in frames]
    return {"config": "topdown_track: C3 top-down pair, TopDownPredictor.predict with labels, 256 tracking-clip frames "
                      "(1024x1024 gray), max 5 animals, B=16", "gpu": gpu_identity(),
            "metric": "frames/s (median of alternating repetitions; host frames in, labeled frames out)", "repetitions": reps,
            "frames_per_s": {k: n / float(np.median(v)) for k, v in times.items()},
            "frames_per_s_spread": {k: [n / max(v), n / min(v)] for k, v in times.items()},
            "instances_per_frame": {k: float(np.mean([len(lf.instances) for lf in v])) for k, v in outs.items()},
            "tracks": {k: len({x.track.name for lf in v for x in lf.instances if x.track}) for k, v in outs.items()},
            "device_tracks_equal_host": names(outs["simple device, fused step"]) == names(outs["simple host"]),
            "device_tracks_equal_host_stable_ties": names(outs["simple device, fused step"]) == names(stable),
            "routes_agree": names(outs["simple device, fused step"]) == names(outs["simple device, per-frame route (fused = False)"])}


def pipeline_bench(steps):
    """predict_on_batch per batch against predict_batches on the same frames, alternating (see the module docstring)."""
    import torch
    from scipy.ndimage import maximum_filter
    from sleap_b200.nn import tracking as T
    from sleap_b200.nn.inference import TopDownMultiClassPredictor
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))
    from flow_clip import clip_frames
    n, B = 128, 16
    gray = torch.from_numpy(np.ascontiguousarray(clip_frames(n)[:, :, :, :1])).pin_memory().numpy()
    cspec = dict(backbone="unet", backbone_cfg=unet(16, 16, 2), head_type="centroid", part_names=None, edges=None,
                 heads=[dict(name="CentroidConfmapsHead", channels=1, output_stride=2)])
    ihead = dict(name="CenteredInstanceConfmapsHead", channels=13, output_stride=4)
    ispec = dict(backbone="unet", backbone_cfg=dict(unet(24, 16, 4), up_interpolate=False), head_type="centered_instance",
                 part_names=FLIES13, edges=None, heads=[ihead])
    classes = ["c0", "c1", "c2", "c3"]
    mspec = dict(ispec, head_type="multi_class_topdown", classes=classes,
                 heads=[ihead, dict(name="ClassVectorsHead", channels=len(classes), output_stride=16, vector=True, num_fc_layers=3,
                                    num_fc_units=64, global_pool=True)])
    sspec = dict(backbone="unet", backbone_cfg=unet(16, 16, 2), head_type="single_instance", part_names=FLIES13, edges=None,
                 heads=[dict(name="SingleInstanceConfmapsHead", channels=13, output_stride=2)])

    def centroid_model():
        m = model_for(cspec, 1, 1003, input_scale=0.5)[0]
        cms = np.concatenate([m.forward(gray[i:i + B])[0][..., 0] for i in range(0, 4 * B, B)])
        fifth = [np.sort(c[c == maximum_filter(c, size=3, mode="constant", cval=-np.inf)])[-5] for c in cms]
        return m, float(np.median(fifth))

    def topdown_model():
        cm, thr = centroid_model()
        pred = TopDownPredictor(cm, model_for(ispec, 1, 1004)[0], crop_size=160, peak_threshold=thr, integral_refinement=True,
                                batch_size=B, max_instances=5)
        pred.inference_model.instance_peaks.peak_threshold = 0.0
        return pred.inference_model

    def identity_model():
        cm, thr = centroid_model()
        icm = A.compile_model(mspec, 1)
        iw = A.make_synthetic_weights(icm, 1004)
        rng = np.random.default_rng(1005)
        dims = [icm.vector_taps["ClassVectorsHead"]["C"], 64, 64, 64, len(classes)]
        for i in range(4):
            iw["ClassVectorsHead" if i == 3 else f"pre_classification{i}_fc"] = dict(
                kernel=(rng.normal(0, 1, dims[i:i + 2]) * np.sqrt(2.0 / dims[i])).astype(np.float32),
                bias=rng.normal(0, 0.1, dims[i + 1]).astype(np.float32))
        pred = TopDownMultiClassPredictor(cm, DeviceModel(mspec, iw, input_channels=1, precision=0), crop_size=160, peak_threshold=thr,
                                          integral_refinement=True, batch_size=B, max_instances=5)
        pred.inference_model.instance_peaks.peak_threshold = 0.0
        return pred.inference_model

    single_im = SingleInstancePredictor(model_for(sspec, 1, 1001)[0], peak_threshold=0.2, integral_refinement=True,
                                        batch_size=B).inference_model
    td_im, td_trk_im = topdown_model(), topdown_model()
    simple = dict(tracker="simple", similarity="instance", match="greedy")
    workloads = {"single-instance UNet 1024x1024x1, 13 nodes": (single_im, None),
                 "C3 top-down pair, max 5 animals": (td_im, None),
                 "C3 top-down pair, max 5 animals, device simple tracker": (td_trk_im, simple),
                 "C3 identity pair (4 classes, 3 x 64 fc units), max 5 animals": (identity_model(), None)}

    def arm(im, trk, streamed):
        im.tracker = T.Tracker.make_tracker_by_name(track_device=0, **trk) if trk else None   # a fresh tracker per run
        try:
            if streamed:
                return list(im.predict_batches(gray, B))
            return [im.predict_on_batch(gray[i:i + B]) for i in range(0, n, B)]
        finally:
            if trk:
                im.detach_tracker()
                im.tracker = None

    def same(a, b):
        return len(a) == len(b) and all(sorted(x) == sorted(y) and all(np.asarray(x[k]).tobytes() == np.asarray(y[k]).tobytes() for k in x)
                                        for x, y in zip(a, b))

    reps = max(10, steps)
    res = {}
    for name, (im, trk) in workloads.items():
        outs = {s: arm(im, trk, s) for s in (False, True)}                # warm-up, and the outputs compared
        times = {False: [], True: []}
        for _ in range(reps):                                            # the two loops alternate
            for s in (False, True):
                t0 = time.perf_counter()
                arm(im, trk, s)
                times[s].append(time.perf_counter() - t0)
        res[name] = {"per_batch_frames_per_s": n / float(np.median(times[False])),
                     "streamed_frames_per_s": n / float(np.median(times[True])),
                     "per_batch_spread": [n / max(times[False]), n / min(times[False])],
                     "streamed_spread": [n / max(times[True]), n / min(times[True])],
                     "speedup": float(np.median(times[False]) / np.median(times[True])),
                     "outputs_equal": same(outs[False], outs[True])}
    return {"config": "pipeline: predict_on_batch per batch vs predict_batches, 128 pinned gray clip frames 1024x1024, B=16",
            "gpu": gpu_identity(), "metric": "frames/s (median of alternating repetitions; host frames in, result dicts out)",
            "repetitions": reps, "post_overlap": not os.environ.get("SB_DISABLE_POST_OVERLAP"), "workloads": res}


if __name__ == "__main__":
    which = [a for a in sys.argv[1:] if not a.startswith("--")] or ["c1", "c2", "c3", "c5"]
    steps = int(sys.argv[sys.argv.index("--steps") + 1]) if "--steps" in sys.argv else 10
    for c in which:
        if c == "c1":
            r = single("C1 single-instance UNet 256x256x1, 5 nodes, B=1", 256, list("abcde"), 1, steps)
        elif c == "c2":
            r = single("C2 single-instance UNet 512x512x1, 13 nodes, B=32", 512, FLIES13, 32, steps)
        elif c in ("c3", "topdown"):
            r = topdown(steps)
        elif c == "topdown_scaled":
            r = topdown_scaled_bench(steps)
        elif c == "topdown_gt":
            r = topdown_gt_bench(steps)
        elif c == "topdown_gt_instances":
            r = topdown_gt_instances_bench(steps)
        elif c == "r50":
            r = resnet50(steps)
        elif c == "track":
            r = track_bench()
        elif c == "multiclass":
            r = multiclass_bench(steps)
        elif c == "topdown_multiclass":
            r = topdown_multiclass_bench(steps)
        elif c == "topdown_track":
            r = topdown_track_bench(steps)
        elif c == "pipeline":
            r = pipeline_bench(steps)
        else:
            b5 = int(sys.argv[sys.argv.index("--c5-batch") + 1]) if "--c5-batch" in sys.argv else 16
            r = hourglass(max(3, steps // 3), b5)
        print(json.dumps(r), flush=True)
