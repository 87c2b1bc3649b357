/*
 * libsleapb200 -- C-ABI of the H100-native SLEAP inference path.
 *
 * The reference (talmolab/sleap v1.4.1) has no FFI: its seam is the Python class surface
 * sleap.nn.inference.{Predictor, InferenceModel, InferenceLayer} plus the function-level
 * modules sleap.nn.peak_finding and sleap.nn.paf_grouping, all of which dispatch TensorFlow
 * ops.  Every entry point below names the reference interface (file:line under
 * /root/reference) whose device work it replaces.  INTEGRATION.md shows the ctypes binding.
 *
 * Conventions
 *   - plain C: pointers + sizes only; all functions return 0 (SB_OK) or a negative SB_ERR_*;
 *     nothing throws.  sb_last_error() returns the message of the last failure.
 *   - one handle per GPU; calls on one handle are serialised by the caller; different handles
 *     are independent.  Device buffers are owned by the handle, host buffers by the caller.
 *   - pointers named *_host are host memory, *_dev are device memory on the handle's GPU.
 *   - images / maps are NHWC, row-major; points are (x, y) float32; missing values are NaN.
 */
#ifndef SLEAP_B200_H_
#define SLEAP_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB_OK 0
#define SB_ERR_INVALID (-1)
#define SB_ERR_CUDA (-2)
#define SB_ERR_UNSUPPORTED (-3)
#define SB_ERR_NO_DEVICE (-4)

/* refinement modes (sleap/nn/peak_finding.py:337-420, 451-532: refinement=None|"integral"|"local") */
#define SB_REFINE_NONE 0
#define SB_REFINE_INTEGRAL 1
#define SB_REFINE_LOCAL 2

/* overflow flags reported per sample (capacity-bounded device buffers; the reference is unbounded).  What is kept:
   PEAKS_TRUNCATED: the first max_peaks_per_sample peaks in tf.where (row-major NHWC) order;
   NODE_PEAKS_TRUNCATED: grouping sees the first max_node_peaks peaks of each node, in the same order;
   INSTANCES_TRUNCATED: the first max_instances instances of the reference's output order. */
#define SB_FLAG_PEAKS_TRUNCATED 1
#define SB_FLAG_NODE_PEAKS_TRUNCATED 2
#define SB_FLAG_INSTANCES_TRUNCATED 4

typedef struct sb_handle_s* sb_handle_t;

/* ---- lifetime --------------------------------------------------------------------------- */
int sb_version(void);
/* replaces the device selection of sleap/nn/system.py:29-110 (one GPU per process) */
int sb_create(int device_id, sb_handle_t* out_handle);
int sb_destroy(sb_handle_t h);
const char* sb_last_error(sb_handle_t h); /* h may be NULL: last error of this thread */
int sb_synchronize(sb_handle_t h);
/* number of kernels this handle has launched so far (bench.py "gpu_launches") */
int sb_gpu_launches(sb_handle_t h);
/* use the caller's CUDA stream (e.g. torch's current stream) for all subsequent work; NULL = own */
int sb_set_stream(sb_handle_t h, void* cuda_stream);

/* ---- stage level: peak finding (host buffers) --------------------------------------------
 * sleap/nn/peak_finding.py:451-532 find_local_peaks (+ :249-308 rough, :646-707 with offsets).
 * cms (B,H,W,C) f32.  offsets_host: NULL, or learned offset maps (B,H,W,2C) -> "with_offsets".
 * Outputs are ordered like tf.where: (sample, y, x, channel) row-major.  At most
 * max_peaks_per_sample peaks are kept per sample (first in order); out arrays must hold
 * B*max_peaks_per_sample entries.  out_flags (B) receives SB_FLAG_* (may be NULL). */
int sb_find_local_peaks(sb_handle_t h, const float* cms_host, int B, int H, int W, int C,
                        float threshold, int refinement, int integral_patch_size,
                        const float* offsets_host, int max_peaks_per_sample,
                        float* out_points, float* out_vals, int32_t* out_sample_inds,
                        int32_t* out_channel_inds, int32_t* out_n_peaks, int32_t* out_flags);

/* sleap/nn/peak_finding.py:337-420 find_global_peaks (+ :193-246 rough, :566-643 with offsets).
 * out_points (B,C,2), out_vals (B,C). */
int sb_find_global_peaks(sb_handle_t h, const float* cms_host, int B, int H, int W, int C,
                         float threshold, int refinement, int integral_patch_size,
                         const float* offsets_host, float* out_points, float* out_vals);

/* sleap/nn/peak_finding.py:135-190 crop_bboxes on make_centered_bboxes
 * (sleap/nn/data/instance_cropping.py:124-166).  images (B,H,W,C) u8 or f32; centroids (n,2) xy;
 * out (n,crop_h,crop_w,C) same dtype as images (u8: float->u8 truncation as the reference). */
int sb_crop_centered(sb_handle_t h, const void* images_host, int images_are_u8, int B, int H,
                     int W, int C, const float* centroids, const int32_t* sample_inds, int n,
                     int crop_h, int crop_w, void* out_crops);

/* CentroidCrop.call with precrop_resize = scale (sleap/nn/inference.py:1836-1841, :1918-1927): the crops of
 * resize_image(images, scale) (sleap/nn/data/resizing.py:71-106: int(float32(W) * scale) x int(float32(H) * scale),
 * bilinear with half-pixel centres, no antialias, cast back to the frame dtype -- uint8 by truncation), byte for byte;
 * centroids are in resized-frame coordinates.  The resized frames are computed on the fly and never stored.
 * SB_ERR_INVALID: a scale that is not finite and positive, or that gives a resized frame with a zero extent. */
int sb_crop_centered_resized(sb_handle_t h, const void* images_host, int images_are_u8, int B, int H, int W, int C,
                             const float* centroids, const int32_t* sample_inds, int n, int crop_h, int crop_w,
                             float scale, void* out_crops);

/* ---- stage level: PAF grouping (host buffers) --------------------------------------------
 * sleap/nn/paf_grouping.py:406-550 score_paf_lines_batch (:82-142 candidates, :145-275 line
 * sampling, :278-403 scoring).  pafs (B,Hp,Wp,2E) f32; peaks (N,2) image px, peak_channel_inds
 * (N), grouped by sample through peak_offsets (B+1).  Outputs: flat candidate lists in
 * (sample, edge, src-major) order; cand_offsets (B+1).  cap = capacity of the out arrays. */
int sb_score_paf_lines_batch(sb_handle_t h, const float* pafs_host, int B, int Hp, int Wp, int C2,
                             const float* peaks, const int32_t* peak_channel_inds,
                             const int32_t* peak_offsets, const int32_t* skeleton_edges,
                             int n_edges, int n_nodes, int n_line_points, int pafs_stride,
                             float max_edge_length_ratio, float dist_penalty_weight,
                             int cap, int32_t* out_edge_inds, int32_t* out_edge_peak_inds,
                             float* out_line_scores, int32_t* out_cand_offsets);

/* sleap/nn/paf_grouping.py:145-222 make_line_subs, :225-275 get_paf_lines, :325-403
 * score_paf_lines for an explicit candidate list of ONE sample.  pafs_sample (Hp,Wp,C2) may be
 * NULL when lines_in (n,P,2) is given (score_paf_lines on pre-gathered lines).  Any of the
 * outputs may be NULL: out_subs (n,P,2) int32 [row,col]; out_lines (n,P,2); out_scores (n). */
int sb_paf_lines(sb_handle_t h, const float* pafs_sample, int Hp, int Wp, int C2,
                 const float* lines_in, const float* peaks, int n_peaks,
                 const int32_t* edge_peak_inds, const int32_t* edge_inds, int n, int n_line_points,
                 int pafs_stride, float max_edge_length, float dist_penalty_weight,
                 int32_t* out_subs, float* out_lines, float* out_scores);

/* sleap/nn/peak_finding.py:311-334 integral_regression: cms (N,h,w,C), xv (w), yv (h) ->
 * x_hat, y_hat (N,C). */
int sb_integral_regression(sb_handle_t h, const float* cms, int N, int Hh, int Ww, int C,
                           const float* xv, const float* yv, float* x_hat, float* y_hat);
/* sleap/nn/peak_finding.py:78-132 find_offsets_local_direction: patches (N,3,3,1) -> (N,2). */
int sb_find_offsets_local_direction(sb_handle_t h, const float* patches, int N, float delta,
                                    float* out_offsets);

/* sleap/nn/utils.py:79-98 tf_linear_sum_assignment, batched, as called from
 * sleap/nn/paf_grouping.py:621-650: problem p is the (n_src[p], n_dst[p]) row-major SCORE
 * matrix at scores + offsets[p]; cost = -score, NaN -> +inf; minimum-cost assignment with
 * SciPy's rectangular shortest-augmenting-path semantics.  Outputs per problem at
 * p*max_k: rows (ascending), cols, matched scores; out_counts[p] (0 when infeasible). */
int sb_linear_sum_assignment_batch(sb_handle_t h, const float* scores, const int32_t* n_src,
                                   const int32_t* n_dst, const int32_t* offsets, int n_problems,
                                   int max_k, int32_t* out_rows, int32_t* out_cols,
                                   float* out_scores, int32_t* out_counts);

/* sleap/nn/paf_grouping.py:1115-1290 group_instances_batch (:984-1112 per sample, :799-914
 * greedy assignment, :917-981 instance assembly).  Matches are edge-LOCAL indices grouped by
 * sample through match_offsets (B+1), in the order produced by match_candidates_batch.
 * Outputs: out_instances (B,max_instances,n_nodes,2), out_peak_scores (B,max_instances,n_nodes),
 * out_instance_scores (B,max_instances), out_n_instances (B). */
int sb_group_instances_batch(sb_handle_t h, int B, int n_nodes, const float* peaks,
                             const float* peak_vals, const int32_t* peak_channel_inds,
                             const int32_t* peak_offsets, const int32_t* match_edge_inds,
                             const int32_t* match_src_peak_inds, const int32_t* match_dst_peak_inds,
                             const float* match_line_scores, const int32_t* match_offsets,
                             const int32_t* edge_types, int n_edges,
                             const int32_t* sorted_edge_inds, int n_sorted, int min_instance_peaks,
                             float min_line_scores, int max_instances, float* out_instances,
                             float* out_peak_scores, float* out_instance_scores,
                             int32_t* out_n_instances);

/* ---- models --------------------------------------------------------------------------------
 * A model is the flat op-list compiled (host side, sleap_b200/nn/architectures.py) from the
 * reference's backbone + heads graph: sleap/nn/model.py:312-364, architectures/unet.py,
 * encoder_decoder.py, hourglass.py, heads.py:42-63.  ops: n_ops records of SB_OP_WORDS int32
 * (layout in sleap_b200/nn/oplist.py); weights: float32 blob the ops index into.
 * Replaces tf.keras.models.load_model + keras_model(imgs) (sleap/nn/inference.py:3203-3213,
 * :2875).  precision: 0 = fp16 tensor-core path (fp32 accumulate), 1 = fp32 CUDA-core path,
 * 2 = fp32-grade results on the tensor-core path: activations / weights as hi + lo fp16 pairs; the op-list must
 * have been compiled for it (compile_model(split=True): 3C physical channels [lo | hi | hi] per fp16 tensor, weight
 * rows [Wh | Wl | Wh], fp32 frame buffer; conv out_C stays the logical C_out) -- DESIGN.md 5.7. */
#define SB_OP_WORDS 24
int sb_load_model(sb_handle_t h, const int32_t* ops, int n_ops, const float* weights,
                  int64_t n_weights, int precision, int* out_model_id);

/* Plan device buffers for (max_batch, H, W, C_in) uint8/float input frames. */
int sb_model_configure(sb_handle_t h, int model_id, int max_batch, int H, int W, int C_in);

/* Forward only (conv parity tests): images_host (B,H,W,C_in) u8 (images_are_u8) or f32 in [0,1].
 * Copies each requested output tensor (op-list buffer id) to host as f32 NHWC. */
int sb_model_forward(sb_handle_t h, int model_id, const void* images_host, int images_are_u8,
                     int B, int n_outputs, const int32_t* output_buffer_ids,
                     float** out_host_ptrs);

/* Device-side timing of one forward pass, op by op (CUDA events on the launching stream).
 * out_kind: 0 other, 1 tensor-core conv, 2 CUDA-core conv; out_flops: 2*MACs for the batch. */
int sb_model_profile_ops(sb_handle_t h, int model_id, const uint8_t* frames_dev, int B, int cap,
                         float* out_ms, int32_t* out_kind, double* out_flops, int32_t* out_n_ops);

/* Live timing of the network part of every step: while enabled, each forward pass (whatever entry point runs it:
 * sb_model_forward, sb_infer_*, the *_submit calls and the top-down collects, sb_infer_topdown) is bracketed by a pair of CUDA events on the
 * launching stream.  A call synchronises that stream, returns the milliseconds of the passes recorded since the last
 * call (at most cap, at most 1024 are kept), clears them, and switches the recording on / off.  bench.py derives
 * `roofline.achieved` from the passes of its timed region.  Replaces nothing in the reference (it has no device
 * timers; tf.profiler is its tool). */
int sb_model_forward_times(sb_handle_t h, int model_id, int enable, int cap, float* out_ms, int32_t* out_n);

/* ---- fused predictors ------------------------------------------------------------------------
 * sleap/nn/inference.py:2737-3003 BottomUpInferenceLayer.call: preprocess -> net -> local peaks
 * -> * cm_output_stride -> PAFScorer.predict -> (/input_scale + 0.5). */
typedef struct sb_bottomup_params {
  int32_t cms_buffer, pafs_buffer, offsets_buffer; /* op-list buffer ids (offsets: -1 if none) */
  int32_t cm_output_stride, paf_output_stride;
  float peak_threshold;
  int32_t refinement, integral_patch_size;
  int32_t n_nodes, n_edges;
  const int32_t* edges;            /* (n_edges, 2) node indices */
  const int32_t* sorted_edge_inds; /* BFS edge order from the topological root */
  int32_t n_sorted;
  int32_t n_line_points;
  float max_edge_length_ratio, dist_penalty_weight, min_line_scores;
  int32_t min_instance_peaks;
  float input_scale;
  int32_t max_peaks_per_sample, max_node_peaks, max_instances;
} sb_bottomup_params;

int sb_bottomup_configure(sb_handle_t h, int model_id, const sb_bottomup_params* params);

/* frames: (B,H,W,C_in) uint8.  *_host variant copies H2D / D2H inside; *_dev takes frames
 * already resident in HBM and leaves results on the device (the records of
 * sb_bottomup_device_records).  Outputs: instance_peaks (B,max_instances,n_nodes,2),
 * instance_peak_vals (B,max_instances,n_nodes), instance_scores (B,max_instances),
 * n_valid (B), flags (B). */
int sb_infer_bottomup(sb_handle_t h, int model_id, const uint8_t* frames_host, int B,
                      float* out_instance_peaks, float* out_instance_peak_vals,
                      float* out_instance_scores, int32_t* out_n_valid, int32_t* out_flags);
int sb_infer_bottomup_dev(sb_handle_t h, int model_id, const uint8_t* frames_dev, int B);
/* Streamed steps.  Streaming form of sb_infer_bottomup for many batches (sleap/nn/inference.py:377-420, the
 * Predictor batch loop): sb_bottomup_submit queues the H2D copy (copy stream), the network and the
 * post-processing of one batch into slot 0/1 and returns; sb_bottomup_collect blocks until that
 * slot's results are in host memory.  Submitting batch i+1 before collecting batch i overlaps its
 * upload with the compute of batch i.  frames_host should be pinned for a truly asynchronous copy.
 * Every *_submit / *_collect pair below (bottom-up, multi-class, global, top-down, top-down identity, ground-truth
 * top-down) follows these rules.  Refused (SB_ERR_INVALID, nothing queued): a submit with a slot other than 0 / 1 or B
 * outside [1, max batch]; a submit into a slot whose batch was not collected; a collect of a slot that holds no
 * batch, with another B than its submit, or before the batch submitted earlier into the other slot.  A slot read
 * (sb_bottomup_tracks, sb_bottomup_gathered, sb_topdown_tracks; slot 0 / 1) takes only the batch last collected from
 * that slot, with its B.  A configure call on the model (or either model of a top-down pipeline) drops the submitted
 * batches after their work has finished; collecting one then fails.
 * The synchronous call of each form (sb_infer_bottomup, sb_infer_multiclass, sb_infer_global, sb_infer_topdown,
 * sb_infer_topdown_multiclass) runs its batch as a submit into slot 0 and its collect: it is refused (SB_ERR_INVALID,
 * nothing queued) while a batch is submitted and not collected, and its batch is then the one last collected from slot
 * 0.  The slots are allocated by the first submit or synchronous call: two of max_batch uint8 frames and pinned record
 * staging per model (per pipeline for the top-down forms). */
int sb_bottomup_submit(sb_handle_t h, int model_id, const uint8_t* frames_host, int B, int slot);
int sb_bottomup_collect(sb_handle_t h, int model_id, int slot, int B, float* out_instance_peaks,
                        float* out_instance_peak_vals, float* out_instance_scores,
                        int32_t* out_n_valid, int32_t* out_flags);

/* sb_infer_bottomup_dev returns as soon as the work is queued: the network runs on the handle's
 * stream and the post-processing on a second stream, so that it overlaps the network of the next
 * call.  sb_get_post_stream exposes the post-processing stream; sb_synchronize joins both. */
int sb_get_post_stream(sb_handle_t h, void** out_stream);
/* Device pointer of the contiguous per-frame result records the grouping kernel writes ([max_batch][width] float32,
 * width = ceil4(max_instances*n_nodes*3 + max_instances + 2): peaks | peak values | instance scores | n_valid | flags). */
int sb_bottomup_device_records(sb_handle_t h, int model_id, float** records_dev);
/* PAF graph of the last bottom-up call (return_paf_graph, inference.py:2995-3001); same layout
 * as sb_find_local_peaks / sb_score_paf_lines_batch outputs. */
int sb_bottomup_fetch_graph(sb_handle_t h, int model_id, int B, int cap_peaks, float* peaks,
                            float* peak_vals, int32_t* peak_channel_inds, int32_t* peak_offsets,
                            int cap_cands, int32_t* edge_inds, int32_t* edge_peak_inds,
                            float* line_scores, int32_t* cand_offsets);

/* The same post-processing chain on caller-supplied maps (no network): cms (B,H,W,n_nodes),
 * pafs (B,Hp,Wp,2*n_edges), optional learned offsets (B,H,W,2*n_nodes).  This is the entry the
 * parity tests drive (identical cms/pafs in -> bit-exact peaks / assignments out).  The PAF-graph
 * outputs are optional (peaks == NULL skips them).  params->*_buffer fields are ignored. */
int sb_bottomup_from_maps(sb_handle_t h, const sb_bottomup_params* params, const float* cms_host,
                          int B, int H, int W, const float* pafs_host, int Hp, int Wp,
                          const float* offsets_host, float* out_instance_peaks,
                          float* out_instance_peak_vals, float* out_instance_scores,
                          int32_t* out_n_valid, int32_t* out_flags, int cap_peaks, float* peaks,
                          float* peak_vals, int32_t* peak_channel_inds, int32_t* peak_offsets,
                          int cap_cands, int32_t* edge_inds, int32_t* edge_peak_inds,
                          float* line_scores, int32_t* cand_offsets);

/* ---- bottom-up multi-class (identity) step -----------------------------------------------------------
 * sleap/nn/inference.py:3351-3589 BottomUpMultiClassInferenceLayer.call: preprocess -> net -> local peaks
 * -> * cm_output_stride -> class probability at each peak (sigmoid of the class-map logit at the rounded class-map cell,
 * 0 outside the map) -> per (frame, node) SciPy assignment of peaks to classes on -probability, a match kept only where
 * it is the peak's most probable class -> (/input_scale + 0.5).  One record per frame comes back.
 * A model runs one post-processing chain at a time (bottom-up, multi-class, global peaks or centroids): any of their
 * configure calls drops the model's previous chain, with its tracker and record exchange, and so does
 * sb_model_configure.  A call for another chain than the model's is refused.  A configure call refused for its
 * arguments leaves the previous chain in place.  The fused top-down pipeline must be configured again
 * (sb_topdown_configure) after either of its models is reconfigured.
 * Caps: n_classes <= SB_MAX_CLASSES (SB_ERR_INVALID).  The grouping kernels keep a node's peaks, their class
 * probabilities and the assignment's scratch in shared memory, about 4 * max_node_peaks * n_classes bytes plus 42 bytes
 * per row or column of the assignment; sb_multiclass_configure and sb_multiclass_from_maps refuse (SB_ERR_UNSUPPORTED) a
 * max_node_peaks that would need more than the device's opt-in shared memory per block (227 KB on an H100: up to 408
 * peaks per node with 128 classes).  sb_bottomup_configure and sb_bottomup_from_maps do the same for the PAF chain,
 * whose matching keeps a max_node_peaks^2 score matrix (up to 235 peaks per node on an H100). */
#define SB_MAX_CLASSES 128
typedef struct sb_multiclass_params {
  int32_t cms_buffer, class_maps_buffer, offsets_buffer; /* op-list buffer ids (offsets: -1 if none) */
  int32_t cm_output_stride, class_maps_output_stride;
  float peak_threshold;
  int32_t refinement, integral_patch_size;
  int32_t n_nodes, n_classes;          /* n_classes <= SB_MAX_CLASSES */
  float input_scale;
  int32_t max_peaks_per_sample, max_node_peaks;
} sb_multiclass_params;

int sb_multiclass_configure(sb_handle_t h, int model_id, const sb_multiclass_params* params);
/* frames (B,H,W,C_in) uint8 or float32.  Outputs, class-indexed and NaN where no peak was assigned:
 * out_points (B,n_classes,n_nodes,2), out_vals (B,n_classes,n_nodes) peak values,
 * out_class_probs (B,n_classes,n_nodes), out_flags (B) SB_FLAG_* (may be NULL). */
int sb_infer_multiclass(sb_handle_t h, int model_id, const void* frames_host, int frames_are_u8, int B,
                        float* out_points, float* out_vals, float* out_class_probs, int32_t* out_flags);
/* The streamed form, as sb_bottomup_submit / sb_bottomup_collect, with the rules of the streamed steps (uint8 frames). */
int sb_multiclass_submit(sb_handle_t h, int model_id, const uint8_t* frames_host, int B, int slot);
int sb_multiclass_collect(sb_handle_t h, int model_id, int slot, int B, float* out_points, float* out_vals,
                          float* out_class_probs, int32_t* out_flags);
/* The same post-processing on caller-supplied maps (no network): cms (B,H,W,n_nodes), class-map logits
 * (B,Hc,Wc,n_classes), optional learned offsets (B,H,W,2*n_nodes).  params->*_buffer fields are ignored. */
int sb_multiclass_from_maps(sb_handle_t h, const sb_multiclass_params* params, const float* cms_host, int B, int H, int W,
                            const float* class_logits_host, int Hc, int Wc, const float* offsets_host, float* out_points,
                            float* out_vals, float* out_class_probs, int32_t* out_flags);

/* ---- multi-GPU: exchange of the per-frame result records over NVLink peer memory -----------------
 * The reference runs on one GPU (sleap/nn/system.py:29-46 rejects more than one visible device); its consumer of the
 * per-frame results is Predictor._make_labeled_frames_from_generator (sleap/nn/inference.py:3230-3343).  Here frames
 * are sharded over one process per GPU and the grouping kernel's epilogue writes every frame's fixed-size record
 * [max_instances*n_nodes*2 peaks | max_instances*n_nodes values | max_instances scores | n_valid | flags] (float32)
 * directly into a gather window in EVERY rank's HBM (CUDA-IPC peer mappings over NVLink / NVSwitch) -- no collective
 * call, no rank waits for another inside a step.  Windows are `generations` deep; a consumer acknowledges a step to
 * all producers, and a producer only ever waits when it is `generations` steps ahead of the slowest consumer.
 *   sb_gather_init     allocate this rank's window, return its 64-byte CUDA IPC handle (exchange the handles of all
 *                      ranks out of band, e.g. torch.distributed.all_gather_object)
 *   sb_gather_connect  map every peer's window (all_ipc_handles: world x 64 bytes, rank order); from now on every
 *                      sb_infer_bottomup* / sb_bottomup_submit call pushes its records (one "step" per call)
 *   sb_gather_collect  host consumer: records of `step` from all ranks -> out_records_host [world][B][width]
 *                      (rank-major = frame order for contiguous shards), out_counts[r] = frames rank r pushed
 *   sb_gather_consume_dev  device consumer: wait + acknowledge on the post-processing stream (step < 0: the next
 *                      unconsumed step; results stay in the window returned by sb_gather_window until `generations`
 *                      later steps have been pushed)
 * All waits are bounded (5 s): a dead peer produces an error from sb_gather_collect / sb_gather_status, not a hang. */
#define SB_IPC_HANDLE_BYTES 64
int sb_gather_init(sb_handle_t h, int model_id, int rank, int world, int generations, void* out_ipc_handle);
int sb_gather_connect(sb_handle_t h, int model_id, const void* all_ipc_handles);
int sb_gather_enabled(sb_handle_t h, int model_id);
int sb_gather_consume_dev(sb_handle_t h, int model_id, int64_t step);
int sb_gather_window(sb_handle_t h, int model_id, int64_t step, float** out_dev_ptr, int64_t* out_floats);
int sb_gather_collect(sb_handle_t h, int model_id, int64_t step, int B, float* out_records_host, int32_t* out_counts);
int sb_gather_status(sb_handle_t h, int model_id, int32_t* out_status, int64_t* out_steps_pushed, int64_t* out_steps_consumed);
/* With the exchange connected, sb_infer_bottomup / sb_bottomup_submit wait (on the device, behind the post-processing) for
 * every rank's records of their step and bring the WHOLE gather window to the host in the one result copy they do anyway
 * (their own outputs are the rank's slice of it).  sb_bottomup_gathered returns the copy of the batch last collected from
 * slot 0 / 1 (slot 0 after sb_infer_bottomup).  out_records [world][B][width], out_counts [world]. */
int sb_bottomup_gathered(sb_handle_t h, int model_id, int slot, int B, float* out_records, int32_t* out_counts);
int sb_gather_close(sb_handle_t h, int model_id);

/* sleap/nn/inference.py:1229-1380 SingleInstanceInferenceLayer.call and :1969-2200
 * FindInstancePeaks.call: net -> global peaks -> * output_stride -> (/input_scale + 0.5)
 * (+ crop_offsets / input_scale when crop_offsets_host != NULL).
 * out_points (B,n_nodes,2), out_vals (B,n_nodes). */
typedef struct sb_global_params {
  int32_t cms_buffer, offsets_buffer;
  int32_t output_stride;
  float peak_threshold;
  int32_t refinement, integral_patch_size;
  float input_scale;
} sb_global_params;
int sb_global_configure(sb_handle_t h, int model_id, const sb_global_params* params);
int sb_infer_global(sb_handle_t h, int model_id, const void* images_host, int images_are_u8,
                    int B, const float* crop_offsets_host, float* out_points, float* out_vals);
/* The streamed form, as sb_bottomup_submit / sb_bottomup_collect (rules, uint8 frames, no crop offsets): the global
 * peaks run on the post-processing stream and the points | values block comes back in one copy per batch. */
int sb_global_submit(sb_handle_t h, int model_id, const uint8_t* frames_host, int B, int slot);
int sb_global_collect(sb_handle_t h, int model_id, int slot, int B, float* out_points, float* out_vals);

/* sleap/nn/inference.py:1638-1966 CentroidCrop.call: net -> local peaks -> * output_stride ->
 * /input_scale + 0.5; returns flat centroid list ordered by (sample, y, x) like the reference
 * (max_instances / top_k selection and cropping are separate calls: sb_crop_centered). */
typedef struct sb_centroid_params {
  int32_t cms_buffer, offsets_buffer;
  int32_t output_stride;
  float peak_threshold;
  int32_t refinement, integral_patch_size;
  float input_scale;
  int32_t max_peaks_per_sample;
} sb_centroid_params;
int sb_centroid_configure(sb_handle_t h, int model_id, const sb_centroid_params* params);
int sb_infer_centroids(sb_handle_t h, int model_id, const void* images_host, int images_are_u8,
                       int B, float* out_centroids, float* out_vals, int32_t* out_sample_inds,
                       int32_t* out_n, int32_t* out_flags);

/* sleap/nn/inference.py:2273-2311 TopDownInferenceModel.call = CentroidCrop.call (:1747-1966) -> FindInstancePeaks.call
 * (:2059-2200), as ONE device pipeline: frames are uploaded once, the centroid peaks, the per-frame top-k
 * (tf.math.top_k(max_instances), :1879-1894), the crops (crop_bboxes on the resident frames, :1918-1927) and the
 * centered-instance network + global peaks (+ crop offsets) never leave the GPU; results come back in one copy.
 * Outputs are dense and NaN padded: centroids (B,K,2), centroid_vals (B,K), instance_peaks (B,K,n_nodes,2),
 * instance_peak_vals (B,K,n_nodes) with K = max_centroids_per_frame; n_valid (B); flags (B).  The instance network is
 * configured for max_crops_per_call crops of crop_size x crop_size and runs as often as the batch's crop count needs.
 * An instance model trained at an input scale s != 1 (CentroidCrop.precrop_resize, :1836-1843): the centroids are
 * multiplied by s (one float32 multiply, before the top-k) and the crops are cut from the frames resized by s, as
 * sb_crop_centered_resized cuts them, without storing the resized frames; the returned centroids are in resized-frame
 * coordinates, the instance peaks in frame coordinates (/ s + 0.5, + crop offset / s, with instance.input_scale = s). */
typedef struct sb_topdown_params {
  int32_t centroid_model, instance_model;
  sb_centroid_params centroid;      /* as sb_centroid_configure */
  sb_global_params instance;        /* as sb_global_configure */
  int32_t crop_size;
  int32_t max_instances;            /* top-k per frame by centroid confidence; <= 0: keep every centroid */
  int32_t max_centroids_per_frame;  /* K */
  int32_t max_crops_per_call;       /* batch the instance network is planned for */
  float precrop_resize;             /* s: resize the frames by s before cropping; 1 or 0: no resize.  SB_ERR_INVALID at
                                       configure time: negative, NaN or infinite, or a resized frame with a zero extent */
} sb_topdown_params;
int sb_topdown_configure(sb_handle_t h, const sb_topdown_params* params, int max_batch, int H, int W, int C_in);
int sb_infer_topdown(sb_handle_t h, int centroid_model_id, const void* frames_host, int frames_are_u8, int B,
                     float* out_centroids, float* out_centroid_vals, float* out_instance_peaks,
                     float* out_instance_peak_vals, int32_t* out_n_valid, int32_t* out_flags);
/* The streamed form (uint8 frames; arguments and rules as sb_bottomup_submit / _collect, outputs as sb_infer_topdown).  A
 * step is a centroid stage (network, peaks, top-k, crop list, the crop count's copy to the host) and an instance stage
 * (crops, instance network, peaks, records, tracker, the records' copy).  sb_topdown_submit queues the batch's upload on
 * a copy stream into slot `slot`, then the instance stage of the batch submitted before it (waiting on the host for that
 * batch's crop count, which its centroid stage produced while the GPU ran it), then the batch's own centroid stage.
 * sb_topdown_collect queues the batch's instance stage if no submit did, and blocks until its records are on the host.
 * Also refused (SB_ERR_INVALID): sb_infer_centroids on the centroid model and sb_topdown_attach_tracker while a batch
 * is submitted and not collected; a submit or collect of the other pipeline form.
 * A batch's instance stage, and with it the attached tracker's step, is queued by the next submit or by its collect:
 * sb_tracker_reset between a batch's submit and that point applies before the batch is tracked, and the attached tracker
 * must not be destroyed while a batch is submitted. */
int sb_topdown_submit(sb_handle_t h, int centroid_model_id, const uint8_t* frames_host, int B, int slot);
/* model_id: the pipeline's owner -- the centroid model, or the instance model of a ground-truth pipeline. */
int sb_topdown_collect(sb_handle_t h, int model_id, int slot, int B, float* out_centroids, float* out_centroid_vals,
                       float* out_instance_peaks, float* out_instance_peak_vals, int32_t* out_n_valid, int32_t* out_flags);

/* ---- ground-truth centroids ------------------------------------------------------------------------
 * sleap/nn/inference.py:743-809 CentroidCropGroundTruth.call -> FindInstancePeaks.call (or TopDownMultiClassFindPeaks.call):
 * the instance step above on centroids the caller supplies.  sb_topdown_configure and sb_topdown_multiclass_configure with
 * params.centroid_model = -1 configure it: the pipeline belongs to the instance model and is addressed by its id;
 * `centroid` and `max_instances` are ignored (no top-k); max_centroids_per_frame (K) is the per-frame capacity;
 * precrop_resize is CentroidCropGroundTruth.input_scale (the multi-class form refuses one other than 0 or 1, as above).
 * A batch holds at most max_batch x K crops, so the instance network is configured for min(max_crops_per_call,
 * max_batch x K) crops per chunk.
 * The pipeline owns two slots of max_batch uint8 frames of H x W x C_in, allocated at its first submit.  A configure call
 * on the instance model drops the pipeline and its submitted batches.
 * sb_topdown_gt_submit queues one whole step into slot 0 / 1 without waiting on the host: the frames and the centroid
 * table (B,K,2) (frame coordinates, float32, rows past a frame's count ignored, NaN allowed) with counts (B), each in
 * [0, K], are copied on a copy stream; the centroids are multiplied by precrop_resize (one float32 multiply), their
 * values are 1, and the crops, instance network, peaks and records follow as in sb_topdown_submit.  Refused
 * (SB_ERR_INVALID, nothing queued, the slot stays free): a count outside [0, K], and as every streamed submit.  Results come back through sb_topdown_collect or sb_topdown_multiclass_collect with the instance model's
 * id (outputs as there, flags all zero), under their rules.  On a ground-truth pipeline sb_infer_topdown*,
 * sb_topdown_submit, sb_topdown_multiclass_submit and sb_topdown_attach_tracker are refused (SB_ERR_INVALID), and
 * sb_topdown_gt_submit is refused on a pipeline with a centroid model. */
int sb_topdown_gt_submit(sb_handle_t h, int instance_model_id, const uint8_t* frames_host, const float* centroids_host,
                         const int32_t* counts_host, int B, int slot);

/* ---- ground-truth instances ------------------------------------------------------------------------
 * sleap/nn/inference.py:1747-1966 CentroidCrop.call -> :812-893 FindInstancePeaksGroundTruth.call: the centroid stage of
 * sb_topdown_submit, then every kept centroid gets the labelled instance whose nearest visible node is closest to it, as
 * ONE device step with no instance model.  sb_topdown_gt_instances_configure: params.instance_model must be -1 and
 * params.centroid_model a configured model; `centroid`, `max_instances`, max_centroids_per_frame (K) and precrop_resize
 * as in sb_topdown_configure; `instance`, crop_size and max_crops_per_call are ignored.  The table holds up to
 * max_instances_per_frame (N) instances of n_nodes nodes per frame.  The pipeline belongs to the centroid model and is
 * addressed by its id; a configure call on that model drops the pipeline and its submitted batches.  It owns two slots of
 * max_batch uint8 frames of H x W x C_in and two instance tables, allocated at its first submit.
 * sb_topdown_gt_instances_submit queues one whole step into slot 0 / 1 without waiting on the host: the frames, the
 * instance table (B,N,n_nodes,2) (frame coordinates, float32, NaN allowed, rows past a frame's count ignored) and the
 * counts (B), each in [0, N], are copied on a copy stream; the centroid network, local peaks, (/ input_scale + 0.5) and
 * the per-frame top-k run as in sb_topdown_submit; then per centroid d[j] = min over the non-NaN nodes of sqrtf((x - cx)^2
 * + (y - cy)^2) in float32, each operation rounded on its own (NaN: an instance without a visible node).  A centroid
 * whose d is all NaN is dropped; otherwise it takes instance 0 unless a later one is strictly nearer (ties: the lower
 * index; an all-NaN instance 0 is kept).  The kept rows, in centroid order, carry the instance's points unchanged
 * (NaN included) with values 1.  Refused (SB_ERR_INVALID, nothing queued, the slot stays free): a count outside [0, N],
 * and as every streamed submit.
 * sb_topdown_gt_instances_collect, under the rules of the streamed steps: out_centroids (B,K,2), out_centroid_vals (B,K),
 * out_n_centroids (B), out_instance_peaks (B,K,n_nodes,2), out_instance_peak_vals (B,K,n_nodes), out_n_rows (B) (row i
 * is not centroid i: unmatched centroids have no row), out_flags (B) as sb_infer_topdown's; NaN padded.
 * On this pipeline sb_infer_topdown*, sb_topdown_submit / _collect, sb_topdown_gt_submit, sb_topdown_multiclass_*,
 * sb_topdown_attach_tracker and sb_topdown_tracks are refused (SB_ERR_INVALID); the other pipeline forms refuse these
 * two calls. */
int sb_topdown_gt_instances_configure(sb_handle_t h, const sb_topdown_params* params, int n_nodes, int max_instances_per_frame,
                                      int max_batch, int H, int W, int C_in);
int sb_topdown_gt_instances_submit(sb_handle_t h, int centroid_model_id, const uint8_t* frames_host, const float* instances_host,
                                   const int32_t* counts_host, int B, int slot);
int sb_topdown_gt_instances_collect(sb_handle_t h, int centroid_model_id, int slot, int B, float* out_centroids,
                                    float* out_centroid_vals, int32_t* out_n_centroids, float* out_instance_peaks,
                                    float* out_instance_peak_vals, int32_t* out_n_rows, int32_t* out_flags);

/* ---- top-down multi-class (identity) step ---------------------------------------------------------
 * sleap/nn/inference.py:4139-4210 TopDownMultiClassInferenceModel.call = CentroidCrop.call -> TopDownMultiClassFindPeaks.call
 * (:3863-4136), as ONE device pipeline: the sb_infer_topdown pipeline up to the instance network, then after every chunk
 * of crops the global peaks (+ crop offsets) and the class-vector head (ClassVectorsHead, sleap/nn/heads.py:431-460:
 * global max pool or Flatten of the tapped feature map -> num_fc_layers x (Dense + ReLU) -> Dense -> softmax), and after
 * the last chunk one SciPy assignment of the frame's crops to the classes on -probability per frame, a match kept only
 * where its probability is the crop's best (sleap/nn/identity.py:182-254 classify_peaks_from_vectors).
 * Head arithmetic (the definition, DESIGN.md 5.14): every unit is the float64 sum of (double)x_i * (double)W_ij in input
 * order plus (double)b_j, rounded once to float32, then ReLU; the softmax runs in float64 over the float32 logits
 * (max subtracted, exp, divided by the sum) and is rounded once to float32.  A split-precision tap [lo | hi | hi] is read
 * as float(lo) + float(hi), one fp32 add.
 * The tap is the feature map the head reads: op-list buffer, physical channel offset, its C channels, and planes (1, or 3
 * for the [lo | hi | hi] planes of a precision-2 fp16 tensor).  dense_weights: float32, Keras layout, packed in order
 * pre_classification{i}_fc kernel (n_in, num_fc_units) + bias for i < num_fc_layers, then the ClassVectorsHead kernel
 * (n_in, n_classes) + bias; n_in of the first layer is C with global_pool, else tap H * W * C (Flatten in H, W, C
 * order).  The weights are copied at configure time and owned by the pipeline.
 * Caps, checked at configure time (SB_ERR_UNSUPPORTED): n_classes <= SB_MAX_CLASSES; num_fc_units and, with global_pool,
 * the tap's C <= SB_MAX_DENSE_WIDTH (the vectors kept in shared memory; 33 KB at both caps, under the 48 KB every
 * device gives without opt-in).  A Flatten input is read from global memory and has no cap.
 * Outputs, class-indexed and NaN where no crop was assigned: out_points (B,n_classes,n_nodes,2), out_vals
 * (B,n_classes,n_nodes), out_class_probs (B,n_classes); then as sb_infer_topdown: out_centroids (B,K,2),
 * out_centroid_vals (B,K), out_n_valid (B) crops per frame, out_flags (B).  out_class_vectors (B,K,n_classes): every
 * crop's class probabilities in crop order, NaN padded (may be NULL).
 * sb_infer_topdown refuses a multi-class pipeline and sb_infer_topdown_multiclass a plain one; the chain rules of
 * sb_topdown_configure hold.  Instance models trained at an input scale != 1 are not covered: a precrop_resize other
 * than 0 or 1 is refused (SB_ERR_UNSUPPORTED). */
#define SB_MAX_DENSE_WIDTH 4096
typedef struct sb_topdown_multiclass_params {
  sb_topdown_params topdown;        /* as sb_topdown_configure */
  int32_t tap_buffer, tap_channel_offset, tap_channels, tap_planes;
  int32_t n_classes, num_fc_layers, num_fc_units, global_pool;
  const float* dense_weights;
  int64_t n_dense_weights;
} sb_topdown_multiclass_params;
int sb_topdown_multiclass_configure(sb_handle_t h, const sb_topdown_multiclass_params* params, int max_batch, int H, int W,
                                    int C_in);
int sb_infer_topdown_multiclass(sb_handle_t h, int centroid_model_id, const void* frames_host, int frames_are_u8, int B,
                                float* out_centroids, float* out_centroid_vals, float* out_points, float* out_vals,
                                float* out_class_probs, int32_t* out_n_valid, int32_t* out_flags, float* out_class_vectors);
/* The double-buffered form, with the rules of sb_topdown_submit / sb_topdown_collect; outputs as
 * sb_infer_topdown_multiclass (out_class_vectors may be NULL). */
int sb_topdown_multiclass_submit(sb_handle_t h, int centroid_model_id, const uint8_t* frames_host, int B, int slot);
/* model_id of sb_topdown_multiclass_collect: the pipeline's owner, as for sb_topdown_collect. */
int sb_topdown_multiclass_collect(sb_handle_t h, int model_id, int slot, int B, float* out_centroids,
                                  float* out_centroid_vals, float* out_points, float* out_vals, float* out_class_probs,
                                  int32_t* out_n_valid, int32_t* out_flags, float* out_class_vectors);
/* The same post-processing on caller-supplied crops (no network): confidence maps (n_crops,H,W,n_nodes), optional learned
 * offsets (n_crops,H,W,2*n_nodes), float32 feature maps (n_crops,Hf,Wf,Cf) read as the tap, optional crop offsets
 * (n_crops,2), crop_sample_inds (n_crops) non-decreasing in [0, B).  Uses params->topdown.instance and the head fields;
 * the model ids, the centroid stage and the tap fields are ignored.  Outputs as sb_infer_topdown_multiclass without the
 * centroids: out_points, out_vals, out_class_probs (B,...); out_class_vectors (n_crops,n_classes) and out_features
 * (n_crops, n_in of the first dense layer: the pooled or flattened feature vector) may be NULL. */
int sb_topdown_multiclass_from_features(sb_handle_t h, const sb_topdown_multiclass_params* params, const float* cms_host,
                                        int n_crops, int H, int W, int n_nodes, const float* offsets_host,
                                        const float* features_host, int Hf, int Wf, int Cf, const float* crop_offsets_host,
                                        const int32_t* crop_sample_inds, int B, float* out_points, float* out_vals,
                                        float* out_class_probs, float* out_class_vectors, float* out_features);

/* ---- flow shift for the optical-flow trackers ----------------------------------------------
 * sleap/nn/tracking.py:262-360 FlowCandidateMaker.flow_shift_instances = cv2.calcOpticalFlowPyrLK(prev, next,
 * pts, winSize=(window, window), maxLevel=max_levels, criteria=(EPS|COUNT, 30, 0.01)) on gray (cv2.COLOR_BGR2GRAY)
 * frames resized by img_scale.  A flow object keeps the image pyramids and Scharr derivatives of the last `ring`
 * frames on the device, keyed by frame index t, so that every frame's pyramid is built once however many later
 * frames shift points out of it.  Gray conversion, resize, pyramid and derivatives are bit-exact with OpenCV; the
 * LK iteration agrees with it to the size of its stopping step.
 *   window: 3..41; max_levels >= 0; img_scale: 1 or 0.5 (others return SB_ERR_UNSUPPORTED); ring >= 2, with no
 * upper cap: the ring's pyramids are one device allocation, sized at the first frame, and a ring the device cannot
 * hold fails there with SB_ERR_CUDA.
 * frame_host: uint8 (H, W, C), C = 1 or 3 (3 = BGR order, as the reference calls cvtColor).  A frame of another
 * size than the ring holds empties the ring.  replace = 0 keeps a frame already held under t and skips the upload.
 * When every slot is taken, the slot used least recently (added or read by a shift) is replaced.
 * sb_flow_shift: point i (pts[2i], pts[2i+1], in the resized frame's pixels) moves from frame ref_t[i] into frame t.
 * out_status[i] = 1 when found; out_err[i] = mean |J - I| over the window (defined where found).  A frame index that
 * is not held returns SB_ERR_INVALID.  One upload, one launch and one download.
 * sb_flow_fetch_level: level `level` of frame t: img_out (H, W) uint8, deriv_out (H, W, 2) int16 (dx, dy); either
 * may be NULL; *out_n_levels = levels built (maxLevel actually used + 1). */
int sb_flow_create(sb_handle_t h, int window, int max_levels, float img_scale, int ring, int* out_flow_id);
int sb_flow_add_frame(sb_handle_t h, int flow_id, int64_t t, const uint8_t* frame_host, int H, int W, int C,
                      int replace);
int sb_flow_shift(sb_handle_t h, int flow_id, int64_t t, int n, const int64_t* ref_t, const float* pts,
                  float* out_pts, int32_t* out_status, float* out_err);
int sb_flow_fetch_level(sb_handle_t h, int flow_id, int64_t t, int level, uint8_t* img_out, int16_t* deriv_out,
                        int* out_H, int* out_W, int* out_n_levels);
int sb_flow_destroy(sb_handle_t h, int flow_id);

/* ---- identity tracker on the device ----------------------------------------------------------
 * sleap/nn/tracking.py:542-844 Tracker.track with the simple / simple-max-tracks candidate makers, one call per frame,
 * replayed frame by frame by one CTA (k_track): pre-cull (target_instance_count + nms_fast), candidate pool,
 * similarity matrix (float64), robust per-track reduction (max or np.quantile), greedy or Hungarian matching, new
 * tracks, and the track_window queues, which stay on the device between calls.
 * Tie rules: greedy visits pairs in np.argsort(cost, kind="stable") order (ascending flat index among equal costs);
 * nms_fast orders equal instance scores by ascending index.  The host's default sorts leave these orders
 * implementation-defined.
 * Capacities (checked at create, SB_ERR_INVALID): max_instances 1..128 per frame, n_nodes 1..64, track_window 1..64,
 * track_table 1..65536 (simple-max-tracks: the per-track queues; max_tracking requires track_table >= max_tracks).
 * sb_track_instances: points (B, I, n_nodes, 2), point confidences (B, I, n_nodes), scores (B, I), counts (B),
 * img_hw (B, 2) (normalized_instance only; may be NULL otherwise), t (B) frame indices (t < 0: the host's _next_t).
 * Per frame b the output lists the tracked instances in Tracker.track's order: out_index (B, I) index into the input,
 * out_track (B, I) track id in spawn order (name track_{id}), out_score (B, I) tracking score (-cost; 0 for a new
 * track), out_matched (B, I) 1 when matched, out_n (B), out_t (B) the frame index used.  *out_n_done = frames
 * tracked; *out_flag = SB_TRACK_INFEASIBLE when the Hungarian matcher met a matrix SciPy rejects (frame *out_n_done,
 * left untracked, state as before it).  A count above I, or a max-tracks queue table that would grow past
 * track_table, returns SB_ERR_INVALID; the frames before it are tracked (*out_n_done). */
#define SB_TRACK_SIMPLE 0
#define SB_TRACK_SIMPLE_MAX_TRACKS 1
#define SB_TRACK_SIM_INSTANCE 0
#define SB_TRACK_SIM_NORMALIZED_INSTANCE 1
#define SB_TRACK_SIM_OBJECT_KEYPOINT 2
#define SB_TRACK_SIM_CENTROID 3
#define SB_TRACK_SIM_IOU 4
#define SB_TRACK_MATCH_GREEDY 0
#define SB_TRACK_MATCH_HUNGARIAN 1
#define SB_TRACK_OKS_ALL 0
#define SB_TRACK_OKS_REF 1
#define SB_TRACK_OKS_UNION 2
#define SB_TRACK_INFEASIBLE 1
#define SB_TRACK_OVER_CAPACITY 3
typedef struct sb_tracker_params {
  int32_t maker, similarity, match;         /* SB_TRACK_* */
  int32_t track_window;
  int32_t max_tracks, max_tracking;         /* max_tracks <= 0: none */
  int32_t min_match_points, min_new_track_points;
  double robust;                            /* 0 < robust < 1: np.quantile, else max */
  int32_t cull_target;                      /* target_instance_count when pre_cull_to_target, else 0 */
  int32_t cull_use_iou;                     /* pre_cull_iou_threshold given and nonzero */
  double cull_iou_threshold;
  const double* oks_errors;                 /* NULL / n_oks_errors = 0: 1 */
  int32_t n_oks_errors;
  int32_t oks_score_weighting, oks_normalization;
  int32_t n_nodes, max_instances, track_table;
} sb_tracker_params;
int sb_tracker_create(sb_handle_t h, const sb_tracker_params* params, int* out_tracker_id);
int sb_tracker_reset(sb_handle_t h, int tracker_id);
int sb_tracker_destroy(sb_handle_t h, int tracker_id);
int sb_track_instances(sb_handle_t h, int tracker_id, int B, int I, const double* points, const double* point_conf,
                       const double* scores, const int32_t* counts, const double* img_hw, const int64_t* t,
                       int32_t* out_index, int32_t* out_track, double* out_score, int32_t* out_matched,
                       int32_t* out_n, int64_t* out_t, int32_t* out_n_done, int32_t* out_flag);
/* The tracker inside the bottom-up step.  sb_bottomup_attach_tracker(tracker_id = -1 detaches): every later
 * sb_infer_bottomup / sb_infer_bottomup_dev / sb_bottomup_submit call runs k_track on the post-processing stream right
 * after the grouping kernel, on the instance list Predictor._frames_from_example builds from each frame (all-NaN rows
 * skipped; max_instances >= 0: the top scores, stable), with the frame size img_h x img_w (normalized_instance) and
 * t = the host's _next_t.  The tracker must live on the model's handle, have its n_nodes and at least its
 * max_instances, and the record exchange must not be connected (one rank).  The per-frame track records
 * ([B][2 + 3 I] doubles, I = the tracker's max_instances: n, flag, order[I] (index into that instance list), track
 * id[I], tracking score[I]; flag != 0: the frame was not tracked -- SB_TRACK_INFEASIBLE, 2 = queue table full, or
 * SB_TRACK_OVER_CAPACITY, which only the top-down step can meet)
 * are a separate buffer: the result records and record_width do not change.  They come back with the result copy:
 * sb_bottomup_tracks(slot 0 / 1, as every slot read; slot 0 after sb_infer_bottomup); sb_bottomup_device_tracks
 * copies the last step's records after sb_infer_bottomup_dev. */
int sb_bottomup_attach_tracker(sb_handle_t h, int model_id, int tracker_id, int max_instances, double img_h, double img_w);
int sb_bottomup_tracks(sb_handle_t h, int model_id, int slot, int B, double* out_tracks);
int sb_bottomup_device_tracks(sb_handle_t h, int model_id, int B, double* out_tracks);
/* The tracker inside the top-down step.  sb_topdown_attach_tracker(tracker_id = -1 detaches): every later
 * sb_infer_topdown call runs k_track on the handle's stream after the record kernel, on the instance list
 * Predictor._frames_from_example builds from each frame of a top-down batch: the frame's crops in order, rows whose
 * points are all NaN skipped, score = the centroid value, no max_instances cut; with the frame size img_h x img_w
 * (normalized_instance) and t = the host's _next_t.  A frame whose list is longer than the tracker's max_instances
 * stops the batch's tracking there: its record and every later one carry flag SB_TRACK_OVER_CAPACITY, which stays set
 * until sb_tracker_reset (as a full queue table does).  The pipeline must be a plain one (sb_topdown_configure), and the
 * tracker must live on its handle and have its instance model's node count; img_h, img_w > 0.  The attachment lives
 * with the pipeline: a configure call on either model drops it.  sb_infer_topdown's outputs do not change.  Streamed
 * batches are tracked in submit order.  sb_topdown_tracks copies track records in the bottom-up format above, as
 * sb_bottomup_tracks does: those of the batch last collected from slot 0 / 1 (slot 0 after sb_infer_topdown; B must be
 * that batch's frame count). */
int sb_topdown_attach_tracker(sb_handle_t h, int centroid_model_id, int tracker_id, double img_h, double img_w);
int sb_topdown_tracks(sb_handle_t h, int centroid_model_id, int slot, int B, double* out_tracks);

#ifdef __cplusplus
}
#endif
#endif /* SLEAP_B200_H_ */
