// Shared definitions for libsleapb200 (sm_90a).  Internal header; the public C-ABI is
// include/sleap_b200.h.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <string>
#include <vector>

#include "../../include/sleap_b200.h"

struct SbModel;
struct SbFlow;
struct SbTracker;

// Device workspace for the post-processing stages (capacity-bounded, per sample).
struct SbPostWs {
  int B = 0, H = 0, W = 0, C = 0;          // confidence-map shape the workspace was sized for
  int rows_per_chunk = 0, n_chunks = 0, chunk_cap = 0;
  int max_peaks = 0, max_node_peaks = 0, max_instances = 0, n_edges = 0;
  bool node_lists = false;                  // k_local_emit builds node_cnt / node_peaks (PAF matching, class grouping)
  // local peaks
  int* chunk_cnt = nullptr;                 // [B][n_chunks]
  uint2* chunk_items = nullptr;             // [B][n_chunks][chunk_cap]  (flat idx, val bits)
  float* peaks = nullptr;                   // [B][max_peaks][2]   (x, y) already scaled
  float* peak_vals = nullptr;               // [B][max_peaks]
  int* peak_ch = nullptr;                   // [B][max_peaks]
  int* n_peaks = nullptr;                   // [B]
  int* total_peaks = nullptr;               // [B]   (uncapped count)
  int* node_cnt = nullptr;                  // [B][C]  (uncapped count per node)
  int* node_peaks = nullptr;                // [B][C][max_node_peaks]  peak index within sample
  // scoring / matching
  float* score_mat = nullptr;               // [B][E][K*K]
  int* match_cnt = nullptr;                 // [B][E]
  int* match_src = nullptr;                 // [B][E][K]
  int* match_dst = nullptr;                 // [B][E][K]
  float* match_score = nullptr;             // [B][E][K]
  // grouping output
  float* inst_peaks = nullptr;              // [B][max_instances][C][2]
  float* inst_vals = nullptr;               // [B][max_instances][C]
  float* inst_scores = nullptr;             // [B][max_instances]
  int* n_inst = nullptr;                    // [B]
  int* flags = nullptr;                     // [B]  overflow bit flags
  // contiguous per-frame result records written by the grouping kernel's epilogue:
  // [B][I*C*2 peaks | I*C vals | I scores | n_valid | flags]  (sb_record_width floats per frame),
  // or by k_class_group: [B][sb_class_record_width floats]
  float* records = nullptr;
  uint2* sorted_items = nullptr;            // [B][max_peaks]  scanned items in tf.where order (k_local_emit scratch)
  int* edges_dev = nullptr;                 // [E][2]
  int* sorted_edges_dev = nullptr;          // [n_sorted]
  int n_sorted = 0;
  size_t bytes = 0;
};

// ---- peer-memory record exchange (sb_gather.cu; pushed from k_group's epilogue) ----
#define SB_GATHER_MAX_WORLD 8
#define SB_GATHER_TIMEOUT_ARRIVE 1
#define SB_GATHER_TIMEOUT_ACK 2
struct SbGatherDev {                        // by-value kernel argument: one step's view of the exchange
  int on, rank, world, G, Bmax;
  size_t width;
  unsigned long long step, timeout_ns;
  float* data[SB_GATHER_MAX_WORLD];               // every rank's window (own rank: local memory, others: NVLink peer mappings)
  unsigned long long* arrive[SB_GATHER_MAX_WORLD];
  unsigned long long* ack[SB_GATHER_MAX_WORLD];
  unsigned int* done;
  int* status;
};
struct SbGather {
  int rank = 0, world = 0, G = 0, Bmax = 0;
  size_t width = 0;
  void* local = nullptr;
  void* peer[SB_GATHER_MAX_WORLD] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  bool connected = false;
  long long step = 0;                              // steps pushed so far
  long long consumed = 0;                          // steps acknowledged so far (acks are cumulative)
  unsigned long long timeout_ns = 0;
  int *status_host = nullptr, *status_dev = nullptr, *counts_host = nullptr, *counts_dev = nullptr;
};

static __host__ __device__ inline size_t sb_record_width(int max_instances, int n_nodes) {
  // peaks | values | scores | n_valid | flags, padded to a multiple of 4 floats (16-byte rows for vector copies)
  return (((size_t)max_instances * n_nodes * 3 + max_instances + 2) + 3) & ~(size_t)3;
}
static __host__ __device__ inline size_t sb_class_record_width(int n_classes, int n_nodes) {
  // points [n_classes][n_nodes][2] | values [n_classes][n_nodes] | class probabilities [n_classes][n_nodes] | flags,
  // padded to a multiple of 4 floats
  return (((size_t)n_classes * n_nodes * 4 + 1) + 3) & ~(size_t)3;
}

struct sb_handle_s {
  int device = 0;
  cudaStream_t stream = nullptr;       // stream all work is issued on
  cudaStream_t own_stream = nullptr;   // created by sb_create
  cudaStream_t aux_stream[3] = {nullptr, nullptr, nullptr};  // fork/join branches (tconv phases)
  cudaEvent_t fork_ev = nullptr, join_ev[3] = {nullptr, nullptr, nullptr};
  // post-processing of step i runs on its own stream so that it overlaps the network of step i+1
  cudaStream_t post_stream = nullptr;
  cudaEvent_t fwd_done_ev = nullptr, post_done_ev = nullptr;
  bool post_pending = false;
  std::string last_error;
  std::vector<void*> owned;                 // generic device allocations freed at destroy
  std::vector<SbModel*> models;
  std::vector<SbFlow*> flows;               // sb_flow_create objects (sb_flow.cu); index = flow id
  std::vector<SbTracker*> trackers;         // sb_tracker_create objects (sb_track.cu); index = tracker id
  int gpu_launches = 0;                     // kernels launched by this handle (bench: gpu_launches)
  int sm_count = 132;
};

extern thread_local std::string g_sb_last_error;

int sb_fail(sb_handle_s* h, int code, const char* fmt, ...);
void sb_models_free(sb_handle_s* h);
void sb_flows_free(sb_handle_s* h);
void sb_trackers_free(sb_handle_s* h);
// ---- device tracker (sb_track.cu) inside the bottom-up and top-down steps ----
SbTracker* sb_tracker_get(sb_handle_s* h, int id);
int sb_tracker_max_instances(const SbTracker* t);
int sb_tracker_nodes(const SbTracker* t);
static __host__ __device__ inline size_t sb_track_record_width(int I) { return 2 + 3 * (size_t)I; }
// k_track on the grouping output of a batch (ws.inst_*), then one track record per frame into out_records
int sbk_track_step(sb_handle_s* h, SbTracker* tr, int B, const float* inst_peaks, const float* inst_vals,
                   const float* inst_scores, const int* n_inst, int I_src, int max_instances, double img_h, double img_w,
                   double* out_records);
// k_track on the crops of a top-down batch (points / values per crop, centroid values [B][K], crops per frame and
// their frame offsets), then one track record per frame into out_records
int sbk_track_topdown(sb_handle_s* h, SbTracker* tr, int B, const float* ipts, const float* ivals, const float* sel_val,
                      const int* sel_count, const int* offsets, int K, double img_h, double img_w, double* out_records);

#define SB_CUDA(h, expr)                                                              \
  do {                                                                                \
    cudaError_t _e = (expr);                                                          \
    if (_e != cudaSuccess)                                                            \
      return sb_fail((h), SB_ERR_CUDA, "%s failed: %s (%s:%d)", #expr,               \
                     cudaGetErrorString(_e), __FILE__, __LINE__);                     \
  } while (0)

#define SB_CHECK_LAUNCH(h) do { (h)->gpu_launches++; SB_CUDA((h), cudaGetLastError()); } while (0)

template <typename T>
static inline int sb_dev_alloc(sb_handle_s* h, T** p, size_t n) {
  void* q = nullptr;
  cudaError_t e = cudaMalloc(&q, n * sizeof(T) + 16);
  if (e != cudaSuccess) return sb_fail(h, SB_ERR_CUDA, "cudaMalloc(%zu) failed: %s", n * sizeof(T), cudaGetErrorString(e));
  *p = (T*)q;
  return 0;
}

// ---- post-processing launchers (sb_post.cu) ----
struct SbPeakParams {
  float threshold;
  int refinement;      // SB_REFINE_*
  int patch;           // integral patch size (odd)
  float scale;         // multiply refined peaks (cm output stride); 1 for the stage-level API
  float input_scale;   // != 1: then / input_scale + 0.5 (centroid / single-instance paths)
};

// Confidence maps (and learned offsets) are fp32 NHWC: head outputs are always fp32.
int sbk_local_peaks(sb_handle_s* h, const float* cms, const float* offsets, int B, int H, int W, int C,
                    const SbPeakParams& p, SbPostWs& ws);
int sbk_global_peaks(sb_handle_s* h, const float* cms, const float* offsets, int B, int H, int W, int C, const SbPeakParams& p,
                     const float* crop_off_dev, float* part_buf, int n_chunks, int rows_per_chunk,
                     float* out_points, float* out_vals);
int sbk_score_match(sb_handle_s* h, const float* pafs, int B, int Hp, int Wp, int C2,
                    int n_points, int pafs_stride, float max_edge_length, float dist_penalty_weight,
                    SbPostWs& ws);
int sbk_group(sb_handle_s* h, int B, int n_nodes, int min_instance_peaks, float min_line_scores,
              float input_scale, SbPostWs& ws, const SbGatherDev* gather = nullptr);
// identity grouping of the multi-class step on ws's per-node peak lists and the class-map logits (B,Hc,Wc,n_classes):
// one record per frame into ws.records (sb_class_record_width); ws must have node_lists and records
int sbk_class_group(sb_handle_s* h, const float* class_maps, int B, int Hc, int Wc, int n_classes, float class_stride,
                    float input_scale, SbPostWs& ws);
// Dynamic shared memory of k_score_match, k_group and k_class_group: the launchers size their launches by these, and
// the chains' configure calls refuse (SB_ERR_UNSUPPORTED) a max_node_peaks / n_classes whose kernels would not fit in
// the device's opt-in shared memory per block, so a configured chain never fails a step at launch.
size_t sb_score_match_smem(int K);
size_t sb_group_smem(int n_nodes, int n_edges, int K);
size_t sb_class_group_smem(int K, int n_classes);
int sb_check_paf_smem(sb_handle_s* h, int n_nodes, int n_edges, int K);
int sb_check_class_smem(sb_handle_s* h, int K, int n_classes);
int sbk_lsap_batch(sb_handle_s* h, const float* scores, const int* n_src, const int* n_dst,
                   const int* offsets, int n_problems, int max_k, int* out_rows, int* out_cols,
                   float* out_scores, int* out_counts);
int sbk_crop(sb_handle_s* h, const void* images, int img_is_u8, int B, int H, int W, int C,
             const float* centroids, const int* sample_inds, int n, int crop_h, int crop_w,
             void* out, int out_is_u8_trunc);
// The size resize_image gives H x W frames at `scale`: int(float32(H) * scale) x int(float32(W) * scale), as sb_net_size
// and FrameResizer compute it.  Nonzero (no size) when scale is not finite and positive or an extent is below 1.
static inline int sb_resized_size(int H, int W, float scale, int* Hr, int* Wr) {
  const float fh = (float)H * scale, fw = (float)W * scale;
  if (!(scale > 0.f) || !(fh >= 1.f && fh < 2147483648.f) || !(fw >= 1.f && fw < 2147483648.f)) return 1;
  *Hr = (int)fh;
  *Wr = (int)fw;
  return 0;
}
// sbk_crop of the frames resized to Hr x Wr (resize_image, uint8 frames cast back by truncation) without storing them;
// centroids in resized-frame coordinates
int sbk_crop_resized(sb_handle_s* h, const void* images, int img_is_u8, int B, int H, int W, int C, int Hr, int Wr,
                     const float* centroids, const int* sample_inds, int n, int crop_h, int crop_w, void* out);

int sbk_lines(sb_handle_s* h, const float* pafs, int Hp, int Wp, int C2, const float* lines_in,
              const float* peaks, const int* edge_peak_inds, const int* edge_inds, int n, int P,
              float pafs_stride, float max_edge_length, float dist_w, int* out_subs, float* out_lines,
              float* out_scores);
int sbk_integral(sb_handle_s* h, const float* cms, int N, int Hh, int Ww, int C, const float* xv,
                 const float* yv, float* x_hat, float* y_hat);
int sbk_local_dir(sb_handle_s* h, const float* patches, int N, float delta, float* out);

int sb_post_ws_alloc(sb_handle_s* h, SbPostWs& ws, int B, int H, int W, int C, int max_peaks,
                     int max_node_peaks, int max_instances, int n_edges);
void sb_post_ws_free(SbPostWs& ws);

// Global-peak scratch for B frames of (H, C) maps: the partial maxima of ceil(2 * SMs / B) row chunks per frame, the
// points, values and crop offsets (sb_model.cu)
struct SbGlobalScratch {
  float *part = nullptr, *points = nullptr, *vals = nullptr, *crop_off = nullptr;
  int rpc = 1, chunks = 1;   // rows per chunk of the partial maxima, chunks per frame
};
int sb_global_scratch_alloc(sb_handle_s* h, SbGlobalScratch& g, int B, int H, int C);
void sb_global_scratch_free(SbGlobalScratch& g);

// Copies the peak lists of ws's first B frames into caller arrays, concatenated in frame order: points, values, channel
// indices (NULL: not wanted) and frame indices; per-frame flags (NULL: not wanted); *out_n = the number of peaks (sb_api.cu)
int sb_peaks_to_host(sb_handle_s* h, const SbPostWs& ws, int B, float* out_points, float* out_vals, int32_t* out_channel_inds,
                     int32_t* out_sample_inds, int32_t* out_n, int32_t* out_flags);

// Host copies of ws's per-frame PAF candidates (sb_model.cu): peak counts [B], node counts [B][C], node lists [B][C][K]
// and score matrices [B][E][K*K].  sb_graph_download needs the work that wrote them finished.
struct SbGraphHost {
  std::vector<int> n_peaks, node_cnt, node_peaks;
  std::vector<float> score_mat;
};
int sb_graph_download(sb_handle_s* h, const SbPostWs& ws, int B, SbGraphHost& g);
// The candidates in (frame, edge, src, dst) order: edge index, (src, dst) peak indices within the frame and line score each;
// cand_offsets[B + 1] the first candidate of every frame
int sb_graph_flatten(sb_handle_s* h, const SbPostWs& ws, const SbGraphHost& g, const int* edges_host, int B, int cap,
                     int32_t* edge_inds, int32_t* edge_peak_inds, float* line_scores, int32_t* cand_offsets);

// The scratch of a call that takes or returns caller (host) arrays, freed when the call returns: a post-processing
// workspace, a global-peak scratch and device buffers.  Copies are queued on the handle's stream.
struct SbScratch {
  sb_handle_s* h;
  SbPostWs ws;
  SbGlobalScratch gs;
  std::vector<void*> bufs;
  explicit SbScratch(sb_handle_s* handle) : h(handle) {}
  SbScratch(const SbScratch&) = delete;
  SbScratch& operator=(const SbScratch&) = delete;
  ~SbScratch() {
    sb_post_ws_free(ws);
    sb_global_scratch_free(gs);
    for (void* q : bufs) cudaFree(q);
  }
  template <typename T> int alloc(T** dev, size_t n) {      // a device buffer of n elements
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, n * sizeof(T) + 16);
    if (e != cudaSuccess) return sb_fail(h, SB_ERR_CUDA, "cudaMalloc(%zu): %s", n * sizeof(T), cudaGetErrorString(e));
    bufs.push_back(q);
    *dev = (T*)q;
    return 0;
  }
  // a device copy of n elements of `host`; an optional input that is NULL: *dev = NULL
  template <typename T> int upload(const T* host, size_t n, const T** dev, bool optional = false) {
    *dev = nullptr;
    T* q;
    if (optional && !host) return 0;
    if (const int rc = alloc(&q, n)) return rc;
    *dev = q;
    return to_dev(q, host, n);
  }
  template <typename T> int to_dev(T* dev, const T* host, size_t n) {
    SB_CUDA(h, cudaMemcpyAsync(dev, host, n * sizeof(T), cudaMemcpyHostToDevice, h->stream));
    return 0;
  }
  // an optional output that is NULL: nothing
  template <typename T> int to_host(T* host, const T* dev, size_t n, bool optional = false) {
    if (!optional || host) SB_CUDA(h, cudaMemcpyAsync(host, dev, n * sizeof(T), cudaMemcpyDeviceToHost, h->stream));
    return 0;
  }
  int sync() {
    SB_CUDA(h, cudaStreamSynchronize(h->stream));
    return 0;
  }
};

// Splits B fixed-width per-frame records into caller arrays: the float fields in record order (destination, floats per
// frame), then one float per frame for each int field, cast to int32.  A NULL destination skips its field (sb_model.cu).
struct SbRecField {
  float* dst;
  size_t n;
};
void sb_split_records(const float* rec, int B, size_t width, std::initializer_list<SbRecField> floats,
                      std::initializer_list<int32_t*> ints);

// ---- frame preprocessing shared by k_preprocess, the fused first-layer / stem view kernels and the resized crops ----
// Pixel (oy, ox) of an Hin x Win image resized to Hres x Wres: bilinear, half-pixel centres, no antialias
// (tf.image.resize); fetch(y, x) is one source texel as a float.  Explicitly rounded, so that every caller computes the
// same value whatever the contraction setting of its file.
template <typename Fetch>
__device__ __forceinline__ float sb_resize_sample(const Fetch& fetch, int oy, int ox, int Hin, int Win, int Hres, int Wres) {
  const float scy = (float)Hin / (float)Hres, scx = (float)Win / (float)Wres;
  const float sy = __fadd_rn(__fmul_rn(__fadd_rn((float)oy, 0.5f), scy), -0.5f);
  const float sx = __fadd_rn(__fmul_rn(__fadd_rn((float)ox, 0.5f), scx), -0.5f);
  const float fy = floorf(sy), fx = floorf(sx);
  const int y0 = max((int)fy, 0), y1 = min((int)ceilf(sy), Hin - 1);
  const int x0 = max((int)fx, 0), x1 = min((int)ceilf(sx), Win - 1);
  const float ly = __fsub_rn(sy, fy), lx = __fsub_rn(sx, fx);
  const float tl = fetch(y0, x0), tr = fetch(y0, x1), bl = fetch(y1, x0), br = fetch(y1, x1);
  const float tp = __fadd_rn(tl, __fmul_rn(__fadd_rn(tr, -tl), lx));
  const float bt = __fadd_rn(bl, __fmul_rn(__fadd_rn(br, -bl), lx));
  return __fadd_rn(tp, __fmul_rn(__fadd_rn(bt, -tp), ly));
}
// caffe mean of BGR channel c (resnet.py imagenet_preproc_v1)
__device__ __forceinline__ float sb_imagenet_caffe_mean(int c) { return c == 0 ? 103.939f : (c == 1 ? 116.779f : 123.68f); }
// ensure_grayscale of one RGB pixel as a [0, 1] float (u8: truncating round trip like tf.image.rgb_to_grayscale)
template <typename TI>
__device__ __forceinline__ float sb_gray_pre(const TI* p, int in_is_u8) {
  const float sc = in_is_u8 ? (1.0f / 255.0f) : 1.0f;
  const float g = __fadd_rn(__fadd_rn(__fmul_rn(__fmul_rn((float)p[0], sc), 0.2989f),
                                      __fmul_rn(__fmul_rn((float)p[1], sc), 0.5870f)),
                            __fmul_rn(__fmul_rn((float)p[2], sc), 0.1140f));
  return in_is_u8 ? __fmul_rn(truncf(fminf(fmaxf(__fmul_rn(g, 255.5f), 0.f), 255.f)), 1.0f / 255.0f) : g;
}
