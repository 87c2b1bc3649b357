// Fused top-down pipeline on the device: frames -> centroid network -> local peaks -> per-frame top-k ->
// crops of the RESIDENT frames -> centered-instance network -> global peaks (+ crop offsets) -> dense per-frame record.
// One H2D copy of the frames and one D2H copy of the results per batch (+ a 4-byte crop count).
// The multi-class (identity) form runs the class-vector head after every chunk's global peaks (k_class_vectors) and, after
// the last chunk, one assignment of each frame's crops to the classes (k_td_class_assign) in place of k_td_pack.
//
// Reference: TopDownInferenceModel.call (sleap/nn/inference.py:2273-2311) = CentroidCrop.call (:1747-1966: network,
// find_local_peaks, /input_scale + 0.5, tf.math.top_k(max_instances) :1879-1894, crop_bboxes on the full frames :1918-1927)
// followed by FindInstancePeaks.call (:2059-2200: network on the crops, find_global_peaks, + crop_offsets);
// TopDownMultiClassInferenceModel.call (:4139-4210) with TopDownMultiClassFindPeaks.call (:3863-4136), ClassVectorsHead
// (sleap/nn/heads.py:431-460) and classify_peaks_from_vectors (sleap/nn/identity.py:182-254).
// Round 1 ran these as separate host-facing calls: centroids D2H -> host top-k -> frames H2D again -> crops D2H ->
// crops H2D -> instance network (sleap_b200/nn/inference.py CentroidCrop / FindInstancePeaks, kept for the stage-level
// surface).  A pre-crop resize (CentroidCrop.precrop_resize, :1836-1843) scales the kept centroids in k_td_select and cuts
// the crops from the resident frames resized on the fly (sbk_crop_resized).
// Ground-truth centroids (CentroidCropGroundTruth.call, :743-809; centroid_model = -1): the host's centroid table stands
// in for the centroid stage (k_td_gt_select), and the rest of the step is the same instance stage.  The crop count is
// known on the host, so sb_topdown_gt_submit queues a whole step without a mid-step synchronise.
//
// The head's float64 sums use __dmul_rn / __dadd_rn: this file is built with multiply-add contraction on, and a fused
// product would round differently from the definition (include/sleap_b200.h).
#include <algorithm>
#include <limits>

#include <math_constants.h>

#include "sb_common.cuh"
#include "sb_lsap.cuh"
#include "sb_model.h"

namespace {

// Per frame: keep all centroids in tf.where order, or -- more than max_instances -- the max_instances most confident ones
// in tf.math.top_k order (descending value, ties: lower index first).  K = capacity of the dense outputs.  The kept
// centroids are multiplied by the pre-crop resize `scale` (1: unchanged), rounded on its own: the crop offsets subtract
// half the crop size from the product.
__global__ void __launch_bounds__(128) k_td_select(const float* __restrict__ peaks, const float* __restrict__ peak_vals,
                                                   const int* __restrict__ n_peaks, int max_peaks, int max_instances, int K, float scale,
                                                   float* __restrict__ sel_cent, float* __restrict__ sel_val, int* __restrict__ sel_count,
                                                   int* __restrict__ flags) {
  const int b = blockIdx.x;
  const int n = n_peaks[b];
  const float* pk = peaks + (size_t)b * max_peaks * 2;
  const float* pv = peak_vals + (size_t)b * max_peaks;
  const bool topk = max_instances > 0 && max_instances < n;
  const int keep = topk ? max_instances : n;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    int pos = i;
    if (topk) {
      const float v = pv[i];
      int rank = 0;
      for (int j = 0; j < n; ++j) rank += (pv[j] > v || (pv[j] == v && j < i)) ? 1 : 0;
      pos = rank;
    }
    if (pos < keep && pos < K) {
      sel_cent[((size_t)b * K + pos) * 2] = __fmul_rn(pk[2 * i], scale);
      sel_cent[((size_t)b * K + pos) * 2 + 1] = __fmul_rn(pk[2 * i + 1], scale);
      sel_val[(size_t)b * K + pos] = pv[i];
    }
  }
  if (threadIdx.x == 0) {
    sel_count[b] = min(keep, K);
    if (keep > K) atomicOr(&flags[b], SB_FLAG_INSTANCES_TRUNCATED);
  }
}

// Ground-truth centroids (CentroidCropGroundTruth.call, :743-809): the first count[b] rows of frame b's K-row table (the
// host checked count <= K), multiplied by the pre-crop resize `scale` (1: unchanged) with one explicitly rounded
// multiply, as the layer's float32 multiply; value 1; no top-k, so no truncation flag.
__global__ void __launch_bounds__(128) k_td_gt_select(const float* __restrict__ table, const int* __restrict__ count, int K, float scale,
                                                      float* __restrict__ sel_cent, float* __restrict__ sel_val, int* __restrict__ sel_count,
                                                      int* __restrict__ flags) {
  const int b = blockIdx.x;
  const int n = count[b];
  const size_t o = (size_t)b * K;
  for (int i = threadIdx.x; i < 2 * n; i += blockDim.x) sel_cent[2 * o + i] = __fmul_rn(table[2 * o + i], scale);
  for (int i = threadIdx.x; i < n; i += blockDim.x) sel_val[o + i] = 1.f;
  if (threadIdx.x == 0) {
    sel_count[b] = n;
    flags[b] = 0;
  }
}

// Flat crop list in (frame, slot) order + crop offsets (centroid - crop_size / 2, :1911).
__global__ void __launch_bounds__(256) k_td_flatten(const float* __restrict__ sel_cent, const int* __restrict__ sel_count, int B, int K,
                                                    float half_crop, float* __restrict__ flat_cent, float* __restrict__ flat_off,
                                                    int* __restrict__ flat_sample, int* __restrict__ offsets, int* __restrict__ total) {
  __shared__ int s_off[1025];
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int b = 0; b < B; ++b) { s_off[b] = acc; acc += sel_count[b]; }
    s_off[B] = acc;
    *total = acc;
  }
  __syncthreads();
  for (int b = threadIdx.x; b <= B; b += blockDim.x) offsets[b] = s_off[b];
  for (int t = threadIdx.x; t < B * K; t += blockDim.x) {
    const int b = t / K, k = t - b * K;
    if (k >= sel_count[b]) continue;
    const int f = s_off[b] + k;
    const float x = sel_cent[2 * (size_t)t], y = sel_cent[2 * (size_t)t + 1];
    flat_cent[2 * f] = x; flat_cent[2 * f + 1] = y;
    flat_off[2 * f] = x - half_crop; flat_off[2 * f + 1] = y - half_crop;
    flat_sample[f] = b;
  }
}

// The frame's K centroid slots of a record: [K][2] centroids | [K] values, NaN past the frame's count (sel_cent NULL: all NaN)
__device__ void td_write_centroids(const float* __restrict__ sel_cent, const float* __restrict__ sel_val, int b, int cnt, int K,
                                   float* __restrict__ rc) {
  float* rv = rc + K * 2;
  for (int t = threadIdx.x; t < K * 2; t += blockDim.x) rc[t] = (sel_cent && t / 2 < cnt) ? sel_cent[(size_t)b * K * 2 + t] : CUDART_NAN_F;
  for (int t = threadIdx.x; t < K; t += blockDim.x) rv[t] = (sel_val && t < cnt) ? sel_val[(size_t)b * K + t] : CUDART_NAN_F;
}

// Dense per-frame record: [K][2] centroids | [K] centroid values | [K][nodes][2] peaks | [K][nodes] peak values | n_valid | flags
__global__ void __launch_bounds__(128) k_td_pack(const float* __restrict__ sel_cent, const float* __restrict__ sel_val,
                                                 const int* __restrict__ sel_count, const int* __restrict__ offsets,
                                                 const float* __restrict__ ipts, const float* __restrict__ ivals, int K, int nodes,
                                                 const int* __restrict__ flags, float* __restrict__ record, int width) {
  const int b = blockIdx.x;
  const int cnt = sel_count[b], o = offsets[b];
  float* r = record + (size_t)b * width;
  float* rp = r + K * 3;
  float* rq = rp + (size_t)K * nodes * 2;
  td_write_centroids(sel_cent, sel_val, b, cnt, K, r);
  for (int t = threadIdx.x; t < K * nodes * 2; t += blockDim.x) {
    const int k = t / (nodes * 2);
    rp[t] = (k < cnt) ? ipts[(size_t)(o + k) * nodes * 2 + (t - k * nodes * 2)] : CUDART_NAN_F;
  }
  for (int t = threadIdx.x; t < K * nodes; t += blockDim.x) {
    const int k = t / nodes;
    rq[t] = (k < cnt) ? ivals[(size_t)(o + k) * nodes + (t - k * nodes)] : CUDART_NAN_F;
  }
  if (threadIdx.x == 0) {
    rq[(size_t)K * nodes] = (float)cnt;
    rq[(size_t)K * nodes + 1] = (float)flags[b];
  }
}

// Ground-truth instances (FindInstancePeaksGroundTruth.call, :812-893), one CTA per frame: every selected centroid gets
// the labelled instance whose nearest visible node is closest to it.  d[c, j] = min over the non-NaN nodes k of
// sqrtf((x - cx)^2 + (y - cy)^2), each operation rounded on its own as numpy rounds it (NaN: no visible node).  A
// centroid whose d[c, :] is all NaN (no instance, or none with a visible node) is dropped; otherwise the pick starts at
// instance 0 and moves on a strict "<" only, so ties go to the lower index and an all-NaN instance 0 is kept.  One warp
// per centroid, lanes over the instances; `match` ([K] per frame) holds each centroid's pick (-1: dropped), then the
// picks of the kept rows in centroid order.
// Record per frame: [K][2] centroids | [K] centroid values | [K][nodes][2] points | [K][nodes] values (1) | centroid count |
// row count | flags.
__global__ void __launch_bounds__(128) k_td_gt_match(const float* __restrict__ sel_cent, const float* __restrict__ sel_val,
                                                     const int* __restrict__ sel_count, const float* __restrict__ inst,
                                                     const int* __restrict__ inst_count, int N, int nodes, int K,
                                                     const int* __restrict__ flags, int* __restrict__ match, float* __restrict__ record,
                                                     int width) {
  __shared__ int s_rows;
  const int b = blockIdx.x;
  const int cnt = sel_count[b], ni = inst_count[b];
  const float* cent = sel_cent + (size_t)b * K * 2;
  const float* ins = inst + (size_t)b * N * nodes * 2;
  int* mt = match + (size_t)b * K;
  float* r = record + (size_t)b * width;
  float* rp = r + K * 3;
  float* rq = rp + (size_t)K * nodes * 2;
  td_write_centroids(sel_cent, sel_val, b, cnt, K, r);
  const int lane = threadIdx.x & 31;
  for (int c = threadIdx.x >> 5; c < cnt; c += blockDim.x >> 5) {
    const float cx = cent[2 * c], cy = cent[2 * c + 1];
    float bv = 0.f, d0 = CUDART_NAN_F;
    int bj = -1;                                         // the lane's first smallest non-NaN distance (-1: none)
    for (int j = lane; j < ni; j += 32) {
      const float* p = ins + (size_t)j * nodes * 2;
      // np.nanmin over the nodes of the rounded roots: a correctly rounded sqrtf is monotone, so the root of the smallest
      // square is the smallest root, bit for bit (the picks below still compare roots)
      float q = CUDART_NAN_F;
      for (int k = 0; k < nodes; ++k) {
        const float dx = __fsub_rn(p[2 * k], cx), dy = __fsub_rn(p[2 * k + 1], cy);
        const float s = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
        if (s < q || q != q) q = s;
      }
      const float m = __fsqrt_rn(q);
      if (j == 0) d0 = m;
      if (m == m && (bj < 0 || m < bv)) { bv = m; bj = j; }
    }
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_down_sync(0xffffffffu, bv, o);
      const int oj = __shfl_down_sync(0xffffffffu, bj, o);
      if (oj >= 0 && (bj < 0 || ov < bv || (ov == bv && oj < bj))) { bv = ov; bj = oj; }
    }
    // lane 0 ran instance 0: a NaN there is never left by a "<", whatever the others hold
    if (lane == 0) mt[c] = bj < 0 ? -1 : (d0 != d0 ? 0 : bj);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int rows = 0;
    for (int c = 0; c < cnt; ++c)
      if (mt[c] >= 0) mt[rows++] = mt[c];
    s_rows = rows;
  }
  __syncthreads();
  const int rows = s_rows;
  for (int t = threadIdx.x; t < K * nodes * 2; t += blockDim.x) {
    const int k = t / (nodes * 2);
    rp[t] = (k < rows) ? ins[(size_t)mt[k] * nodes * 2 + (t - k * nodes * 2)] : CUDART_NAN_F;
  }
  for (int t = threadIdx.x; t < K * nodes; t += blockDim.x) rq[t] = (t / nodes < rows) ? 1.f : CUDART_NAN_F;
  if (threadIdx.x == 0) {
    rq[(size_t)K * nodes] = (float)cnt;
    rq[(size_t)K * nodes + 1] = (float)rows;
    rq[(size_t)K * nodes + 2] = (float)flags[b];
  }
}

// The class-vector head's shape: the tap (H x W x C logical channels), pooling, the dense stack and its packed weights
struct TdHead {
  int H, W, C;          // tap
  int global_pool;      // 1: max over H x W; 0: Flatten in (H, W, C) order
  int n_fc, units, n_classes;
  int n_in;             // inputs of the first dense layer: C or H * W * C
  int wmax;             // widest vector kept in shared memory (even)
  const float* w;       // packed dense weights (include/sleap_b200.h)
};

__device__ __forceinline__ float tap_value(const float* q, int) { return q[0]; }
__device__ __forceinline__ float tap_value(const __half* q, int hi) {
  // split-precision planes [lo | hi | hi]: lo + hi, one fp32 add (DeviceModel._class_vectors)
  return hi ? __fadd_rn(__half2float(q[0]), __half2float(q[hi])) : __half2float(q[0]);
}

// ------------------------------------------------------------------------------------------
// ClassVectorsHead on the tap of n crops, one CTA per crop: pooled (or flattened) features, num_fc_layers x (Dense + ReLU),
// Dense, softmax -> probs [n][n_classes].  Arithmetic as defined in include/sleap_b200.h.  tap: the crop-0 element of the
// buffer at the tap's channel offset; pitch = the buffer's physical channels; hi = the channel distance of the hi plane
// (0: one plane).  features_out (may be NULL): the first dense layer's input vector of every crop, [n][n_in].
// ------------------------------------------------------------------------------------------
template <typename T>
__global__ void __launch_bounds__(128) k_class_vectors(const T* __restrict__ tap, int pitch, int hi, TdHead d,
                                                       float* __restrict__ probs, float* __restrict__ features_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* s_x = reinterpret_cast<float*>(smem_raw);       // [wmax] layer input
  float* s_y = s_x + d.wmax;                             // [wmax] layer output
  double* s_e = reinterpret_cast<double*>(s_y + d.wmax); // [n_classes] exp terms, then [n_classes] = their sum
  __shared__ double s_sum;
  const int crop = blockIdx.x, HW = d.H * d.W;
  const T* base = tap + (size_t)crop * HW * pitch;
  auto feat = [&](int i) -> float {                      // flat input i = (p, c), Flatten order
    const int p = i / d.C, c = i - p * d.C;
    return tap_value(base + (size_t)p * pitch + c, hi);
  };
  if (d.global_pool) {
    for (int c = threadIdx.x; c < d.C; c += blockDim.x) {
      float m = tap_value(base + c, hi);
      for (int p = 1; p < HW; ++p) {                     // np.max: a NaN propagates
        const float v = tap_value(base + (size_t)p * pitch + c, hi);
        m = (v > m || v != v) ? v : m;
      }
      s_x[c] = m;
      if (features_out) features_out[(size_t)crop * d.n_in + c] = m;
    }
  } else if (features_out) {
    for (int i = threadIdx.x; i < d.n_in; i += blockDim.x) features_out[(size_t)crop * d.n_in + i] = feat(i);
  }
  __syncthreads();
  const float* w = d.w;
  int n_in = d.n_in;
  for (int l = 0; l <= d.n_fc; ++l) {
    const bool last = l == d.n_fc;
    const int n_out = last ? d.n_classes : d.units;
    const float* kern = w;
    const float* bias = w + (size_t)n_in * n_out;
    const bool flat_in = l == 0 && !d.global_pool;       // a Flatten input is read from the tap, not staged
    for (int j = threadIdx.x; j < n_out; j += blockDim.x) {
      double acc = 0.0;
      for (int i = 0; i < n_in; ++i) {
        const float x = flat_in ? feat(i) : s_x[i];
        acc = __dadd_rn(acc, __dmul_rn((double)x, (double)kern[(size_t)i * n_out + j]));
      }
      const float z = __double2float_rn(__dadd_rn(acc, (double)bias[j]));
      s_y[j] = (last || !(z < 0.f)) ? z : 0.f;            // ReLU as np.maximum(z, 0): NaN and -0 pass
    }
    __syncthreads();
    float* t = s_x; s_x = s_y; s_y = t;
    w = bias + n_out;
    n_in = n_out;
  }
  // softmax in float64 over the float32 logits s_x[0..n_classes)
  const int NC = d.n_classes;
  float zmax = s_x[0];
  for (int j = 1; j < NC; ++j) zmax = (s_x[j] > zmax || s_x[j] != s_x[j]) ? s_x[j] : zmax;
  for (int j = threadIdx.x; j < NC; j += blockDim.x) s_e[j] = exp(__dadd_rn((double)s_x[j], -(double)zmax));
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int j = 0; j < NC; ++j) s = __dadd_rn(s, s_e[j]);
    s_sum = s;
  }
  __syncthreads();
  for (int j = threadIdx.x; j < NC; j += blockDim.x) probs[(size_t)crop * NC + j] = __double2float_rn(__ddiv_rn(s_e[j], s_sum));
}

// ------------------------------------------------------------------------------------------
// Identity grouping of the top-down multi-class step: one CTA per frame.  Its crops (rows, crop order) are assigned to
// the classes (columns) by SciPy's assignment on -probability; a match is kept only where its probability is the crop's
// best over all classes (group_class_peaks), whatever its peaks.  Record per frame: points [NC][nodes][2] | peak values
// [NC][nodes] | class probabilities [NC] | centroids [K][2] | centroid values [K] | crop count | flags, padded to 4 floats.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_td_class_assign(const float* __restrict__ sel_cent, const float* __restrict__ sel_val,
                                                         const int* __restrict__ sel_count, const int* __restrict__ offsets,
                                                         const float* __restrict__ ipts, const float* __restrict__ ivals,
                                                         const float* __restrict__ probs, int K, int nodes, int NC,
                                                         const int* __restrict__ flags, float* __restrict__ record, int width) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int b = blockIdx.x;
  const int cnt = sel_count[b], o = offsets[b];
  const int L = max(K, NC), M = min(K, NC);
  int* s_rows = reinterpret_cast<int*>(smem_raw + ((lsap_scratch_bytes(L) + 15) & ~(size_t)15));
  int* s_cols = s_rows + M;
  float* rp = record + (size_t)b * width;
  float* rv = rp + (size_t)NC * nodes * 2;
  float* rpr = rv + (size_t)NC * nodes;
  float* rc = rpr + NC;
  float* tail = rc + 3 * K;
  for (int t = threadIdx.x; t < NC * nodes * 3 + NC; t += blockDim.x) rp[t] = CUDART_NAN_F;
  td_write_centroids(sel_cent, sel_val, b, cnt, K, rc);
  if (threadIdx.x == 0) {
    tail[0] = (float)cnt;
    tail[1] = flags ? (float)flags[b] : 0.f;
    for (float* q = tail + 2; q < record + (size_t)(b + 1) * width; ++q) *q = 0.f;   // padding
  }
  __syncthreads();                       // NaN fill ordered before thread 0's stores
  if (threadIdx.x != 0 || cnt == 0) return;
  const float* P = probs + (size_t)o * NC;
  LsapScratch s = carve_lsap(smem_raw, L);
  const int nm = lsap_solve_cost([P, NC](int i, int k) { return -(double)P[(size_t)i * NC + k]; }, cnt, NC, s, s_rows, s_cols);
  for (int q = 0; q < nm; ++q) {
    const int i = s_rows[q], k = s_cols[q];
    const float p = P[(size_t)i * NC + k];
    float best = P[(size_t)i * NC];
    for (int j = 1; j < NC; ++j) {       // np.max: a NaN propagates
      const float v = P[(size_t)i * NC + j];
      best = (v > best || v != v) ? v : best;
    }
    if (!(p == best)) continue;
    for (int t = 0; t < nodes * 2; ++t) rp[(size_t)k * nodes * 2 + t] = ipts[(size_t)(o + i) * nodes * 2 + t];
    for (int t = 0; t < nodes; ++t) rv[(size_t)k * nodes + t] = ivals[(size_t)(o + i) * nodes + t];
    rpr[k] = p;
  }
}

size_t td_class_record_width(int NC, int nodes, int K) {
  return (((size_t)NC * nodes * 3 + NC + 3 * (size_t)K + 2) + 3) & ~(size_t)3;
}

size_t class_vectors_smem(const TdHead& d) { return (size_t)2 * d.wmax * sizeof(float) + (size_t)d.n_classes * sizeof(double); }

// k_class_vectors on n crops of a tap in fp32 or fp16 storage
int launch_class_vectors(sb_handle_s* h, const void* tap, bool half, int pitch, int hi, const TdHead& d, int n, float* probs,
                         float* features_out) {
  if (n <= 0) return 0;
  const size_t sm = class_vectors_smem(d);
  if (half)
    k_class_vectors<__half><<<n, 128, sm, h->stream>>>((const __half*)tap, pitch, hi, d, probs, features_out);
  else
    k_class_vectors<float><<<n, 128, sm, h->stream>>>((const float*)tap, pitch, hi, d, probs, features_out);
  SB_CHECK_LAUNCH(h);
  return 0;
}

int launch_class_assign(sb_handle_s* h, const float* sel_cent, const float* sel_val, const int* sel_count, const int* offsets,
                        const float* ipts, const float* ivals, const float* probs, int B, int K, int nodes, int NC, const int* flags,
                        float* record) {
  const int L = std::max(K, NC), M = std::min(K, NC);
  const size_t sm = ((lsap_scratch_bytes(L) + 15) & ~(size_t)15) + 2 * (size_t)M * sizeof(int);
  if (sm > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(k_td_class_assign, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    if (e != cudaSuccess) return sb_fail(h, SB_ERR_CUDA, "class assignment smem %zu: %s", sm, cudaGetErrorString(e));
  }
  k_td_class_assign<<<B, 128, sm, h->stream>>>(sel_cent, sel_val, sel_count, offsets, ipts, ivals, probs, K, nodes, NC, flags, record,
                                               (int)td_class_record_width(NC, nodes, K));
  SB_CHECK_LAUNCH(h);
  return 0;
}

// The head fields of the parameters (everything but the tap's storage), checked against the tap's logical shape H x W x C:
// caps, layer sizes and the length of the packed weights.
int head_from_params(sb_handle_s* h, const sb_topdown_multiclass_params* p, int H, int W, int C, TdHead& d) {
  if (p->n_classes < 1 || p->n_classes > SB_MAX_CLASSES)
    return sb_fail(h, SB_ERR_UNSUPPORTED, "%d classes (1 to %d)", p->n_classes, SB_MAX_CLASSES);
  if (p->num_fc_layers < 0 || (p->num_fc_layers > 0 && p->num_fc_units < 1) || H <= 0 || W <= 0 || C <= 0)
    return sb_fail(h, SB_ERR_INVALID, "class-vector head: bad layer sizes");
  if (p->num_fc_units > SB_MAX_DENSE_WIDTH || (p->global_pool && C > SB_MAX_DENSE_WIDTH))
    return sb_fail(h, SB_ERR_UNSUPPORTED, "class-vector head: dense width above %d", SB_MAX_DENSE_WIDTH);
  d.H = H; d.W = W; d.C = C;
  d.global_pool = p->global_pool != 0;
  d.n_fc = p->num_fc_layers; d.units = d.n_fc > 0 ? p->num_fc_units : 0; d.n_classes = p->n_classes;
  d.n_in = d.global_pool ? C : H * W * C;
  d.wmax = std::max(std::max(d.global_pool ? C : 0, d.units), d.n_classes);
  d.wmax += d.wmax & 1;                                     // keeps the float64 exp terms 8-byte aligned
  d.w = nullptr;
  int64_t need = 0, n_in = d.n_in;
  for (int l = 0; l <= d.n_fc; ++l) {
    const int64_t n_out = l == d.n_fc ? d.n_classes : d.units;
    need += n_in * n_out + n_out;
    n_in = n_out;
  }
  if (!p->dense_weights || p->n_dense_weights != need)
    return sb_fail(h, SB_ERR_INVALID, "class-vector head: %lld dense weights given, %lld expected", (long long)p->n_dense_weights,
                   (long long)need);
  return 0;
}

// The forms of the pipeline by their centroid source: a centroid model (sb_topdown_configure, held by the centroid
// model), ground-truth centroids (centroid_model = -1, held by the instance model), a centroid model with ground-truth
// instances (sb_topdown_gt_instances_configure, no instance model, held by the centroid model).  A call takes a mask.
enum { TD_MODEL = 1, TD_GT = 2, TD_GTI = 4 };

}  // namespace

struct SbTopdown {
  sb_topdown_params p{};
  int form = TD_MODEL;
  SbModel* inst = nullptr;          // the instance model (NULL in the TD_GTI form)
  unsigned gen_c = 0, gen_i = 0;    // chain_gen of the centroid and the instance model when it was configured
  int K = 0, nodes = 0, width = 0, Bmax = 0;
  int H = 0, W = 0, C = 0;          // the uint8 or float frames of a batch
  float scale = 1.f;                // pre-crop resize (1: none) and the resized frame the crops are cut from
  int Hr = 0, Wr = 0;
  int* flags = nullptr;             // per-frame flags: the centroid model's ws.flags, or gt_flags
  float *sel_cent = nullptr, *sel_val = nullptr, *flat_cent = nullptr, *flat_off = nullptr, *ipts = nullptr, *ivals = nullptr, *record = nullptr;
  int *sel_count = nullptr, *flat_sample = nullptr, *offsets = nullptr, *total = nullptr;
  float* crops = nullptr;           // one chunk of float or uint8 crops
  // multi-class form (sb_topdown_multiclass_configure)
  bool multiclass = false;
  TdHead head{};
  int tap_buf = -1, tap_coff = 0, tap_hi = 0;
  bool tap_half = false, all_stores = false;   // fp16 storage; the production program elides the tap buffer
  float* dense = nullptr;                      // packed dense weights
  float* probs = nullptr;                      // [Bmax * K][n_classes] per-crop class probabilities
  // the steps (sb_topdown_submit / _collect, sb_topdown_gt_submit, and sb_infer_topdown* into slot 0), allocated at the
  // first of them: the slots (frames, record staging), and per slot the pinned crop count and its event, the frames its
  // crops are cut from and, multi-class, the pinned class probabilities of its crops; `pending` is the slot whose instance
  // stage is not queued yet (-1: none)
  SbSlots slots;
  int* count_host = nullptr;                   // [2]
  float* probs_stage[2] = {nullptr, nullptr};  // [Bmax * K][n_classes]
  cudaEvent_t count_ev[2] = {nullptr, nullptr};
  struct { const void* dev; int is_u8; } src[2] = {};   // the slot's frames, or a synchronous call's frames_dev
  int pending = -1;
  // the table-fed forms (TD_GT, TD_GTI): per slot the device copy of the batch's host table and its counts -- the
  // ground-truth centroids [Bmax][K][2], which k_td_gt_select reads, or the ground-truth instances [Bmax][N][nodes][2],
  // which k_td_gt_match reads -- allocated at the first step; a frame's floats and row cap (K or N) of the table.
  float* table[2] = {nullptr, nullptr};
  int* table_count[2] = {nullptr, nullptr};    // [Bmax]
  int table_floats = 0, table_rows = 0;
  int* gt_flags = nullptr;                     // TD_GT: [Bmax] the per-frame flags, which k_td_gt_select zeroes
  int* match = nullptr;                        // TD_GTI: [Bmax][K] k_td_gt_match's per-centroid picks
};

void sb_topdown_free(SbModel* m) {
  SbTopdown* t = m->td;
  if (!t) return;
  void* dev[] = {t->sel_cent, t->sel_val, t->flat_cent, t->flat_off, t->ipts, t->ivals, t->record, t->sel_count, t->flat_sample,
                 t->offsets, t->total, t->crops, t->dense, t->probs, t->table[0], t->table[1], t->table_count[0], t->table_count[1],
                 t->gt_flags, t->match};
  for (void* p : dev) if (p) cudaFree(p);
  t->slots.release();
  for (void* p : {(void*)t->count_host, (void*)t->probs_stage[0], (void*)t->probs_stage[1]})
    if (p) cudaFreeHost(p);
  for (cudaEvent_t e : t->count_ev) if (e) cudaEventDestroy(e);
  delete t;
  m->td = nullptr;
  m->trk = nullptr;                              // an attached tracker lives with the pipeline
}

namespace {

// The pre-crop resize of the parameters (0: 1) and the size of the H x W frames resized by it
int precrop_size(sb_handle_s* h, const sb_topdown_params* p, int H, int W, float* s, int* Hr, int* Wr) {
  *s = p->precrop_resize == 0.f ? 1.f : p->precrop_resize;
  if (sb_resized_size(H, W, *s, Hr, Wr))
    return sb_fail(h, SB_ERR_INVALID, "sb_topdown_configure: precrop_resize %g of %d x %d frames", p->precrop_resize, H, W);
  return 0;
}

// The arguments every top-down configure call checks before anything is dropped, for the pipeline of `form`; *mc is NULL
// in the TD_GT form, *mi in the TD_GTI form, which has no instance model and ignores `instance`, crop_size and
// max_crops_per_call but takes a table of N rows of n_nodes nodes per frame.
int check_topdown(sb_handle_s* h, const char* what, const sb_topdown_params* p, int form, int max_batch, int H, int W, int n_nodes,
                  int N, SbModel** mc, SbModel** mi) {
  const bool has_c = form != TD_GT, has_i = form != TD_GTI;
  if (!has_i && p->instance_model != -1) return sb_fail(h, SB_ERR_INVALID, "%s: instance_model must be -1", what);
  *mc = has_c ? chain_model(h, p->centroid_model, SB_CHAIN_ANY, "bad model ids") : nullptr;
  *mi = has_i ? chain_model(h, p->instance_model, SB_CHAIN_ANY, "bad model ids") : nullptr;
  if ((has_c && !*mc) || (has_i && !*mi) || *mc == *mi) return sb_fail(h, SB_ERR_INVALID, "%s: bad model ids", what);
  if (p->max_centroids_per_frame <= 0 || max_batch <= 0 || (has_i && (p->crop_size <= 0 || p->max_crops_per_call <= 0)) ||
      (!has_i && (n_nodes <= 0 || N <= 0)))
    return sb_fail(h, SB_ERR_INVALID, "%s: bad sizes", what);
  if (max_batch > 1024) return sb_fail(h, SB_ERR_UNSUPPORTED, "%s: more than 1024 frames per batch", what);
  if (has_i && (p->instance.cms_buffer < 0 || p->instance.cms_buffer >= (int)(*mi)->buffers.size()))
    return sb_fail(h, SB_ERR_INVALID, "bad cms buffer");
  float s;
  int Hr, Wr;
  return precrop_size(h, p, H, W, &s, &Hr, &Wr);
}

// Configures the networks of the form and their chains, then the pipeline of the form: on success the new pipeline is
// the td of its owner, the centroid model (whose configure dropped the previous one) or in the TD_GT form the instance
// model (whose global configure did).  n_classes > 0: the multi-class record; n_nodes and N: the TD_GTI table.
int topdown_setup(sb_handle_s* h, const sb_topdown_params* p, int form, int max_batch, int H, int W, int C_in, SbModel* mc, SbModel* mi,
                  int n_classes, int n_nodes, int N) {
  SB_CUDA(h, cudaSetDevice(h->device));
  int rc;
  if (mc && (rc = sb_model_configure(h, p->centroid_model, max_batch, H, W, C_in))) return rc;
  // the instance network runs chunks of up to max_crops_per_call crops; a ground-truth batch has at most max_batch x K
  // crops, so that form plans it for no more than those
  const int chunk = mc ? p->max_crops_per_call
                       : (int)std::min<long long>(p->max_crops_per_call, (long long)max_batch * p->max_centroids_per_frame);
  if (mi && (rc = sb_model_configure(h, p->instance_model, chunk, p->crop_size, p->crop_size, C_in))) return rc;
  if (mc && (rc = sb_centroid_configure(h, p->centroid_model, &p->centroid))) return rc;
  if (mi && (rc = sb_global_configure(h, p->instance_model, &p->instance))) return rc;
  SbTopdown* t = new SbTopdown();
  SbModel* owner = mc ? mc : mi;
  owner->td = t;
  t->p = *p; t->form = form; t->inst = mi; t->K = p->max_centroids_per_frame; t->Bmax = max_batch;
  t->gen_c = mc ? mc->chain_gen : 0; t->gen_i = mi ? mi->chain_gen : 0;
  t->H = H; t->W = W; t->C = C_in;
  precrop_size(h, p, H, W, &t->scale, &t->Hr, &t->Wr);     // checked by check_topdown
  t->nodes = mi ? mi->buffers[p->instance.cms_buffer].C : n_nodes;
  t->multiclass = n_classes > 0;
  // the dense per-frame record of k_td_class_assign, k_td_pack or k_td_gt_match
  const int K = t->K, nodes = t->nodes;
  t->width = t->multiclass ? (int)td_class_record_width(n_classes, nodes, K) : K * (3 + nodes * 3) + (form == TD_GTI ? 3 : 2);
  t->table_rows = form == TD_GT ? K : N;
  t->table_floats = form == TD_GT ? K * 2 : N * nodes * 2;
  const size_t KB = (size_t)max_batch * K;
  if ((rc = sb_dev_alloc(h, &t->sel_cent, KB * 2)) || (rc = sb_dev_alloc(h, &t->sel_val, KB)) ||
      (rc = sb_dev_alloc(h, &t->sel_count, (size_t)max_batch)) || (rc = sb_dev_alloc(h, &t->record, (size_t)max_batch * t->width)) ||
      (mi && ((rc = sb_dev_alloc(h, &t->flat_cent, KB * 2)) || (rc = sb_dev_alloc(h, &t->flat_off, KB * 2)) ||
              (rc = sb_dev_alloc(h, &t->flat_sample, KB)) || (rc = sb_dev_alloc(h, &t->offsets, (size_t)max_batch + 1)) ||
              (rc = sb_dev_alloc(h, &t->total, 1)) || (rc = sb_dev_alloc(h, &t->ipts, KB * nodes * 2)) ||
              (rc = sb_dev_alloc(h, &t->ivals, KB * nodes)) ||
              (rc = sb_dev_alloc(h, &t->crops, (size_t)chunk * p->crop_size * p->crop_size * C_in)))) ||
      (t->multiclass && (rc = sb_dev_alloc(h, &t->probs, KB * n_classes))) ||
      (form == TD_GT && (rc = sb_dev_alloc(h, &t->gt_flags, (size_t)max_batch))) ||
      (form == TD_GTI && (rc = sb_dev_alloc(h, &t->match, KB)))) {
    sb_topdown_free(owner);
    return rc;
  }
  t->flags = mc ? mc->ws.flags : t->gt_flags;
  return SB_OK;
}

// The calls of each form and kind: the refusals of a call on the wrong form or kind name the pipeline's own.  The
// table-fed forms have no synchronous call: a batch is a submit and a collect.
struct TdCalls {
  const char *source, *submit, *collect, *sync, *configure;
};

const TdCalls& td_calls(const SbTopdown* t) {
  static const TdCalls calls[3][2] = {
      {{"runs a centroid model", "sb_topdown_submit", "sb_topdown_collect", "sb_infer_topdown", "sb_topdown_configure"},
       {"runs a centroid model", "sb_topdown_multiclass_submit", "sb_topdown_multiclass_collect", "sb_infer_topdown_multiclass",
        "sb_topdown_multiclass_configure"}},
      {{"takes ground-truth centroids", "sb_topdown_gt_submit", "sb_topdown_collect", "sb_topdown_gt_submit", "sb_topdown_configure"},
       {"takes ground-truth centroids", "sb_topdown_gt_submit", "sb_topdown_multiclass_collect", "sb_topdown_gt_submit",
        "sb_topdown_multiclass_configure"}},
      {{"takes ground-truth instances", "sb_topdown_gt_instances_submit", "sb_topdown_gt_instances_collect",
        "sb_topdown_gt_instances_submit", "sb_topdown_gt_instances_configure"},
       {}}};                                       // no multi-class form
  return calls[t->form == TD_MODEL ? 0 : t->form == TD_GT ? 1 : 2][t->multiclass];
}

// The pipeline of model `id` (its owner) when it is of one of the forms `sources` (a mask of TD_*) and of the kind
// `multiclass` (-1: either), and no model of it was reconfigured since.  `streamed`: a refusal names the pipeline's submit
// and collect calls, not its synchronous one.
SbTopdown* topdown_of(sb_handle_s* h, int id, int sources, int multiclass, bool streamed) {
  static const char* const none = "top-down pipeline not configured";
  SbModel* owner = chain_model(h, id, SB_CHAIN_ANY, none);
  if (!owner) return nullptr;
  SbTopdown* t = owner->td;
  if (!t) { sb_fail(h, SB_ERR_INVALID, none); return nullptr; }
  const TdCalls& c = td_calls(t);
  const char* why = !(sources & t->form)                          ? c.source
                    : multiclass >= 0 && t->multiclass != (multiclass != 0) ? (t->multiclass ? "is multi-class" : "is not multi-class")
                                                                  : nullptr;
  if (why) {
    if (streamed)
      sb_fail(h, SB_ERR_INVALID, "top-down pipeline %s: call %s / %s", why, c.submit, c.collect);
    else
      sb_fail(h, SB_ERR_INVALID, "top-down pipeline %s: call %s", why, c.sync);
    return nullptr;
  }
  // a configure call on the owner dropped the pipeline with its chain; one on the instance model of the TD_MODEL form
  // outside the pipeline's configure moved its chain_gen (sb_model_configure included)
  const SbModel* mi = t->inst;
  if (t->form == TD_MODEL && (owner->chain != SB_CHAIN_CENTROID || owner->chain_gen != t->gen_c || mi->chain != SB_CHAIN_GLOBAL ||
                              mi->chain_gen != t->gen_i)) {
    sb_fail(h, SB_ERR_INVALID, "top-down pipeline: a model was reconfigured; call %s again", c.configure);
    return nullptr;
  }
  return t;
}

// The flat crop list and crop offsets of the B frames' selected centroids, on the handle's stream
int flatten(sb_handle_s* h, SbTopdown* t, int B) {
  k_td_flatten<<<1, 256, 0, h->stream>>>(t->sel_cent, t->sel_count, B, t->K, (float)t->p.crop_size * 0.5f, t->flat_cent, t->flat_off,
                                         t->flat_sample, t->offsets, t->total);
  SB_CHECK_LAUNCH(h);
  return 0;
}

// The centroids of B frames resident at frames_dev in the selection buffers: centroid network, local peaks, top-k
int select_centroids(sb_handle_s* h, SbModel* mc, SbTopdown* t, const void* frames_dev, int frames_are_u8, int B) {
  int rc = sb_run_ops(h, mc, frames_dev, frames_are_u8, B);
  if (rc) return rc;
  const sb_centroid_params& cp = mc->ce;
  SbBuffer& cb = mc->buffers[cp.cms_buffer];
  const float* coff = cp.offsets_buffer >= 0 ? (const float*)mc->buffers[cp.offsets_buffer].dev : nullptr;
  SbPeakParams pc{cp.peak_threshold, cp.refinement, cp.integral_patch_size, (float)cp.output_stride, cp.input_scale};
  if ((rc = sbk_local_peaks(h, (const float*)cb.dev, coff, B, cb.H, cb.W, cb.C, pc, mc->ws))) return rc;
  k_td_select<<<B, 128, 0, h->stream>>>(mc->ws.peaks, mc->ws.peak_vals, mc->ws.n_peaks, mc->ws.max_peaks, t->p.max_instances, t->K, t->scale,
                                        t->sel_cent, t->sel_val, t->sel_count, mc->ws.flags);
  SB_CHECK_LAUNCH(h);
  return 0;
}

// The centroid stage of B frames resident at frames_dev: centroid network, local peaks, top-k, the flat crop list, then
// the crop count's copy into *count_host and, given, count_ev.
int centroid_stage(sb_handle_s* h, SbModel* mc, SbTopdown* t, const void* frames_dev, int frames_are_u8, int B, int* count_host,
                   cudaEvent_t count_ev) {
  cudaStream_t s = h->stream;
  int rc;
  if ((rc = select_centroids(h, mc, t, frames_dev, frames_are_u8, B)) || (rc = flatten(h, t, B))) return rc;
  SB_CUDA(h, cudaMemcpyAsync(count_host, t->total, 4, cudaMemcpyDeviceToHost, s));
  if (count_ev) SB_CUDA(h, cudaEventRecord(count_ev, s));
  return 0;
}

// The instance stage of the batch the centroid stage left in the selection buffers (`total` crops of the B frames at
// frames_dev): per chunk of crops the crop kernel, the instance network, the global peaks and, multi-class, the class
// vectors; frames_free (given) after the last crop kernel; then the records -- k_td_class_assign, or k_td_pack and the
// attached tracker of the centroid model mc (NULL in the ground-truth form) -- copied into rec_dst, the track records into
// trk_host and, given, the crops' class probabilities into probs_host.
int instance_stage(sb_handle_s* h, const SbModel* mc, SbTopdown* t, const void* frames_dev, int frames_are_u8, int B, int total,
                   float* rec_dst, double* trk_host, float* probs_host, cudaEvent_t frames_free) {
  cudaStream_t s = h->stream;
  SbModel* mi = t->inst;
  const sb_global_params& gp = mi->gl;
  SbBuffer& ib = mi->buffers[gp.cms_buffer];
  const float* ioff = gp.offsets_buffer >= 0 ? (const float*)mi->buffers[gp.offsets_buffer].dev : nullptr;
  SbPeakParams pi{gp.peak_threshold, gp.refinement, gp.integral_patch_size, (float)gp.output_stride, gp.input_scale};
  const int cs = t->p.crop_size, NC = t->head.n_classes;
  const SbBuffer* tb = t->multiclass ? &mi->buffers[t->tap_buf] : nullptr;
  int rc;
  for (int c0 = 0; c0 < total; c0 += mi->B) {
    const int n = std::min(mi->B, total - c0);
    // crops of the frames already resident in HBM (uint8 frames: float -> uint8 truncation, as tf.cast in crop_bboxes),
    // with a pre-crop resize of those frames resized on the fly
    const float* cent = t->flat_cent + 2 * (size_t)c0;
    if ((rc = t->scale != 1.f ? sbk_crop_resized(h, frames_dev, frames_are_u8, B, t->H, t->W, t->C, t->Hr, t->Wr, cent,
                                                 t->flat_sample + c0, n, cs, cs, t->crops)
                              : sbk_crop(h, frames_dev, frames_are_u8, B, t->H, t->W, t->C, cent, t->flat_sample + c0, n, cs, cs,
                                         t->crops, frames_are_u8)))
      return rc;
    if ((rc = sb_run_ops(h, mi, t->crops, frames_are_u8, n, t->all_stores))) return rc;
    if ((rc = sbk_global_peaks(h, (const float*)ib.dev, ioff, n, ib.H, ib.W, ib.C, pi, t->flat_off + 2 * (size_t)c0, mi->gs.part, mi->gs.chunks, mi->gs.rpc,
                               t->ipts + (size_t)c0 * t->nodes * 2, t->ivals + (size_t)c0 * t->nodes))) return rc;
    if (tb && (rc = launch_class_vectors(h, (const char*)tb->dev + (size_t)t->tap_coff * (t->tap_half ? 2 : 4), t->tap_half, tb->C,
                                         t->tap_hi, t->head, n, t->probs + (size_t)c0 * NC, nullptr)))
      return rc;
  }
  if (frames_free) SB_CUDA(h, cudaEventRecord(frames_free, s));
  if (t->multiclass) {
    if ((rc = launch_class_assign(h, t->sel_cent, t->sel_val, t->sel_count, t->offsets, t->ipts, t->ivals, t->probs, B, t->K, t->nodes,
                                  NC, t->flags, t->record)))
      return rc;
    if (probs_host && total > 0)
      SB_CUDA(h, cudaMemcpyAsync(probs_host, t->probs, (size_t)total * NC * 4, cudaMemcpyDeviceToHost, s));
  } else {
    k_td_pack<<<B, 128, 0, s>>>(t->sel_cent, t->sel_val, t->sel_count, t->offsets, t->ipts, t->ivals, t->K, t->nodes, t->flags,
                                t->record, t->width);
    SB_CHECK_LAUNCH(h);
    if (mc && mc->trk) {
      // the attached tracker on the frames' instance lists; its records come back with the step's records
      if ((rc = sbk_track_topdown(h, mc->trk, B, t->ipts, t->ivals, t->sel_val, t->sel_count, t->offsets, t->K, mc->trk_h, mc->trk_w,
                                  mc->trk_dev)))
        return rc;
      SB_CUDA(h, cudaMemcpyAsync(trk_host, mc->trk_dev, (size_t)B * sb_track_record_width(mc->trk_I) * sizeof(double),
                                 cudaMemcpyDeviceToHost, s));
    }
  }
  SB_CUDA(h, cudaMemcpyAsync(rec_dst, t->record, (size_t)B * t->width * 4, cudaMemcpyDeviceToHost, s));
  return 0;
}

// Queues the instance stage of the pending batch (its count event waited for on the host) behind whatever the handle's
// stream holds.  The slot is dropped when it fails.
int queue_pending_instance(sb_handle_s* h, const SbModel* mc, SbTopdown* t) {
  const int k = t->pending;
  SbSlots& sl = t->slots;
  t->pending = -1;
  cudaError_t e = cudaEventSynchronize(t->count_ev[k]);
  int rc = e == cudaSuccess ? 0 : sb_fail(h, SB_ERR_CUDA, "crop count: %s", cudaGetErrorString(e));
  if (!rc) {
    rc = instance_stage(h, mc, t, t->src[k].dev, t->src[k].is_u8, sl.slot_B[k], t->count_host[k], sl.stage[k], mc->trk_host[k],
                        t->probs_stage[k], sl.frames_free[k]);
  }
  if (!rc) {
    e = cudaEventRecord(sl.result[k], h->stream);
    if (e != cudaSuccess) rc = sb_fail(h, SB_ERR_CUDA, "event record: %s", cudaGetErrorString(e));
  }
  if (rc) sl.drop(k);
  return rc;
}

// The slot buffers of the pipeline, allocated at its first step
int stream_alloc(sb_handle_s* h, SbTopdown* t) {
  int rc = t->slots.alloc(h, (size_t)t->Bmax * t->H * t->W * t->C, (size_t)t->Bmax * t->width);
  if (rc || t->count_host) return rc;
  const size_t probs_bytes = (size_t)t->Bmax * t->K * t->head.n_classes * 4;
  for (int i = 0; i < 2; ++i) {
    if (t->multiclass && !t->probs_stage[i]) SB_CUDA(h, cudaHostAlloc((void**)&t->probs_stage[i], probs_bytes, cudaHostAllocDefault));
    if (!t->count_ev[i]) SB_CUDA(h, cudaEventCreateWithFlags(&t->count_ev[i], cudaEventDisableTiming));
    if (t->form != TD_MODEL && !t->table[i] && (rc = sb_dev_alloc(h, &t->table[i], (size_t)t->Bmax * t->table_floats))) return rc;
    if (t->form != TD_MODEL && !t->table_count[i] && (rc = sb_dev_alloc(h, &t->table_count[i], (size_t)t->Bmax))) return rc;
  }
  SB_CUDA(h, cudaHostAlloc((void**)&t->count_host, 2 * sizeof(int), cudaHostAllocDefault));   // last: marks it complete
  return 0;
}

// The centroid stage of B frames at frames_dev queued as the batch of `slot`; its instance stage is queued by the next
// submit or by the slot's collect.
int queue_centroids(sb_handle_s* h, SbModel* mc, SbTopdown* t, const void* frames_dev, int frames_are_u8, int B, int slot) {
  if (const int rc = centroid_stage(h, mc, t, frames_dev, frames_are_u8, B, t->count_host + slot, t->count_ev[slot])) return rc;
  t->slots.submitted(slot, B);
  t->src[slot] = {frames_dev, frames_are_u8};
  t->pending = slot;
  return SB_OK;
}

// Streamed batch into `slot`: (1) its upload on the copy stream into the slot's frames, once the crops of the batch that
// last used them have run; (2) the instance stage of the batch submitted before it, if no collect queued it yet;
// (3) its own centroid stage.  The stream order instance(k) -> centroid(k + 1) lets one set of selection buffers serve.
int topdown_submit(sb_handle_s* h, int id, const uint8_t* frames_host, int B, int slot, bool multiclass) {
  SbTopdown* t = topdown_of(h, id, TD_MODEL, multiclass, true);
  if (!t) return SB_ERR_INVALID;
  SbModel* mc = h->models[id];
  SbSlots& sl = t->slots;
  int rc = sl.check_submit(h, "top-down submit", slot, B, t->Bmax, frames_host);
  if (rc) return rc;
  SB_CUDA(h, cudaSetDevice(h->device));
  if ((rc = stream_alloc(h, t)) || (rc = sl.upload(h, slot, frames_host, (size_t)B * t->H * t->W * t->C))) return rc;
  if (t->pending >= 0 && (rc = queue_pending_instance(h, mc, t))) return rc;
  SB_CUDA(h, cudaStreamWaitEvent(h->stream, sl.h2d_done[slot], 0));
  return queue_centroids(h, mc, t, sl.frames[slot], 1, B, slot);
}

// Streamed batch of a table-fed form into `slot` (sb_topdown_gt_submit, sb_topdown_gt_instances_submit), the whole step
// queued at once, since nothing in it waits on the host: the frames, the table and its counts (each in [0, table_rows])
// on the copy stream into the slot; behind that copy on the handle's stream, the form's launches -- ground-truth
// centroids: k_td_gt_select, the crop list and the instance stage; ground-truth instances: the centroid stage,
// k_td_gt_match and the records' copy.  The table has its own per-slot staging: the batch before may still be reading
// the selection buffers when the copy lands; it is free again once the slot's frames are (frames_free).
int table_submit(sb_handle_s* h, int id, int form, const uint8_t* frames_host, const float* table_host, const int32_t* counts_host,
                 int B, int slot) {
  SbTopdown* t = topdown_of(h, id, form, -1, true);
  if (!t) return SB_ERR_INVALID;
  const char* what = td_calls(t).submit;
  SbSlots& sl = t->slots;
  int rc = sl.check_submit(h, what, slot, B, t->Bmax, table_host && counts_host ? frames_host : nullptr);
  if (rc) return rc;
  int total = 0;
  for (int b = 0; b < B; ++b) {
    if (counts_host[b] < 0 || counts_host[b] > t->table_rows)
      return sb_fail(h, SB_ERR_INVALID, "%s: frame %d has %d %s, not 0 to %d (%s)", what, b, counts_host[b],
                     form == TD_GT ? "centroids" : "instances", t->table_rows,
                     form == TD_GT ? "max_centroids_per_frame" : "max_instances_per_frame");
    total += counts_host[b];
  }
  SB_CUDA(h, cudaSetDevice(h->device));
  if ((rc = stream_alloc(h, t)) ||
      (rc = sl.upload(h, slot, frames_host, (size_t)B * t->H * t->W * t->C,
                      {{t->table[slot], table_host, (size_t)B * t->table_floats * sizeof(float)},
                       {t->table_count[slot], counts_host, (size_t)B * sizeof(int32_t)}})))
    return rc;
  SB_CUDA(h, cudaStreamWaitEvent(h->stream, sl.h2d_done[slot], 0));
  if (form == TD_GT) {
    k_td_gt_select<<<B, 128, 0, h->stream>>>(t->table[slot], t->table_count[slot], t->K, t->scale, t->sel_cent, t->sel_val, t->sel_count,
                                             t->flags);
    SB_CHECK_LAUNCH(h);
    if ((rc = flatten(h, t, B)) ||
        (rc = instance_stage(h, nullptr, t, sl.frames[slot], 1, B, total, sl.stage[slot], nullptr, t->probs_stage[slot], sl.frames_free[slot])))
      return rc;
  } else {
    if ((rc = select_centroids(h, h->models[id], t, sl.frames[slot], 1, B))) return rc;
    k_td_gt_match<<<B, 128, 0, h->stream>>>(t->sel_cent, t->sel_val, t->sel_count, t->table[slot], t->table_count[slot], t->table_rows,
                                            t->nodes, t->K, t->flags, t->match, t->record, t->width);
    SB_CHECK_LAUNCH(h);
    SB_CUDA(h, cudaEventRecord(sl.frames_free[slot], h->stream));
    SB_CUDA(h, cudaMemcpyAsync(sl.stage[slot], t->record, (size_t)B * t->width * 4, cudaMemcpyDeviceToHost, h->stream));
  }
  SB_CUDA(h, cudaEventRecord(sl.result[slot], h->stream));
  sl.submitted(slot, B);
  return SB_OK;
}

// The streamed batch of `slot` of the pipeline held by model `id` in its pinned staging: its instance stage queued if
// still pending, then its record event waited for.  The slot is free again afterwards.
int topdown_collect(sb_handle_s* h, int id, SbTopdown* t, int slot, int B) {
  int rc = t->slots.check_collect(h, "top-down collect", slot, B);
  if (rc) return rc;
  SB_CUDA(h, cudaSetDevice(h->device));
  if (t->pending == slot && (rc = queue_pending_instance(h, h->models[id], t))) return rc;
  return t->slots.collect(h, slot);
}

// A synchronous batch of the pipeline held by centroid model `id`: the uint8 or float32 frames uploaded on the handle's
// stream into the model's frames_dev, the step queued into slot 0, then slot 0 collected.
int topdown_call(sb_handle_s* h, int id, SbTopdown* t, const void* frames_host, int frames_are_u8, int B, const char* what) {
  SbModel* mc = h->models[id];
  if (B <= 0 || B > t->Bmax || B > mc->B) return sb_fail(h, SB_ERR_INVALID, "bad batch");
  int rc = t->slots.check_idle(h, what);
  if (rc) return rc;
  SB_CUDA(h, cudaSetDevice(h->device));
  if ((rc = stream_alloc(h, t))) return rc;
  SB_CUDA(h, cudaMemcpyAsync(mc->frames_dev, frames_host, (size_t)B * mc->Hin * mc->Win * mc->Cin * (frames_are_u8 ? 1 : 4),
                             cudaMemcpyHostToDevice, h->stream));
  if ((rc = queue_centroids(h, mc, t, mc->frames_dev, frames_are_u8, B, 0))) return rc;
  return topdown_collect(h, id, t, 0, B);
}

// A plain record's fields into the caller's arrays
void split_topdown(const SbTopdown* t, const float* rec, int B, float* out_centroids, float* out_centroid_vals, float* out_instance_peaks,
                   float* out_instance_peak_vals, int32_t* out_n_valid, int32_t* out_flags) {
  const size_t K = t->K, nd = t->nodes;
  sb_split_records(rec, B, t->width,
                   {{out_centroids, K * 2}, {out_centroid_vals, K}, {out_instance_peaks, K * nd * 2}, {out_instance_peak_vals, K * nd}},
                   {out_n_valid, out_flags});
}

// A multi-class record's fields into the caller's arrays, and the crops' class probabilities (pr: the batch's crops in
// order, on the host) scattered to (frame, slot)
void split_topdown_multiclass(const SbTopdown* t, const float* rec, const float* pr, int B, float* out_centroids,
                              float* out_centroid_vals, float* out_points, float* out_vals, float* out_class_probs, int32_t* out_n_valid,
                              int32_t* out_flags, float* out_class_vectors) {
  const int NC = t->head.n_classes;
  const size_t K = t->K, n1 = (size_t)NC * t->nodes;
  if (out_class_vectors) {
    int o = 0;
    for (int b = 0; b < B; ++b) {
      const int cnt = (int)rec[(size_t)b * t->width + n1 * 3 + NC + 3 * K];
      float* dst = out_class_vectors + (size_t)b * K * NC;
      std::fill(dst, dst + K * NC, std::numeric_limits<float>::quiet_NaN());
      std::copy(pr + (size_t)o * NC, pr + (size_t)(o + cnt) * NC, dst);
      o += cnt;
    }
  }
  sb_split_records(rec, B, t->width,
                   {{out_points, n1 * 2}, {out_vals, n1}, {out_class_probs, (size_t)NC}, {out_centroids, K * 2}, {out_centroid_vals, K}},
                   {out_n_valid, out_flags});
}

}  // namespace

bool sb_topdown_busy(const SbModel* m) { return m->td && m->td->slots.busy(); }

extern "C" {

int sb_topdown_configure(sb_handle_t h, const sb_topdown_params* p, int max_batch, int H, int W, int C_in) {
  if (!h || !p) return sb_fail(h, SB_ERR_INVALID, "sb_topdown_configure: null argument");
  SbModel *mc, *mi;
  const int form = p->centroid_model == -1 ? TD_GT : TD_MODEL;
  if (const int rc = check_topdown(h, "sb_topdown_configure", p, form, max_batch, H, W, 0, 0, &mc, &mi)) return rc;
  return topdown_setup(h, p, form, max_batch, H, W, C_in, mc, mi, 0, 0, 0);
}

int sb_infer_topdown(sb_handle_t h, int centroid_model_id, const void* frames_host, int frames_are_u8, int B, float* out_centroids,
                     float* out_centroid_vals, float* out_instance_peaks, float* out_instance_peak_vals, int32_t* out_n_valid,
                     int32_t* out_flags) {
  SbTopdown* t = topdown_of(h, centroid_model_id, TD_MODEL, 0, false);
  if (!t) return SB_ERR_INVALID;
  if (const int rc = topdown_call(h, centroid_model_id, t, frames_host, frames_are_u8, B, "sb_infer_topdown")) return rc;
  split_topdown(t, t->slots.stage[0], B, out_centroids, out_centroid_vals, out_instance_peaks, out_instance_peak_vals, out_n_valid, out_flags);
  return SB_OK;
}

int sb_topdown_submit(sb_handle_t h, int centroid_model_id, const uint8_t* frames_host, int B, int slot) {
  return topdown_submit(h, centroid_model_id, frames_host, B, slot, false);
}

int sb_topdown_collect(sb_handle_t h, int model_id, int slot, int B, float* out_centroids, float* out_centroid_vals,
                       float* out_instance_peaks, float* out_instance_peak_vals, int32_t* out_n_valid, int32_t* out_flags) {
  SbTopdown* t = topdown_of(h, model_id, TD_MODEL | TD_GT, 0, true);
  if (!t) return SB_ERR_INVALID;
  if (const int rc = topdown_collect(h, model_id, t, slot, B)) return rc;
  split_topdown(t, t->slots.stage[slot], B, out_centroids, out_centroid_vals, out_instance_peaks, out_instance_peak_vals, out_n_valid, out_flags);
  return SB_OK;
}

int sb_topdown_gt_submit(sb_handle_t h, int instance_model_id, const uint8_t* frames_host, const float* centroids_host,
                         const int32_t* counts_host, int B, int slot) {
  return table_submit(h, instance_model_id, TD_GT, frames_host, centroids_host, counts_host, B, slot);
}

int sb_topdown_gt_instances_configure(sb_handle_t h, const sb_topdown_params* p, int n_nodes, int max_instances_per_frame, int max_batch,
                                      int H, int W, int C_in) {
  if (!h || !p) return sb_fail(h, SB_ERR_INVALID, "sb_topdown_gt_instances_configure: null argument");
  SbModel *mc, *mi;
  if (const int rc = check_topdown(h, "sb_topdown_gt_instances_configure", p, TD_GTI, max_batch, H, W, n_nodes, max_instances_per_frame,
                                   &mc, &mi))
    return rc;
  return topdown_setup(h, p, TD_GTI, max_batch, H, W, C_in, mc, nullptr, 0, n_nodes, max_instances_per_frame);
}

int sb_topdown_gt_instances_submit(sb_handle_t h, int centroid_model_id, const uint8_t* frames_host, const float* instances_host,
                                   const int32_t* counts_host, int B, int slot) {
  return table_submit(h, centroid_model_id, TD_GTI, frames_host, instances_host, counts_host, B, slot);
}

int sb_topdown_gt_instances_collect(sb_handle_t h, int centroid_model_id, int slot, int B, float* out_centroids, float* out_centroid_vals,
                                    int32_t* out_n_centroids, float* out_instance_peaks, float* out_instance_peak_vals,
                                    int32_t* out_n_rows, int32_t* out_flags) {
  SbTopdown* t = topdown_of(h, centroid_model_id, TD_GTI, -1, true);
  if (!t) return SB_ERR_INVALID;
  if (const int rc = topdown_collect(h, centroid_model_id, t, slot, B)) return rc;
  const size_t K = t->K, nd = t->nodes;
  sb_split_records(t->slots.stage[slot], B, t->width,
                   {{out_centroids, K * 2}, {out_centroid_vals, K}, {out_instance_peaks, K * nd * 2}, {out_instance_peak_vals, K * nd}},
                   {out_n_centroids, out_n_rows, out_flags});
  return SB_OK;
}

int sb_topdown_attach_tracker(sb_handle_t h, int centroid_model_id, int tracker_id, double img_h, double img_w) {
  SbTopdown* t = topdown_of(h, centroid_model_id, TD_MODEL, 0, false);
  if (!t) return SB_ERR_INVALID;
  SbModel* mc = h->models[centroid_model_id];
  if (const int rc = t->slots.check_idle(h, "sb_topdown_attach_tracker")) return rc;
  if (tracker_id < 0) { mc->trk = nullptr; return SB_OK; }
  SbTracker* tr = sb_tracker_get(h, tracker_id);
  if (!tr) return sb_fail(h, SB_ERR_INVALID, "sb_topdown_attach_tracker: no tracker %d on this handle", tracker_id);
  if (sb_tracker_nodes(tr) != t->nodes)
    return sb_fail(h, SB_ERR_INVALID, "sb_topdown_attach_tracker: tracker of %d nodes, instance model of %d", sb_tracker_nodes(tr),
                   t->nodes);
  if (!(img_h > 0) || !(img_w > 0)) return sb_fail(h, SB_ERR_INVALID, "sb_topdown_attach_tracker: image %g x %g", img_h, img_w);
  SB_CUDA(h, cudaSetDevice(h->device));
  if (const int rc = sb_track_records_alloc(h, mc, t->Bmax, sb_tracker_max_instances(tr))) return rc;
  mc->trk = tr; mc->trk_h = img_h; mc->trk_w = img_w;
  return SB_OK;
}

int sb_topdown_tracks(sb_handle_t h, int centroid_model_id, int slot, int B, double* out_tracks) {
  SbTopdown* t = topdown_of(h, centroid_model_id, TD_MODEL, 0, true);
  if (!t) return SB_ERR_INVALID;
  const SbModel* mc = h->models[centroid_model_id];
  if (!mc->trk) return sb_fail(h, SB_ERR_INVALID, "sb_topdown_tracks: no tracker attached");
  if (slot < 0 || slot > 1 || B <= 0 || B > t->Bmax || !out_tracks)
    return sb_fail(h, SB_ERR_INVALID, "sb_topdown_tracks: bad slot / batch");
  if (const int rc = t->slots.check_read(h, "sb_topdown_tracks", slot, B)) return rc;
  memcpy(out_tracks, mc->trk_host[slot], (size_t)B * sb_track_record_width(mc->trk_I) * sizeof(double));
  return SB_OK;
}

int sb_topdown_multiclass_configure(sb_handle_t h, const sb_topdown_multiclass_params* p, int max_batch, int H, int W, int C_in) {
  if (!h || !p) return sb_fail(h, SB_ERR_INVALID, "sb_topdown_multiclass_configure: null argument");
  SbModel *mc, *mi;
  const int form = p->topdown.centroid_model == -1 ? TD_GT : TD_MODEL;
  int rc = check_topdown(h, "sb_topdown_multiclass_configure", &p->topdown, form, max_batch, H, W, 0, 0, &mc, &mi);
  if (rc) return rc;
  if (p->topdown.precrop_resize != 0.f && p->topdown.precrop_resize != 1.f)
    return sb_fail(h, SB_ERR_UNSUPPORTED, "sb_topdown_multiclass_configure: instance models trained at an input scale != 1 (precrop_resize %g)",
                   p->topdown.precrop_resize);
  // the tap: a buffer of the instance network holding C logical channels at the offset, in one plane or [lo | hi | hi]
  if (p->tap_buffer < 0 || p->tap_buffer >= (int)mi->buffers.size() || p->tap_channels <= 0 || p->tap_channel_offset < 0 ||
      (p->tap_planes != 1 && p->tap_planes != 3))
    return sb_fail(h, SB_ERR_INVALID, "sb_topdown_multiclass_configure: bad class-vector tap");
  const SbBuffer& tb = mi->buffers[p->tap_buffer];
  const bool half = !(tb.f32 || mi->precision == 1);
  if (p->tap_channel_offset + p->tap_planes * p->tap_channels > tb.C || (p->tap_planes == 3 && !(half && mi->precision == 2)))
    return sb_fail(h, SB_ERR_INVALID, "sb_topdown_multiclass_configure: the tap does not fit its buffer's storage");
  int Hres, Wres, Hnet, Wnet;
  if ((rc = sb_net_size(h, mi, p->topdown.crop_size, p->topdown.crop_size, &Hres, &Wres, &Hnet, &Wnet))) return rc;
  if (Hnet % tb.stride_den || Wnet % tb.stride_den) return sb_fail(h, SB_ERR_INVALID, "crop size not divisible by the tap's stride");
  TdHead d;
  if ((rc = head_from_params(h, p, Hnet / tb.stride_den, Wnet / tb.stride_den, p->tap_channels, d))) return rc;
  // arguments checked: from here the previous chains are dropped
  if ((rc = topdown_setup(h, &p->topdown, form, max_batch, H, W, C_in, mc, mi, p->n_classes, 0, 0))) return rc;
  SbModel* owner = mc ? mc : mi;
  SbTopdown* t = owner->td;
  t->head = d;
  t->tap_buf = p->tap_buffer; t->tap_coff = p->tap_channel_offset; t->tap_hi = p->tap_planes == 3 ? p->tap_channels : 0;
  t->tap_half = half;
  t->all_stores = mi->buf_elided[p->tap_buffer] != 0;       // the rule sb_model_forward follows
  if (cudaMalloc((void**)&t->dense, (size_t)p->n_dense_weights * 4) != cudaSuccess ||
      cudaMemcpy(t->dense, p->dense_weights, (size_t)p->n_dense_weights * 4, cudaMemcpyHostToDevice) != cudaSuccess) {
    sb_topdown_free(owner);
    return sb_fail(h, SB_ERR_CUDA, "sb_topdown_multiclass_configure: dense weights");
  }
  t->head.w = t->dense;
  return SB_OK;
}

int sb_infer_topdown_multiclass(sb_handle_t h, int centroid_model_id, const void* frames_host, int frames_are_u8, int B,
                                float* out_centroids, float* out_centroid_vals, float* out_points, float* out_vals,
                                float* out_class_probs, int32_t* out_n_valid, int32_t* out_flags, float* out_class_vectors) {
  SbTopdown* t = topdown_of(h, centroid_model_id, TD_MODEL, 1, false);
  if (!t) return SB_ERR_INVALID;
  if (const int rc = topdown_call(h, centroid_model_id, t, frames_host, frames_are_u8, B, "sb_infer_topdown_multiclass")) return rc;
  split_topdown_multiclass(t, t->slots.stage[0], t->probs_stage[0], B, out_centroids, out_centroid_vals, out_points, out_vals,
                           out_class_probs, out_n_valid, out_flags, out_class_vectors);
  return SB_OK;
}

int sb_topdown_multiclass_submit(sb_handle_t h, int centroid_model_id, const uint8_t* frames_host, int B, int slot) {
  return topdown_submit(h, centroid_model_id, frames_host, B, slot, true);
}

int sb_topdown_multiclass_collect(sb_handle_t h, int model_id, int slot, int B, float* out_centroids, float* out_centroid_vals,
                                  float* out_points, float* out_vals, float* out_class_probs, int32_t* out_n_valid, int32_t* out_flags,
                                  float* out_class_vectors) {
  SbTopdown* t = topdown_of(h, model_id, TD_MODEL | TD_GT, 1, true);
  if (!t) return SB_ERR_INVALID;
  if (const int rc = topdown_collect(h, model_id, t, slot, B)) return rc;
  split_topdown_multiclass(t, t->slots.stage[slot], t->probs_stage[slot], B, out_centroids, out_centroid_vals, out_points, out_vals,
                           out_class_probs, out_n_valid, out_flags, out_class_vectors);
  return SB_OK;
}

int sb_topdown_multiclass_from_features(sb_handle_t h, const sb_topdown_multiclass_params* p, const float* cms_host, int n_crops, int H,
                                        int W, int n_nodes, const float* offsets_host, const float* features_host, int Hf, int Wf,
                                        int Cf, const float* crop_offsets_host, const int32_t* crop_sample_inds, int B,
                                        float* out_points, float* out_vals, float* out_class_probs, float* out_class_vectors,
                                        float* out_features) {
  if (!h || !p) return sb_fail(h, SB_ERR_INVALID, "null handle / params");
  if ((n_crops > 0 && (!cms_host || !features_host || !crop_sample_inds)) || !out_points || !out_vals || !out_class_probs)
    return sb_fail(h, SB_ERR_INVALID, "sb_topdown_multiclass_from_features: null argument");
  if (n_crops < 0 || B <= 0 || H <= 0 || W <= 0 || n_nodes <= 0 || n_nodes > 256)
    return sb_fail(h, SB_ERR_INVALID, "sb_topdown_multiclass_from_features: bad shape");
  TdHead d;
  int rc = head_from_params(h, p, Hf, Wf, Cf, d);
  if (rc) return rc;
  std::vector<int> count(B, 0), offsets(B + 1, 0);
  for (int i = 0; i < n_crops; ++i) {
    const int b = crop_sample_inds[i];
    if (b < 0 || b >= B || (i > 0 && b < crop_sample_inds[i - 1]))
      return sb_fail(h, SB_ERR_INVALID, "crop sample indices must be non-decreasing in [0, B)");
    ++count[b];
  }
  int K = 1;
  for (int b = 0; b < B; ++b) { offsets[b + 1] = offsets[b] + count[b]; K = std::max(K, count[b]); }
  SB_CUDA(h, cudaSetDevice(h->device));
  const int NC = d.n_classes, nc = std::max(n_crops, 1);
  SbScratch s(h);
  const float *cms = nullptr, *off = nullptr, *feats = nullptr, *coff = nullptr, *dense = nullptr;
  const int *d_count = nullptr, *d_offsets = nullptr;
  float *pts, *vals, *probs, *rec, *fout = nullptr;
  const size_t width = td_class_record_width(NC, n_nodes, K);
  const size_t ncm = (size_t)n_crops * H * W * n_nodes;
  if ((rc = sb_global_scratch_alloc(h, s.gs, nc, H, n_nodes)) || (rc = s.alloc(&pts, (size_t)nc * n_nodes * 2)) ||
      (rc = s.alloc(&vals, (size_t)nc * n_nodes)) || (rc = s.alloc(&probs, (size_t)nc * NC)) || (rc = s.alloc(&rec, (size_t)B * width)) ||
      (out_features && (rc = s.alloc(&fout, (size_t)nc * d.n_in))) ||
      (rc = s.upload(p->dense_weights, (size_t)p->n_dense_weights, &dense)) || (rc = s.upload(count.data(), (size_t)B, &d_count)) ||
      (rc = s.upload(offsets.data(), (size_t)B + 1, &d_offsets)))
    return rc;
  d.w = dense;
  if (n_crops > 0) {
    if ((rc = s.upload(cms_host, ncm, &cms)) || (rc = s.upload(offsets_host, 2 * ncm, &off, true)) ||
        (rc = s.upload(features_host, (size_t)n_crops * Hf * Wf * Cf, &feats)) ||
        (rc = s.upload(crop_offsets_host, (size_t)n_crops * 2, &coff, true)))
      return rc;
    const sb_global_params& gp = p->topdown.instance;
    SbPeakParams pp{gp.peak_threshold, gp.refinement, gp.integral_patch_size, (float)gp.output_stride, gp.input_scale};
    if ((rc = sbk_global_peaks(h, cms, off, n_crops, H, W, n_nodes, pp, coff, s.gs.part, s.gs.chunks, s.gs.rpc, pts, vals)) ||
        (rc = launch_class_vectors(h, feats, false, Cf, 0, d, n_crops, probs, fout)))
      return rc;
  }
  if ((rc = launch_class_assign(h, nullptr, nullptr, d_count, d_offsets, pts, vals, probs, B, K, n_nodes, NC, nullptr, rec))) return rc;
  std::vector<float> records((size_t)B * width);
  if ((rc = s.to_host(records.data(), rec, records.size())) ||
      (n_crops > 0 && (rc = s.to_host(out_class_vectors, probs, (size_t)n_crops * NC, true))) ||
      (n_crops > 0 && (rc = s.to_host(out_features, (const float*)fout, (size_t)n_crops * d.n_in, true))) || (rc = s.sync()))
    return rc;
  const size_t n1 = (size_t)NC * n_nodes;
  sb_split_records(records.data(), B, width, {{out_points, n1 * 2}, {out_vals, n1}, {out_class_probs, (size_t)NC}}, {});
  return SB_OK;
}

}  // extern "C"
