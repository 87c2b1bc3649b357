// Fused top-down pipeline on the device: frames -> centroid network -> local peaks -> per-frame top-k ->
// crops of the RESIDENT frames -> centered-instance network -> global peaks (+ crop offsets) -> dense per-frame record.
// One H2D copy of the frames and one D2H copy of the results per batch (+ a 4-byte crop count).
//
// Reference: TopDownInferenceModel.call (sleap/nn/inference.py:2273-2311) = CentroidCrop.call (:1747-1966: network,
// find_local_peaks, /input_scale + 0.5, tf.math.top_k(max_instances) :1879-1894, crop_bboxes on the full frames :1918-1927)
// followed by FindInstancePeaks.call (:2059-2200: network on the crops, find_global_peaks, + crop_offsets).
// Round 1 ran these as separate host-facing calls: centroids D2H -> host top-k -> frames H2D again -> crops D2H ->
// crops H2D -> instance network (sleap_b200/nn/inference.py CentroidCrop / FindInstancePeaks, kept for the stage-level
// surface and for models that need a pre-crop resize).
#include <algorithm>
#include <time.h>

#include <math_constants.h>

#include "sb_common.cuh"
#include "sb_model.h"

namespace {

// Per frame: keep all centroids in tf.where order, or -- more than max_instances -- the max_instances most confident ones
// in tf.math.top_k order (descending value, ties: lower index first).  K = capacity of the dense outputs.
__global__ void __launch_bounds__(128) k_td_select(const float* __restrict__ peaks, const float* __restrict__ peak_vals,
                                                   const int* __restrict__ n_peaks, int max_peaks, int max_instances, int K,
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
      sel_cent[((size_t)b * K + pos) * 2] = pk[2 * i];
      sel_cent[((size_t)b * K + pos) * 2 + 1] = pk[2 * i + 1];
      sel_val[(size_t)b * K + pos] = pv[i];
    }
  }
  if (threadIdx.x == 0) {
    sel_count[b] = min(keep, K);
    if (keep > K) atomicOr(&flags[b], SB_FLAG_INSTANCES_TRUNCATED);
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

// Dense per-frame record: [K][2] centroids | [K] centroid values | [K][nodes][2] peaks | [K][nodes] peak values | n_valid | flags
__global__ void __launch_bounds__(128) k_td_pack(const float* __restrict__ sel_cent, const float* __restrict__ sel_val,
                                                 const int* __restrict__ sel_count, const int* __restrict__ offsets,
                                                 const float* __restrict__ ipts, const float* __restrict__ ivals, int K, int nodes,
                                                 const int* __restrict__ flags, float* __restrict__ record, int width) {
  const int b = blockIdx.x;
  const int cnt = sel_count[b], o = offsets[b];
  float* r = record + (size_t)b * width;
  float* rc = r;
  float* rv = rc + K * 2;
  float* rp = rv + K;
  float* rq = rp + (size_t)K * nodes * 2;
  for (int t = threadIdx.x; t < K * 2; t += blockDim.x) rc[t] = (t / 2 < cnt) ? sel_cent[(size_t)b * K * 2 + t] : CUDART_NAN_F;
  for (int t = threadIdx.x; t < K; t += blockDim.x) rv[t] = (t < cnt) ? sel_val[(size_t)b * K + t] : CUDART_NAN_F;
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

}  // namespace

struct SbTopdown {
  sb_topdown_params p{};
  SbModel* inst = nullptr;
  unsigned gen_c = 0, gen_i = 0;    // chain_gen of the centroid and the instance model when it was configured
  int K = 0, nodes = 0, width = 0, Bmax = 0, crop_elem = 1;
  float *sel_cent = nullptr, *sel_val = nullptr, *flat_cent = nullptr, *flat_off = nullptr, *ipts = nullptr, *ivals = nullptr, *record = nullptr;
  int *sel_count = nullptr, *flat_sample = nullptr, *offsets = nullptr, *total = nullptr;
  void* crops = nullptr;
  float* record_host = nullptr;
  int* total_host = nullptr;
};

void sb_topdown_free(SbModel* m) {
  SbTopdown* t = m->td;
  if (!t) return;
  void* dev[] = {t->sel_cent, t->sel_val, t->flat_cent, t->flat_off, t->ipts, t->ivals, t->record, t->sel_count, t->flat_sample, t->offsets, t->total, t->crops};
  for (void* p : dev) if (p) cudaFree(p);
  if (t->record_host) cudaFreeHost(t->record_host);
  if (t->total_host) cudaFreeHost(t->total_host);
  delete t;
  m->td = nullptr;
}

extern "C" {

int sb_topdown_configure(sb_handle_t h, const sb_topdown_params* p, int max_batch, int H, int W, int C_in) {
  if (!h || !p) return sb_fail(h, SB_ERR_INVALID, "sb_topdown_configure: null argument");
  static const char* const bad_ids = "sb_topdown_configure: bad model ids";
  SbModel* mc = chain_model(h, p->centroid_model, SB_CHAIN_ANY, bad_ids);
  SbModel* mi = chain_model(h, p->instance_model, SB_CHAIN_ANY, bad_ids);
  if (!mc || !mi || mc == mi) return sb_fail(h, SB_ERR_INVALID, bad_ids);
  if (p->crop_size <= 0 || p->max_centroids_per_frame <= 0 || p->max_crops_per_call <= 0 || max_batch <= 0)
    return sb_fail(h, SB_ERR_INVALID, "sb_topdown_configure: bad sizes");
  if (max_batch > 1024) return sb_fail(h, SB_ERR_UNSUPPORTED, "sb_topdown_configure: more than 1024 frames per batch");
  SB_CUDA(h, cudaSetDevice(h->device));
  int rc;
  if ((rc = sb_model_configure(h, p->centroid_model, max_batch, H, W, C_in))) return rc;
  if ((rc = sb_model_configure(h, p->instance_model, p->max_crops_per_call, p->crop_size, p->crop_size, C_in))) return rc;
  if ((rc = sb_centroid_configure(h, p->centroid_model, &p->centroid))) return rc;
  if ((rc = sb_global_configure(h, p->instance_model, &p->instance))) return rc;
  SbTopdown* t = new SbTopdown();           // the centroid configure dropped the previous one
  mc->td = t;
  t->p = *p; t->inst = mi; t->K = p->max_centroids_per_frame; t->Bmax = max_batch;
  t->gen_c = mc->chain_gen; t->gen_i = mi->chain_gen;
  t->nodes = mi->buffers[p->instance.cms_buffer].C;
  t->width = t->K * (3 + t->nodes * 3) + 2;
  t->crop_elem = 1;                                                    // uint8 frames (float frames: 4, decided per call)
  const size_t N = (size_t)max_batch * t->K;
  auto A = [&](void** q, size_t bytes) { return cudaMalloc(q, bytes + 16) == cudaSuccess; };
  const bool ok = A((void**)&t->sel_cent, N * 2 * 4) && A((void**)&t->sel_val, N * 4) && A((void**)&t->sel_count, (size_t)max_batch * 4) &&
                  A((void**)&t->flat_cent, N * 2 * 4) && A((void**)&t->flat_off, N * 2 * 4) && A((void**)&t->flat_sample, N * 4) &&
                  A((void**)&t->offsets, ((size_t)max_batch + 1) * 4) && A((void**)&t->total, 4) &&
                  A((void**)&t->ipts, N * t->nodes * 2 * 4) && A((void**)&t->ivals, N * t->nodes * 4) &&
                  A((void**)&t->record, (size_t)max_batch * t->width * 4) &&
                  A(&t->crops, (size_t)p->max_crops_per_call * p->crop_size * p->crop_size * C_in * 4);
  if (!ok || cudaHostAlloc((void**)&t->record_host, (size_t)max_batch * t->width * 4, cudaHostAllocDefault) != cudaSuccess ||
      cudaHostAlloc((void**)&t->total_host, 4, cudaHostAllocDefault) != cudaSuccess) {
    sb_topdown_free(mc);
    return sb_fail(h, SB_ERR_CUDA, "sb_topdown_configure: allocation failed");
  }
  return SB_OK;
}

int sb_infer_topdown(sb_handle_t h, int centroid_model_id, const void* frames_host, int frames_are_u8, int B, float* out_centroids,
                     float* out_centroid_vals, float* out_instance_peaks, float* out_instance_peak_vals, int32_t* out_n_valid,
                     int32_t* out_flags) {
  SbModel* mc = chain_model(h, centroid_model_id, SB_CHAIN_ANY, "top-down pipeline not configured");
  if (!mc || !mc->td) return sb_fail(h, SB_ERR_INVALID, "top-down pipeline not configured");
  SbTopdown* t = mc->td;
  SbModel* mi = t->inst;
  // a configure call on either model outside sb_topdown_configure moved its chain_gen (sb_model_configure included)
  if (mc->chain != SB_CHAIN_CENTROID || mc->chain_gen != t->gen_c || mi->chain != SB_CHAIN_GLOBAL || mi->chain_gen != t->gen_i)
    return sb_fail(h, SB_ERR_INVALID, "top-down pipeline: a model was reconfigured; call sb_topdown_configure again");
  if (B <= 0 || B > t->Bmax || B > mc->B) return sb_fail(h, SB_ERR_INVALID, "bad batch");
  SB_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t s = h->stream;
  const size_t esz = frames_are_u8 ? 1 : 4;
  static const bool dbg = getenv("SB_DEBUG_TD") != nullptr;      // stage timing (host clock around stream syncs), profiling only
  auto now = []() { timespec t; clock_gettime(CLOCK_MONOTONIC, &t); return t.tv_sec * 1e3 + t.tv_nsec * 1e-6; };
  double t0 = now(), t1 = 0, t2 = 0, t3 = 0;
  SB_CUDA(h, cudaMemcpyAsync(mc->frames_dev, frames_host, (size_t)B * mc->Hin * mc->Win * mc->Cin * esz, cudaMemcpyHostToDevice, s));
  if (dbg) { cudaStreamSynchronize(s); t1 = now(); }
  int rc = sb_run_ops(h, mc, mc->frames_dev, frames_are_u8, B);
  if (rc) return rc;
  const sb_centroid_params& cp = mc->ce;
  SbBuffer& cb = mc->buffers[cp.cms_buffer];
  const float* coff = cp.offsets_buffer >= 0 ? (const float*)mc->buffers[cp.offsets_buffer].dev : nullptr;
  SbPeakParams pc{cp.peak_threshold, cp.refinement, cp.integral_patch_size, (float)cp.output_stride, cp.input_scale};
  if ((rc = sbk_local_peaks(h, (const float*)cb.dev, coff, B, cb.H, cb.W, cb.C, pc, mc->ws))) return rc;
  k_td_select<<<B, 128, 0, s>>>(mc->ws.peaks, mc->ws.peak_vals, mc->ws.n_peaks, mc->ws.max_peaks, t->p.max_instances, t->K, t->sel_cent,
                                t->sel_val, t->sel_count, mc->ws.flags);
  SB_CHECK_LAUNCH(h);
  k_td_flatten<<<1, 256, 0, s>>>(t->sel_cent, t->sel_count, B, t->K, (float)t->p.crop_size * 0.5f, t->flat_cent, t->flat_off,
                                 t->flat_sample, t->offsets, t->total);
  SB_CHECK_LAUNCH(h);
  SB_CUDA(h, cudaMemcpyAsync(t->total_host, t->total, 4, cudaMemcpyDeviceToHost, s));
  SB_CUDA(h, cudaStreamSynchronize(s));                     // the one mid-pipeline sync: how many crops the instance net runs on
  const int total = *t->total_host;
  if (dbg) t2 = now();
  const sb_global_params& gp = mi->gl;
  SbBuffer& ib = mi->buffers[gp.cms_buffer];
  const float* ioff = gp.offsets_buffer >= 0 ? (const float*)mi->buffers[gp.offsets_buffer].dev : nullptr;
  SbPeakParams pi{gp.peak_threshold, gp.refinement, gp.integral_patch_size, (float)gp.output_stride, gp.input_scale};
  const int cs = t->p.crop_size;
  for (int c0 = 0; c0 < total; c0 += mi->B) {
    const int n = std::min(mi->B, total - c0);
    // crops of the frames already resident in HBM (uint8 frames: float -> uint8 truncation, as tf.cast in crop_bboxes)
    if ((rc = sbk_crop(h, mc->frames_dev, frames_are_u8, B, mc->Hin, mc->Win, mc->Cin, t->flat_cent + 2 * (size_t)c0, t->flat_sample + c0, n,
                       cs, cs, t->crops, frames_are_u8))) return rc;
    if ((rc = sb_run_ops(h, mi, t->crops, frames_are_u8, n))) return rc;
    if ((rc = sbk_global_peaks(h, (const float*)ib.dev, ioff, n, ib.H, ib.W, ib.C, pi, t->flat_off + 2 * (size_t)c0, mi->gs.part, mi->gs.chunks, mi->gs.rpc,
                               t->ipts + (size_t)c0 * t->nodes * 2, t->ivals + (size_t)c0 * t->nodes))) return rc;
  }
  k_td_pack<<<B, 128, 0, s>>>(t->sel_cent, t->sel_val, t->sel_count, t->offsets, t->ipts, t->ivals, t->K, t->nodes, mc->ws.flags, t->record,
                              t->width);
  SB_CHECK_LAUNCH(h);
  SB_CUDA(h, cudaMemcpyAsync(t->record_host, t->record, (size_t)B * t->width * 4, cudaMemcpyDeviceToHost, s));
  SB_CUDA(h, cudaStreamSynchronize(s));
  if (dbg) {
    t3 = now();
    fprintf(stderr, "[sb_infer_topdown] B=%d crops=%d: H2D %.3f ms, centroid stage %.3f ms, instance stage + D2H %.3f ms\n", B, total, t1 - t0,
            t2 - t1, t3 - t2);
  }
  const size_t K = t->K, nd = t->nodes;
  sb_split_records(t->record_host, B, t->width,
                   {{out_centroids, K * 2}, {out_centroid_vals, K}, {out_instance_peaks, K * nd * 2}, {out_instance_peak_vals, K * nd}},
                   {out_n_valid, out_flags});
  return SB_OK;
}

}  // extern "C"
