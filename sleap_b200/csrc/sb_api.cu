// C-ABI entry points: handle lifetime and the stage-level (host-buffer) post-processing calls.
// The model / fused-predictor entry points live in sb_model.cu.
#include <stdarg.h>

#include <algorithm>

#include "sb_common.cuh"

thread_local std::string g_sb_last_error;

int sb_fail(sb_handle_s* h, int code, const char* fmt, ...) {
  char buf[1024];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof(buf), fmt, ap);
  va_end(ap);
  g_sb_last_error = buf;
  if (h) h->last_error = buf;
  return code;
}

extern "C" {

int sb_version(void) { return 100; }

int sb_create(int device_id, sb_handle_t* out_handle) {
  if (!out_handle) return sb_fail(nullptr, SB_ERR_INVALID, "sb_create: null out_handle");
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0)
    return sb_fail(nullptr, SB_ERR_NO_DEVICE,
                   "sb_create: no CUDA device (%s); libsleapb200 has no CPU fallback",
                   e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
  if (device_id < 0 || device_id >= n)
    return sb_fail(nullptr, SB_ERR_INVALID, "sb_create: device %d out of range [0,%d)", device_id, n);
  sb_handle_s* h = new sb_handle_s();
  h->device = device_id;
  SB_CUDA(h, cudaSetDevice(device_id));
  cudaDeviceProp prop;
  SB_CUDA(h, cudaGetDeviceProperties(&prop, device_id));
  h->sm_count = prop.multiProcessorCount;
  if (prop.major != 9 || prop.minor != 0)
    fprintf(stderr, "[sleap_b200] warning: device %d is sm_%d%d; kernels are built for sm_90a\n",
            device_id, prop.major, prop.minor);
  SB_CUDA(h, cudaStreamCreateWithFlags(&h->own_stream, cudaStreamNonBlocking));
  h->stream = h->own_stream;
  for (int i = 0; i < 3; ++i) {
    SB_CUDA(h, cudaStreamCreateWithFlags(&h->aux_stream[i], cudaStreamNonBlocking));
    SB_CUDA(h, cudaEventCreateWithFlags(&h->join_ev[i], cudaEventDisableTiming));
  }
  SB_CUDA(h, cudaEventCreateWithFlags(&h->fork_ev, cudaEventDisableTiming));
  SB_CUDA(h, cudaStreamCreateWithFlags(&h->post_stream, cudaStreamNonBlocking));
  SB_CUDA(h, cudaEventCreateWithFlags(&h->fwd_done_ev, cudaEventDisableTiming));
  SB_CUDA(h, cudaEventCreateWithFlags(&h->post_done_ev, cudaEventDisableTiming));
  *out_handle = h;
  return SB_OK;
}

int sb_destroy(sb_handle_t h) {
  if (!h) return SB_OK;
  cudaSetDevice(h->device);
  cudaDeviceSynchronize();
  sb_models_free(h);
  sb_flows_free(h);
  sb_trackers_free(h);
  for (void* p : h->owned) cudaFree(p);
  for (int i = 0; i < 3; ++i) { if (h->aux_stream[i]) cudaStreamDestroy(h->aux_stream[i]); if (h->join_ev[i]) cudaEventDestroy(h->join_ev[i]); }
  if (h->fork_ev) cudaEventDestroy(h->fork_ev);
  if (h->post_stream) cudaStreamDestroy(h->post_stream);
  if (h->fwd_done_ev) cudaEventDestroy(h->fwd_done_ev);
  if (h->post_done_ev) cudaEventDestroy(h->post_done_ev);
  if (h->own_stream) cudaStreamDestroy(h->own_stream);
  delete h;
  return SB_OK;
}

const char* sb_last_error(sb_handle_t h) {
  if (h) return h->last_error.c_str();
  return g_sb_last_error.c_str();
}

int sb_synchronize(sb_handle_t h) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  SB_CUDA(h, cudaStreamSynchronize(h->post_stream));
  h->post_pending = false;
  return SB_OK;
}

int sb_gpu_launches(sb_handle_t h) { return h ? h->gpu_launches : 0; }

int sb_set_stream(sb_handle_t h, void* cuda_stream) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  h->stream = cuda_stream ? (cudaStream_t)cuda_stream : h->own_stream;
  return SB_OK;
}

}  // extern "C"

namespace {

struct DevBuf {  // RAII temporary device buffer for the stage-level calls
  void* p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
  int alloc(sb_handle_s* h, size_t bytes) {
    cudaError_t e = cudaMalloc(&p, bytes ? bytes : 16);
    if (e != cudaSuccess) return sb_fail(h, SB_ERR_CUDA, "cudaMalloc(%zu): %s", bytes, cudaGetErrorString(e));
    return 0;
  }
  template <typename T> T* as() { return (T*)p; }
};

struct WsGuard {
  SbPostWs ws;
  ~WsGuard() { sb_post_ws_free(ws); }
};

#define H2D(h, dst, src, bytes) SB_CUDA(h, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, (h)->stream))
#define D2H(h, dst, src, bytes) SB_CUDA(h, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, (h)->stream))

}  // namespace

extern "C" {

int sb_find_local_peaks(sb_handle_t h, const float* cms_host, int B, int H, int W, int C,
                        float threshold, int refinement, int integral_patch_size,
                        const float* offsets_host, int max_peaks_per_sample, float* out_points,
                        float* out_vals, int32_t* out_sample_inds, int32_t* out_channel_inds,
                        int32_t* out_n_peaks, int32_t* out_flags) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0 || max_peaks_per_sample <= 0)
    return sb_fail(h, SB_ERR_INVALID, "sb_find_local_peaks: bad shape");
  if ((long long)H * W * C >= (1ll << 31)) return sb_fail(h, SB_ERR_UNSUPPORTED, "map too large");
  SB_CUDA(h, cudaSetDevice(h->device));
  WsGuard g;
  int rc = sb_post_ws_alloc(h, g.ws, B, H, W, C, max_peaks_per_sample, 1, 1, 0);
  if (rc) return rc;
  const size_t n = (size_t)B * H * W * C;
  DevBuf d_cms, d_off;
  if ((rc = d_cms.alloc(h, n * sizeof(float)))) return rc;
  H2D(h, d_cms.p, cms_host, n * sizeof(float));
  if (offsets_host) {
    if ((rc = d_off.alloc(h, 2 * n * sizeof(float)))) return rc;
    H2D(h, d_off.p, offsets_host, 2 * n * sizeof(float));
  }
  SbPeakParams p{threshold, refinement, integral_patch_size, 1.0f, 1.0f};
  if ((rc = sbk_local_peaks(h, d_cms.p, 0, offsets_host ? d_off.as<float>() : nullptr, B, H, W, C, p, g.ws))) return rc;
  std::vector<int> cnt(B), flags(B);
  D2H(h, cnt.data(), g.ws.n_peaks, B * sizeof(int));
  D2H(h, flags.data(), g.ws.flags, B * sizeof(int));
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  int total = 0;
  for (int b = 0; b < B; ++b) {
    const int nb = cnt[b];
    if (nb > 0) {
      D2H(h, out_points + 2 * (size_t)total, g.ws.peaks + (size_t)b * max_peaks_per_sample * 2, nb * 2 * sizeof(float));
      D2H(h, out_vals + total, g.ws.peak_vals + (size_t)b * max_peaks_per_sample, nb * sizeof(float));
      D2H(h, out_channel_inds + total, g.ws.peak_ch + (size_t)b * max_peaks_per_sample, nb * sizeof(int));
      for (int i = 0; i < nb; ++i) out_sample_inds[total + i] = b;
    }
    total += nb;
    if (out_flags) out_flags[b] = flags[b];
  }
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  *out_n_peaks = total;
  return SB_OK;
}

int sb_find_global_peaks(sb_handle_t h, const float* cms_host, int B, int H, int W, int C,
                         float threshold, int refinement, int integral_patch_size,
                         const float* offsets_host, float* out_points, float* out_vals) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0) return sb_fail(h, SB_ERR_INVALID, "sb_find_global_peaks: bad shape");
  SB_CUDA(h, cudaSetDevice(h->device));
  const size_t n = (size_t)B * H * W * C;
  int rc;
  DevBuf d_cms, d_off, d_part, d_pts, d_vals;
  int target = (2 * h->sm_count + B - 1) / B;
  int rpc = std::max(1, (H + target - 1) / target);
  const int n_chunks = (H + rpc - 1) / rpc;
  if ((rc = d_cms.alloc(h, n * sizeof(float)))) return rc;
  if ((rc = d_part.alloc(h, (size_t)B * n_chunks * C * 3 * sizeof(float)))) return rc;
  if ((rc = d_pts.alloc(h, (size_t)B * C * 2 * sizeof(float)))) return rc;
  if ((rc = d_vals.alloc(h, (size_t)B * C * sizeof(float)))) return rc;
  H2D(h, d_cms.p, cms_host, n * sizeof(float));
  if (offsets_host) {
    if ((rc = d_off.alloc(h, 2 * n * sizeof(float)))) return rc;
    H2D(h, d_off.p, offsets_host, 2 * n * sizeof(float));
  }
  SbPeakParams p{threshold, refinement, integral_patch_size, 1.0f, 1.0f};
  if ((rc = sbk_global_peaks(h, d_cms.p, 0, offsets_host ? d_off.as<float>() : nullptr, B, H, W, C, p, nullptr,
                             d_part.as<float>(), n_chunks, rpc, d_pts.as<float>(), d_vals.as<float>()))) return rc;
  D2H(h, out_points, d_pts.p, (size_t)B * C * 2 * sizeof(float));
  D2H(h, out_vals, d_vals.p, (size_t)B * C * sizeof(float));
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  return SB_OK;
}

int sb_crop_centered(sb_handle_t h, const void* images_host, int images_are_u8, int B, int H, int W,
                     int C, const float* centroids, const int32_t* sample_inds, int n, int crop_h,
                     int crop_w, void* out_crops) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  if (n <= 0) return SB_OK;
  SB_CUDA(h, cudaSetDevice(h->device));
  const size_t esz = images_are_u8 ? 1 : 4;
  const size_t nimg = (size_t)B * H * W * C * esz, nout = (size_t)n * crop_h * crop_w * C * esz;
  int rc;
  DevBuf d_img, d_c, d_s, d_out;
  if ((rc = d_img.alloc(h, nimg)) || (rc = d_c.alloc(h, (size_t)n * 2 * sizeof(float))) ||
      (rc = d_s.alloc(h, (size_t)n * sizeof(int))) || (rc = d_out.alloc(h, nout))) return rc;
  H2D(h, d_img.p, images_host, nimg);
  H2D(h, d_c.p, centroids, (size_t)n * 2 * sizeof(float));
  H2D(h, d_s.p, sample_inds, (size_t)n * sizeof(int));
  if ((rc = sbk_crop(h, d_img.p, images_are_u8, B, H, W, C, d_c.as<float>(), d_s.as<int>(), n, crop_h, crop_w,
                     d_out.p, images_are_u8))) return rc;
  D2H(h, out_crops, d_out.p, nout);
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  return SB_OK;
}

// Builds the per-node ascending peak lists on the host (stable argsort by channel,
// paf_grouping.py:106-109) for the stage-level calls that receive caller-supplied peaks.
static int upload_peaks(sb_handle_s* h, SbPostWs& ws, int B, int n_nodes, const float* peaks,
                        const float* peak_vals, const int32_t* ch, const int32_t* off) {
  const int K = ws.max_node_peaks, MP = ws.max_peaks;
  std::vector<float> pk((size_t)B * MP * 2, 0.f), pv((size_t)B * MP, 0.f);
  std::vector<int> cnt((size_t)B * n_nodes, 0), lst((size_t)B * n_nodes * K, 0), np(B, 0);
  for (int b = 0; b < B; ++b) {
    const int n = off[b + 1] - off[b];
    np[b] = n;
    for (int i = 0; i < n; ++i) {
      pk[((size_t)b * MP + i) * 2] = peaks[2 * (size_t)(off[b] + i)];
      pk[((size_t)b * MP + i) * 2 + 1] = peaks[2 * (size_t)(off[b] + i) + 1];
      if (peak_vals) pv[(size_t)b * MP + i] = peak_vals[off[b] + i];
      const int c = ch[off[b] + i];
      if (c < 0 || c >= n_nodes) return sb_fail(h, SB_ERR_INVALID, "peak channel %d out of range", c);
      int& k = cnt[(size_t)b * n_nodes + c];
      lst[((size_t)b * n_nodes + c) * K + k] = i;
      ++k;
    }
  }
  H2D(h, ws.peaks, pk.data(), pk.size() * sizeof(float));
  H2D(h, ws.peak_vals, pv.data(), pv.size() * sizeof(float));
  H2D(h, ws.node_cnt, cnt.data(), cnt.size() * sizeof(int));
  H2D(h, ws.node_peaks, lst.data(), lst.size() * sizeof(int));
  H2D(h, ws.n_peaks, np.data(), np.size() * sizeof(int));
  SB_CUDA(h, cudaMemsetAsync(ws.flags, 0, B * sizeof(int), h->stream));
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  return 0;
}

static void node_caps(int B, int n_nodes, const int32_t* ch, const int32_t* off, int* max_peaks, int* max_node) {
  int mp = 1, mk = 1;
  std::vector<int> cnt(n_nodes);
  for (int b = 0; b < B; ++b) {
    std::fill(cnt.begin(), cnt.end(), 0);
    mp = std::max(mp, off[b + 1] - off[b]);
    for (int i = off[b]; i < off[b + 1]; ++i)
      if (ch[i] >= 0 && ch[i] < n_nodes) mk = std::max(mk, ++cnt[ch[i]]);
  }
  *max_peaks = mp; *max_node = mk;
}

int sb_score_paf_lines_batch(sb_handle_t h, const float* pafs_host, int B, int Hp, int Wp, int C2,
                             const float* peaks, const int32_t* peak_channel_inds,
                             const int32_t* peak_offsets, const int32_t* skeleton_edges, int n_edges,
                             int n_nodes, int n_line_points, int pafs_stride,
                             float max_edge_length_ratio, float dist_penalty_weight, int cap,
                             int32_t* out_edge_inds, int32_t* out_edge_peak_inds,
                             float* out_line_scores, int32_t* out_cand_offsets) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  if (B <= 0 || n_edges <= 0 || n_nodes <= 0) return sb_fail(h, SB_ERR_INVALID, "sb_score_paf_lines_batch: bad shape");
  SB_CUDA(h, cudaSetDevice(h->device));
  int MP, K;
  node_caps(B, n_nodes, peak_channel_inds, peak_offsets, &MP, &K);
  WsGuard g;
  int rc = sb_post_ws_alloc(h, g.ws, B, 1, 1, n_nodes, MP, K, 1, n_edges);
  if (rc) return rc;
  if ((rc = upload_peaks(h, g.ws, B, n_nodes, peaks, nullptr, peak_channel_inds, peak_offsets))) return rc;
  H2D(h, g.ws.edges_dev, skeleton_edges, (size_t)n_edges * 2 * sizeof(int));
  DevBuf d_pafs;
  const size_t npaf = (size_t)B * Hp * Wp * C2;
  if ((rc = d_pafs.alloc(h, npaf * sizeof(float)))) return rc;
  H2D(h, d_pafs.p, pafs_host, npaf * sizeof(float));
  // max_edge_length = ratio * max(Hp, Wp, C2) * stride  (paf_grouping.py:469-473), in f32
  const float max_len = max_edge_length_ratio * (float)std::max(std::max(Hp, Wp), C2) * (float)pafs_stride;
  if ((rc = sbk_score_match(h, d_pafs.as<float>(), B, Hp, Wp, C2, n_line_points, pafs_stride, max_len,
                            dist_penalty_weight, g.ws))) return rc;
  std::vector<float> mat((size_t)B * n_edges * K * K);
  D2H(h, mat.data(), g.ws.score_mat, mat.size() * sizeof(float));
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  // flatten: (sample, edge, src-major) using the same node lists
  int total = 0;
  std::vector<std::vector<int>> lists(n_nodes);
  for (int b = 0; b < B; ++b) {
    out_cand_offsets[b] = total;
    for (auto& l : lists) l.clear();
    for (int i = peak_offsets[b]; i < peak_offsets[b + 1]; ++i) lists[peak_channel_inds[i]].push_back(i - peak_offsets[b]);
    for (int e = 0; e < n_edges; ++e) {
      const auto& s = lists[skeleton_edges[2 * e]];
      const auto& d = lists[skeleton_edges[2 * e + 1]];
      const int nd = (int)d.size();
      for (size_t i = 0; i < s.size(); ++i)
        for (int j = 0; j < nd; ++j) {
          if (total >= cap) return sb_fail(h, SB_ERR_INVALID, "candidate capacity %d exceeded", cap);
          out_edge_inds[total] = e;
          out_edge_peak_inds[2 * total] = s[i];
          out_edge_peak_inds[2 * total + 1] = d[j];
          out_line_scores[total] = mat[((size_t)b * n_edges + e) * K * K + i * nd + j];
          ++total;
        }
    }
  }
  out_cand_offsets[B] = total;
  return SB_OK;
}

int sb_paf_lines(sb_handle_t h, const float* pafs_sample, int Hp, int Wp, int C2,
                 const float* lines_in, const float* peaks, int n_peaks,
                 const int32_t* edge_peak_inds, const int32_t* edge_inds, int n, int n_line_points,
                 int pafs_stride, float max_edge_length, float dist_penalty_weight,
                 int32_t* out_subs, float* out_lines, float* out_scores) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  if (n <= 0) return SB_OK;
  if (n_line_points <= 0 || n_peaks <= 0) return sb_fail(h, SB_ERR_INVALID, "sb_paf_lines: bad sizes");
  for (int i = 0; i < 2 * n; ++i)
    if (edge_peak_inds[i] < 0 || edge_peak_inds[i] >= n_peaks) return sb_fail(h, SB_ERR_INVALID, "peak index out of range");
  SB_CUDA(h, cudaSetDevice(h->device));
  int rc;
  const size_t P = n_line_points;
  DevBuf d_paf, d_lin, d_pk, d_epi, d_ei, d_subs, d_ol, d_os;
  if (pafs_sample) {
    if ((rc = d_paf.alloc(h, (size_t)Hp * Wp * C2 * 4))) return rc;
    H2D(h, d_paf.p, pafs_sample, (size_t)Hp * Wp * C2 * 4);
  }
  if (lines_in) {
    if ((rc = d_lin.alloc(h, (size_t)n * P * 2 * 4))) return rc;
    H2D(h, d_lin.p, lines_in, (size_t)n * P * 2 * 4);
  }
  if ((rc = d_pk.alloc(h, (size_t)n_peaks * 2 * 4)) || (rc = d_epi.alloc(h, (size_t)n * 2 * 4)) ||
      (rc = d_ei.alloc(h, (size_t)n * 4)) || (rc = d_subs.alloc(h, (size_t)n * P * 2 * 4)) ||
      (rc = d_ol.alloc(h, (size_t)n * P * 2 * 4)) || (rc = d_os.alloc(h, (size_t)n * 4))) return rc;
  H2D(h, d_pk.p, peaks, (size_t)n_peaks * 2 * 4);
  H2D(h, d_epi.p, edge_peak_inds, (size_t)n * 2 * 4);
  if (edge_inds) H2D(h, d_ei.p, edge_inds, (size_t)n * 4);
  if ((rc = sbk_lines(h, pafs_sample ? d_paf.as<float>() : nullptr, Hp, Wp, C2, lines_in ? d_lin.as<float>() : nullptr,
                      d_pk.as<float>(), d_epi.as<int>(), edge_inds ? d_ei.as<int>() : nullptr, n, n_line_points,
                      (float)pafs_stride, max_edge_length, dist_penalty_weight, d_subs.as<int>(), d_ol.as<float>(),
                      d_os.as<float>()))) return rc;
  if (out_subs) D2H(h, out_subs, d_subs.p, (size_t)n * P * 2 * 4);
  if (out_lines) D2H(h, out_lines, d_ol.p, (size_t)n * P * 2 * 4);
  if (out_scores) D2H(h, out_scores, d_os.p, (size_t)n * 4);
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  return SB_OK;
}

int sb_integral_regression(sb_handle_t h, const float* cms, int N, int Hh, int Ww, int C,
                           const float* xv, const float* yv, float* x_hat, float* y_hat) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  if (N <= 0) return SB_OK;
  SB_CUDA(h, cudaSetDevice(h->device));
  int rc;
  DevBuf d_c, d_x, d_y, d_ox, d_oy;
  const size_t n = (size_t)N * Hh * Ww * C;
  if ((rc = d_c.alloc(h, n * 4)) || (rc = d_x.alloc(h, Ww * 4)) || (rc = d_y.alloc(h, Hh * 4)) ||
      (rc = d_ox.alloc(h, (size_t)N * C * 4)) || (rc = d_oy.alloc(h, (size_t)N * C * 4))) return rc;
  H2D(h, d_c.p, cms, n * 4);
  H2D(h, d_x.p, xv, Ww * 4);
  H2D(h, d_y.p, yv, Hh * 4);
  if ((rc = sbk_integral(h, d_c.as<float>(), N, Hh, Ww, C, d_x.as<float>(), d_y.as<float>(), d_ox.as<float>(), d_oy.as<float>()))) return rc;
  D2H(h, x_hat, d_ox.p, (size_t)N * C * 4);
  D2H(h, y_hat, d_oy.p, (size_t)N * C * 4);
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  return SB_OK;
}

int sb_find_offsets_local_direction(sb_handle_t h, const float* patches, int N, float delta,
                                    float* out_offsets) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  if (N <= 0) return SB_OK;
  SB_CUDA(h, cudaSetDevice(h->device));
  int rc;
  DevBuf d_p, d_o;
  if ((rc = d_p.alloc(h, (size_t)N * 9 * 4)) || (rc = d_o.alloc(h, (size_t)N * 2 * 4))) return rc;
  H2D(h, d_p.p, patches, (size_t)N * 9 * 4);
  if ((rc = sbk_local_dir(h, d_p.as<float>(), N, delta, d_o.as<float>()))) return rc;
  D2H(h, out_offsets, d_o.p, (size_t)N * 2 * 4);
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  return SB_OK;
}

int sb_linear_sum_assignment_batch(sb_handle_t h, const float* scores, const int32_t* n_src,
                                   const int32_t* n_dst, const int32_t* offsets, int n_problems,
                                   int max_k, int32_t* out_rows, int32_t* out_cols,
                                   float* out_scores, int32_t* out_counts) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  if (n_problems <= 0) return SB_OK;
  SB_CUDA(h, cudaSetDevice(h->device));
  size_t total = 0;
  for (int p = 0; p < n_problems; ++p) {
    if (n_src[p] > max_k || n_dst[p] > max_k) return sb_fail(h, SB_ERR_INVALID, "problem %d exceeds max_k", p);
    total = std::max(total, (size_t)offsets[p] + (size_t)n_src[p] * n_dst[p]);
  }
  int rc;
  DevBuf d_sc, d_ns, d_nd, d_of, d_r, d_c, d_s, d_n;
  const size_t np = (size_t)n_problems;
  if ((rc = d_sc.alloc(h, total * sizeof(float))) || (rc = d_ns.alloc(h, np * 4)) || (rc = d_nd.alloc(h, np * 4)) ||
      (rc = d_of.alloc(h, np * 4)) || (rc = d_r.alloc(h, np * max_k * 4)) || (rc = d_c.alloc(h, np * max_k * 4)) ||
      (rc = d_s.alloc(h, np * max_k * 4)) || (rc = d_n.alloc(h, np * 4))) return rc;
  H2D(h, d_sc.p, scores, total * sizeof(float));
  H2D(h, d_ns.p, n_src, np * 4);
  H2D(h, d_nd.p, n_dst, np * 4);
  H2D(h, d_of.p, offsets, np * 4);
  if ((rc = sbk_lsap_batch(h, d_sc.as<float>(), d_ns.as<int>(), d_nd.as<int>(), d_of.as<int>(), n_problems, max_k,
                           d_r.as<int>(), d_c.as<int>(), d_s.as<float>(), d_n.as<int>()))) return rc;
  D2H(h, out_rows, d_r.p, np * max_k * 4);
  D2H(h, out_cols, d_c.p, np * max_k * 4);
  D2H(h, out_scores, d_s.p, np * max_k * 4);
  D2H(h, out_counts, d_n.p, np * 4);
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  return SB_OK;
}

int sb_group_instances_batch(sb_handle_t h, int B, int n_nodes, const float* peaks,
                             const float* peak_vals, const int32_t* peak_channel_inds,
                             const int32_t* peak_offsets, const int32_t* match_edge_inds,
                             const int32_t* match_src_peak_inds, const int32_t* match_dst_peak_inds,
                             const float* match_line_scores, const int32_t* match_offsets,
                             const int32_t* edge_types, int n_edges, const int32_t* sorted_edge_inds,
                             int n_sorted, int min_instance_peaks, float min_line_scores,
                             int max_instances, float* out_instances, float* out_peak_scores,
                             float* out_instance_scores, int32_t* out_n_instances) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  if (B <= 0 || n_nodes <= 0 || n_edges <= 0 || max_instances <= 0)
    return sb_fail(h, SB_ERR_INVALID, "sb_group_instances_batch: bad shape");
  SB_CUDA(h, cudaSetDevice(h->device));
  int MP, K;
  node_caps(B, n_nodes, peak_channel_inds, peak_offsets, &MP, &K);
  // K must also cover the largest per-edge match count and every referenced local index
  std::vector<int> ecnt((size_t)B * n_edges, 0);
  for (int b = 0; b < B; ++b)
    for (int m = match_offsets[b]; m < match_offsets[b + 1]; ++m) {
      const int e = match_edge_inds[m];
      if (e < 0 || e >= n_edges) return sb_fail(h, SB_ERR_INVALID, "match edge %d out of range", e);
      K = std::max(K, ++ecnt[(size_t)b * n_edges + e]);
      K = std::max(K, std::max(match_src_peak_inds[m], match_dst_peak_inds[m]) + 1);
    }
  WsGuard g;
  int rc = sb_post_ws_alloc(h, g.ws, B, 1, 1, n_nodes, MP, K, max_instances, n_edges);
  if (rc) return rc;
  if ((rc = upload_peaks(h, g.ws, B, n_nodes, peaks, peak_vals, peak_channel_inds, peak_offsets))) return rc;
  std::vector<int> msrc((size_t)B * n_edges * K, 0), mdst((size_t)B * n_edges * K, 0);
  std::vector<float> msc((size_t)B * n_edges * K, 0.f);
  std::fill(ecnt.begin(), ecnt.end(), 0);
  for (int b = 0; b < B; ++b)
    for (int m = match_offsets[b]; m < match_offsets[b + 1]; ++m) {
      const int e = match_edge_inds[m];
      int& k = ecnt[(size_t)b * n_edges + e];
      const size_t o = ((size_t)b * n_edges + e) * K + k;
      msrc[o] = match_src_peak_inds[m];
      mdst[o] = match_dst_peak_inds[m];
      msc[o] = match_line_scores[m];
      ++k;
    }
  H2D(h, g.ws.match_cnt, ecnt.data(), ecnt.size() * 4);
  H2D(h, g.ws.match_src, msrc.data(), msrc.size() * 4);
  H2D(h, g.ws.match_dst, mdst.data(), mdst.size() * 4);
  H2D(h, g.ws.match_score, msc.data(), msc.size() * 4);
  H2D(h, g.ws.edges_dev, edge_types, (size_t)n_edges * 2 * 4);
  if (n_sorted > n_edges) return sb_fail(h, SB_ERR_INVALID, "n_sorted > n_edges");
  if (n_sorted > 0) H2D(h, g.ws.sorted_edges_dev, sorted_edge_inds, (size_t)n_sorted * 4);
  g.ws.n_sorted = n_sorted;
  // Note: stage-level peaks lists hold *all* peaks of a node, so node_cnt >= every local index.
  if ((rc = sbk_group(h, B, n_nodes, min_instance_peaks, min_line_scores, 1.0f, g.ws))) return rc;
  D2H(h, out_instances, g.ws.inst_peaks, (size_t)B * max_instances * n_nodes * 2 * 4);
  D2H(h, out_peak_scores, g.ws.inst_vals, (size_t)B * max_instances * n_nodes * 4);
  D2H(h, out_instance_scores, g.ws.inst_scores, (size_t)B * max_instances * 4);
  D2H(h, out_n_instances, g.ws.n_inst, (size_t)B * 4);
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  return SB_OK;
}

}  // extern "C"
