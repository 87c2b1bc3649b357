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

int sb_peaks_to_host(sb_handle_s* h, const SbPostWs& ws, int B, float* out_points, float* out_vals, int32_t* out_channel_inds,
                     int32_t* out_sample_inds, int32_t* out_n, int32_t* out_flags) {
  SbScratch s(h);
  std::vector<int> cnt(B), flags(B);
  int rc;
  if ((rc = s.to_host(cnt.data(), ws.n_peaks, (size_t)B)) || (rc = s.to_host(flags.data(), ws.flags, (size_t)B)) || (rc = s.sync()))
    return rc;
  const size_t MP = ws.max_peaks;
  int total = 0;
  for (int b = 0; b < B; ++b) {
    const size_t nb = cnt[b];
    if (nb > 0) {
      if ((rc = s.to_host(out_points + 2 * (size_t)total, ws.peaks + b * MP * 2, nb * 2)) ||
          (rc = s.to_host(out_vals + total, ws.peak_vals + b * MP, nb)) ||
          (rc = s.to_host(out_channel_inds ? out_channel_inds + total : nullptr, ws.peak_ch + b * MP, nb, true)))
        return rc;
      for (size_t i = 0; i < nb; ++i) out_sample_inds[total + i] = b;
    }
    total += cnt[b];
    if (out_flags) out_flags[b] = flags[b];
  }
  *out_n = total;
  return s.sync();
}

// sb_crop_centered (resized: false) and sb_crop_centered_resized (the frames resized to Hr x Wr) on host arrays
static int crop_centered(sb_handle_s* h, const void* images_host, int images_are_u8, int B, int H, int W, int C,
                         const float* centroids, const int32_t* sample_inds, int n, int crop_h, int crop_w, bool resized, int Hr,
                         int Wr, void* out_crops) {
  if (n <= 0) return SB_OK;
  SB_CUDA(h, cudaSetDevice(h->device));
  const size_t esz = images_are_u8 ? 1 : 4;
  const size_t nimg = (size_t)B * H * W * C * esz, nout = (size_t)n * crop_h * crop_w * C * esz;
  SbScratch s(h);
  const uint8_t* d_img;
  const float* d_c;
  const int* d_s;
  uint8_t* d_out;
  int rc;
  if ((rc = s.upload((const uint8_t*)images_host, nimg, &d_img)) || (rc = s.upload(centroids, (size_t)n * 2, &d_c)) ||
      (rc = s.upload(sample_inds, (size_t)n, &d_s)) || (rc = s.alloc(&d_out, nout)) ||
      (rc = resized ? sbk_crop_resized(h, d_img, images_are_u8, B, H, W, C, Hr, Wr, d_c, d_s, n, crop_h, crop_w, d_out)
                    : sbk_crop(h, d_img, images_are_u8, B, H, W, C, d_c, d_s, n, crop_h, crop_w, d_out, images_are_u8)) ||
      (rc = s.to_host((uint8_t*)out_crops, d_out, nout)))
    return rc;
  return s.sync();
}

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
  SbScratch s(h);
  const size_t n = (size_t)B * H * W * C;
  const float *d_cms, *d_off;
  int rc = sb_post_ws_alloc(h, s.ws, B, H, W, C, max_peaks_per_sample, 1, 1, 0);
  if (rc || (rc = s.upload(cms_host, n, &d_cms)) || (rc = s.upload(offsets_host, 2 * n, &d_off, true))) return rc;
  SbPeakParams p{threshold, refinement, integral_patch_size, 1.0f, 1.0f};
  if ((rc = sbk_local_peaks(h, d_cms, d_off, B, H, W, C, p, s.ws))) return rc;
  return sb_peaks_to_host(h, s.ws, B, out_points, out_vals, out_channel_inds, out_sample_inds, out_n_peaks, out_flags);
}

int sb_find_global_peaks(sb_handle_t h, const float* cms_host, int B, int H, int W, int C,
                         float threshold, int refinement, int integral_patch_size,
                         const float* offsets_host, float* out_points, float* out_vals) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  if (B <= 0 || H <= 0 || W <= 0 || C <= 0) return sb_fail(h, SB_ERR_INVALID, "sb_find_global_peaks: bad shape");
  SB_CUDA(h, cudaSetDevice(h->device));
  SbScratch s(h);
  const size_t n = (size_t)B * H * W * C;
  const float *d_cms, *d_off;
  int rc = sb_global_scratch_alloc(h, s.gs, B, H, C);
  if (rc || (rc = s.upload(cms_host, n, &d_cms)) || (rc = s.upload(offsets_host, 2 * n, &d_off, true))) return rc;
  SbPeakParams p{threshold, refinement, integral_patch_size, 1.0f, 1.0f};
  const SbGlobalScratch& g = s.gs;
  if ((rc = sbk_global_peaks(h, d_cms, d_off, B, H, W, C, p, nullptr, g.part, g.chunks, g.rpc, g.points, g.vals)) ||
      (rc = s.to_host(out_points, g.points, (size_t)B * C * 2)) || (rc = s.to_host(out_vals, g.vals, (size_t)B * C)))
    return rc;
  return s.sync();
}

int sb_crop_centered(sb_handle_t h, const void* images_host, int images_are_u8, int B, int H, int W,
                     int C, const float* centroids, const int32_t* sample_inds, int n, int crop_h,
                     int crop_w, void* out_crops) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  return crop_centered(h, images_host, images_are_u8, B, H, W, C, centroids, sample_inds, n, crop_h, crop_w, false, H, W, out_crops);
}

int sb_crop_centered_resized(sb_handle_t h, const void* images_host, int images_are_u8, int B, int H, int W, int C,
                             const float* centroids, const int32_t* sample_inds, int n, int crop_h, int crop_w, float scale,
                             void* out_crops) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  int Hr, Wr;
  if (sb_resized_size(H, W, scale, &Hr, &Wr))
    return sb_fail(h, SB_ERR_INVALID, "sb_crop_centered_resized: scale %g of %d x %d frames", scale, H, W);
  return crop_centered(h, images_host, images_are_u8, B, H, W, C, centroids, sample_inds, n, crop_h, crop_w, true, Hr, Wr, out_crops);
}

// Builds the per-node ascending peak lists on the host (stable argsort by channel,
// paf_grouping.py:106-109) for the stage-level calls that receive caller-supplied peaks.
static int upload_peaks(SbScratch& s, int B, int n_nodes, const float* peaks, const float* peak_vals, const int32_t* ch,
                        const int32_t* off) {
  SbPostWs& ws = s.ws;
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
      if (c < 0 || c >= n_nodes) return sb_fail(s.h, SB_ERR_INVALID, "peak channel %d out of range", c);
      int& k = cnt[(size_t)b * n_nodes + c];
      lst[((size_t)b * n_nodes + c) * K + k] = i;
      ++k;
    }
  }
  int rc;
  if ((rc = s.to_dev(ws.peaks, pk.data(), pk.size())) || (rc = s.to_dev(ws.peak_vals, pv.data(), pv.size())) ||
      (rc = s.to_dev(ws.node_cnt, cnt.data(), cnt.size())) || (rc = s.to_dev(ws.node_peaks, lst.data(), lst.size())) ||
      (rc = s.to_dev(ws.n_peaks, np.data(), np.size())))
    return rc;
  SB_CUDA(s.h, cudaMemsetAsync(ws.flags, 0, B * sizeof(int), s.h->stream));
  return s.sync();
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
  SbScratch s(h);
  const float* d_pafs;
  int rc = sb_post_ws_alloc(h, s.ws, B, 1, 1, n_nodes, MP, K, 1, n_edges);
  if (rc || (rc = upload_peaks(s, B, n_nodes, peaks, nullptr, peak_channel_inds, peak_offsets)) ||
      (rc = s.to_dev(s.ws.edges_dev, skeleton_edges, (size_t)n_edges * 2)) ||
      (rc = s.upload(pafs_host, (size_t)B * Hp * Wp * C2, &d_pafs)))
    return rc;
  // max_edge_length = ratio * max(Hp, Wp, C2) * stride  (paf_grouping.py:469-473), in f32
  const float max_len = max_edge_length_ratio * (float)std::max(std::max(Hp, Wp), C2) * (float)pafs_stride;
  SbGraphHost g;
  if ((rc = sbk_score_match(h, d_pafs, B, Hp, Wp, C2, n_line_points, pafs_stride, max_len, dist_penalty_weight, s.ws)) ||
      (rc = s.sync()) || (rc = sb_graph_download(h, s.ws, B, g)))
    return rc;
  // the node lists are the ones upload_peaks built: (sample, edge, src-major) order
  return sb_graph_flatten(h, s.ws, g, skeleton_edges, B, cap, out_edge_inds, out_edge_peak_inds, out_line_scores, out_cand_offsets);
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
  const size_t P = n_line_points;
  SbScratch s(h);
  const float *d_paf, *d_lin, *d_pk;
  const int *d_epi, *d_ei;
  int* d_subs;
  float *d_ol, *d_os;
  int rc;
  if ((rc = s.upload(pafs_sample, (size_t)Hp * Wp * C2, &d_paf, true)) || (rc = s.upload(lines_in, n * P * 2, &d_lin, true)) ||
      (rc = s.upload(peaks, (size_t)n_peaks * 2, &d_pk)) || (rc = s.upload(edge_peak_inds, (size_t)n * 2, &d_epi)) ||
      (rc = s.upload(edge_inds, (size_t)n, &d_ei, true)) || (rc = s.alloc(&d_subs, n * P * 2)) ||
      (rc = s.alloc(&d_ol, n * P * 2)) || (rc = s.alloc(&d_os, (size_t)n)) ||
      (rc = sbk_lines(h, d_paf, Hp, Wp, C2, d_lin, d_pk, d_epi, d_ei, n, n_line_points, (float)pafs_stride, max_edge_length,
                      dist_penalty_weight, d_subs, d_ol, d_os)) ||
      (rc = s.to_host(out_subs, d_subs, n * P * 2, true)) || (rc = s.to_host(out_lines, d_ol, n * P * 2, true)) ||
      (rc = s.to_host(out_scores, d_os, (size_t)n, true)))
    return rc;
  return s.sync();
}

int sb_integral_regression(sb_handle_t h, const float* cms, int N, int Hh, int Ww, int C,
                           const float* xv, const float* yv, float* x_hat, float* y_hat) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  if (N <= 0) return SB_OK;
  SB_CUDA(h, cudaSetDevice(h->device));
  SbScratch s(h);
  const float *d_c, *d_x, *d_y;
  float *d_ox, *d_oy;
  const size_t n = (size_t)N * Hh * Ww * C;
  int rc;
  if ((rc = s.upload(cms, n, &d_c)) || (rc = s.upload(xv, (size_t)Ww, &d_x)) || (rc = s.upload(yv, (size_t)Hh, &d_y)) ||
      (rc = s.alloc(&d_ox, (size_t)N * C)) || (rc = s.alloc(&d_oy, (size_t)N * C)) ||
      (rc = sbk_integral(h, d_c, N, Hh, Ww, C, d_x, d_y, d_ox, d_oy)) ||
      (rc = s.to_host(x_hat, d_ox, (size_t)N * C)) || (rc = s.to_host(y_hat, d_oy, (size_t)N * C)))
    return rc;
  return s.sync();
}

int sb_find_offsets_local_direction(sb_handle_t h, const float* patches, int N, float delta,
                                    float* out_offsets) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  if (N <= 0) return SB_OK;
  SB_CUDA(h, cudaSetDevice(h->device));
  SbScratch s(h);
  const float* d_p;
  float* d_o;
  int rc;
  if ((rc = s.upload(patches, (size_t)N * 9, &d_p)) || (rc = s.alloc(&d_o, (size_t)N * 2)) ||
      (rc = sbk_local_dir(h, d_p, N, delta, d_o)) || (rc = s.to_host(out_offsets, d_o, (size_t)N * 2)))
    return rc;
  return s.sync();
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
  SbScratch s(h);
  const float* d_sc;
  const int *d_ns, *d_nd, *d_of;
  int *d_r, *d_c, *d_n;
  float* d_s;
  const size_t np = (size_t)n_problems;
  int rc;
  if ((rc = s.upload(scores, total, &d_sc)) || (rc = s.upload(n_src, np, &d_ns)) || (rc = s.upload(n_dst, np, &d_nd)) ||
      (rc = s.upload(offsets, np, &d_of)) || (rc = s.alloc(&d_r, np * max_k)) || (rc = s.alloc(&d_c, np * max_k)) ||
      (rc = s.alloc(&d_s, np * max_k)) || (rc = s.alloc(&d_n, np)) ||
      (rc = sbk_lsap_batch(h, d_sc, d_ns, d_nd, d_of, n_problems, max_k, d_r, d_c, d_s, d_n)) ||
      (rc = s.to_host(out_rows, d_r, np * max_k)) || (rc = s.to_host(out_cols, d_c, np * max_k)) ||
      (rc = s.to_host(out_scores, d_s, np * max_k)) || (rc = s.to_host(out_counts, d_n, np)))
    return rc;
  return s.sync();
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
  SbScratch s(h);
  SbPostWs& ws = s.ws;
  int rc = sb_post_ws_alloc(h, ws, B, 1, 1, n_nodes, MP, K, max_instances, n_edges);
  if (rc || (rc = upload_peaks(s, B, n_nodes, peaks, peak_vals, peak_channel_inds, peak_offsets))) return rc;
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
  if ((rc = s.to_dev(ws.match_cnt, ecnt.data(), ecnt.size())) || (rc = s.to_dev(ws.match_src, msrc.data(), msrc.size())) ||
      (rc = s.to_dev(ws.match_dst, mdst.data(), mdst.size())) || (rc = s.to_dev(ws.match_score, msc.data(), msc.size())) ||
      (rc = s.to_dev(ws.edges_dev, edge_types, (size_t)n_edges * 2)))
    return rc;
  if (n_sorted > n_edges) return sb_fail(h, SB_ERR_INVALID, "n_sorted > n_edges");
  if (n_sorted > 0 && (rc = s.to_dev(ws.sorted_edges_dev, sorted_edge_inds, (size_t)n_sorted))) return rc;
  ws.n_sorted = n_sorted;
  // Note: stage-level peaks lists hold *all* peaks of a node, so node_cnt >= every local index.
  const size_t I = max_instances;
  if ((rc = sbk_group(h, B, n_nodes, min_instance_peaks, min_line_scores, 1.0f, ws)) ||
      (rc = s.to_host(out_instances, ws.inst_peaks, B * I * n_nodes * 2)) || (rc = s.to_host(out_peak_scores, ws.inst_vals, B * I * n_nodes)) ||
      (rc = s.to_host(out_instance_scores, ws.inst_scores, B * I)) || (rc = s.to_host(out_n_instances, ws.n_inst, (size_t)B)))
    return rc;
  return s.sync();
}

}  // extern "C"
