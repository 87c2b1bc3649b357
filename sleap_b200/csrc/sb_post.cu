// Post-processing kernels of the SLEAP inference path for sm_90a: local / global peak finding
// with sub-pixel refinement, PAF line scoring, per-edge assignment and greedy instance grouping.
//
// Compiled with -fmad=false: the reference computes these quantities in float32 with separately
// rounded TensorFlow ops, and peak indices / instance assignments must match bit for bit, so no
// multiply-add may be contracted here.  All of this is HBM/L2-bound scan + gather work.
//
// Reference semantics restated per kernel (file:line under /root/reference):
//   k_local_scan / k_local_emit : sleap/nn/peak_finding.py:249-308 (rough NMS peaks),
//                                 :451-532 (refinement), :646-707 (learned offsets),
//                                 :135-190 crop_bboxes, :311-334 integral_regression, :78-132 local
//                                 sleap/nn/data/instance_cropping.py:58-90,124-166 (bboxes)
//   k_global_partial / k_global_final : sleap/nn/peak_finding.py:193-246, :337-420, :566-643
//   k_score_match : sleap/nn/paf_grouping.py:82-142, :145-275, :278-403, :406-550 (scoring),
//                   :553-670 (matching) + SciPy rectangular LSAP (sleap/nn/utils.py:79-98)
//   k_group       : sleap/nn/paf_grouping.py:799-914, :917-981, :984-1112
#include "sb_common.cuh"

#include <algorithm>
#include <cstdio>
#include <math_constants.h>
#include "sb_lsap.cuh"

namespace {

__device__ __forceinline__ float ldf(const float* p) { return __ldg(p); }

// ------------------------------------------------------------------------------------------
// tf.image.crop_and_resize(bilinear) of a p x p patch centred on integer pixel (px, py) of one
// channel plane of an NHWC map, followed by integral regression or the local-direction offset.
// Restates, op for op in f32: make_centered_bboxes -> normalize_bboxes -> crop_and_resize.
// ------------------------------------------------------------------------------------------
__device__ void refine_offset(const float* __restrict__ plane /* &cms[b][0][0][c] */, int H, int W,
                              int C, float px, float py, int mode, int p, float* dx, float* dy) {
  const float Hm1 = (float)(H - 1), Wm1 = (float)(W - 1);
  const float half = (float)(p - 1) * 0.5f;
  // bbox = (y,x,y,x) + 0.5*(-p+1, -p+1, p-1, p-1); normalised by (H-1, W-1).
  const float y1 = (py + (float)(-p + 1) * 0.5f) / Hm1;
  const float x1 = (px + (float)(-p + 1) * 0.5f) / Wm1;
  const float y2 = (py + (float)(p - 1) * 0.5f) / Hm1;
  const float x2 = (px + (float)(p - 1) * 0.5f) / Wm1;
  const float hs = (p > 1) ? ((y2 - y1) * Hm1) / (float)(p - 1) : 0.f;
  const float wsx = (p > 1) ? ((x2 - x1) * Wm1) / (float)(p - 1) : 0.f;
  float z = 0.f, sx = 0.f, sy = 0.f;
  float left = 0.f, right = 0.f, top = 0.f, bottom = 0.f;  // for the 3x3 local mode
  for (int i = 0; i < p; ++i) {
    const float in_y = (p > 1) ? (y1 * Hm1 + (float)i * hs) : (0.5f * (y1 + y2) * Hm1);
    const bool yok = !(in_y < 0.f || in_y > Hm1);
    int ty = 0, by = 0;
    float ly = 0.f;
    if (yok) {
      ty = (int)floorf(in_y);
      by = (int)ceilf(in_y);
      ly = in_y - (float)ty;
    }
    for (int j = 0; j < p; ++j) {
      float v = 0.f;
      if (yok) {
        const float in_x = (p > 1) ? (x1 * Wm1 + (float)j * wsx) : (0.5f * (x1 + x2) * Wm1);
        if (!(in_x < 0.f || in_x > Wm1)) {
          const int lx = (int)floorf(in_x), rx = (int)ceilf(in_x);
          const float xl = in_x - (float)lx;
          const float tl = ldf(plane + ((size_t)ty * W + lx) * C);
          const float tr = ldf(plane + ((size_t)ty * W + rx) * C);
          const float bl = ldf(plane + ((size_t)by * W + lx) * C);
          const float br = ldf(plane + ((size_t)by * W + rx) * C);
          const float t = tl + (tr - tl) * xl;
          const float bt = bl + (br - bl) * xl;
          v = t + (bt - t) * ly;
        }
      }
      if (mode == SB_REFINE_INTEGRAL) {
        z += v;
        sx += ((float)j - half) * v;
        sy += ((float)i - half) * v;
      } else {
        if (i == 1 && j == 0) left = v;
        if (i == 1 && j == 2) right = v;
        if (i == 0 && j == 1) top = v;
        if (i == 2 && j == 1) bottom = v;
      }
    }
  }
  if (mode == SB_REFINE_INTEGRAL) {
    *dx = sx / z;
    *dy = sy / z;
  } else {
    const float gx = right - left, gy = bottom - top;
    *dx = (gx > 0.f ? 0.25f : (gx < 0.f ? -0.25f : gx * 0.f));  // sign(x)*0.25 (NaN stays NaN)
    *dy = (gy > 0.f ? 0.25f : (gy < 0.f ? -0.25f : gy * 0.f));
  }
}

// ------------------------------------------------------------------------------------------
// Local peaks, pass A: one CTA per (row chunk, sample); flat, coalesced walk over the NHWC map;
// strict 8-neighbour NMS (out-of-image taps skipped, centre-1 tap) + strict threshold; ordered
// compaction of (flat index, value) into the chunk's list.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_local_scan(const float* __restrict__ cms, int H, int W, int C,
                                                    int rows_per_chunk, int chunk_cap,
                                                    float threshold, int* __restrict__ chunk_cnt,
                                                    uint2* __restrict__ chunk_items) {
  const int chunk = blockIdx.x, b = blockIdx.y, n_chunks = gridDim.x;
  const int y0 = chunk * rows_per_chunk;
  const int y1 = min(H, y0 + rows_per_chunk);
  const int rowlen = W * C;
  const float* base = cms + (size_t)b * H * rowlen;
  const int f0 = y0 * rowlen, f1 = y1 * rowlen;
  uint2* items = chunk_items + ((size_t)b * n_chunks + chunk) * chunk_cap;
  __shared__ int warp_tot[8];
  __shared__ int running;
  if (threadIdx.x == 0) running = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int fbase = f0; fbase < f1; fbase += 256) {
    const int f = fbase + threadIdx.x;
    bool is_peak = false;
    float v = 0.f;
    if (f < f1) {
      v = ldf(base + f);
      if (v > threshold) {
        const int y = f / rowlen;
        const int r = f - y * rowlen;
        const int x = r / C;
        float m = v - 1.0f;  // centre tap: v + (-1)
        const bool up = y > 0, dn = y < H - 1, lf = x > 0, rt = x < W - 1;
        const float* q = base + f;
        if (up) {
          if (lf) m = fmaxf(m, ldf(q - rowlen - C));
          m = fmaxf(m, ldf(q - rowlen));
          if (rt) m = fmaxf(m, ldf(q - rowlen + C));
        }
        if (lf) m = fmaxf(m, ldf(q - C));
        if (rt) m = fmaxf(m, ldf(q + C));
        if (dn) {
          if (lf) m = fmaxf(m, ldf(q + rowlen - C));
          m = fmaxf(m, ldf(q + rowlen));
          if (rt) m = fmaxf(m, ldf(q + rowlen + C));
        }
        is_peak = v > m;
      }
    }
    const int any = __syncthreads_count(is_peak);
    if (any == 0) continue;
    const unsigned bal = __ballot_sync(0xffffffffu, is_peak);
    const int rank = __popc(bal & ((1u << lane) - 1u));
    if (lane == 0) warp_tot[wid] = __popc(bal);
    __syncthreads();
    int off = running;
    for (int w = 0; w < wid; ++w) off += warp_tot[w];
    if (is_peak) {
      const int pos = off + rank;
      if (pos < chunk_cap) items[pos] = make_uint2((unsigned)f, __float_as_uint(v));
    }
    __syncthreads();
    if (threadIdx.x == 0) running += any;
    // next iteration's first barrier (__syncthreads_count) orders this write before its read
  }
  __syncthreads();
  if (threadIdx.x == 0) chunk_cnt[b * n_chunks + chunk] = running;
}

// Vectorised scan (float maps whose rows are a multiple of 4 elements): a pure streaming pass, no block barrier.
// A scan with one scalar load in flight per thread and a __syncthreads_count per 256 elements is latency bound.
// Here every thread keeps UN 16-byte loads in flight, elements above the
// threshold (a fraction of a percent of the map) take the 8-neighbour slow path, and a peak is appended to its
// chunk's list with one atomicAdd -- the list is therefore UNORDERED inside a chunk; k_local_emit restores the
// tf.where order by ranking the (unique) flat indices of a chunk.  chunk_cap can never overflow: strict
// 8-neighbour maxima are at most one per 2x2 block.  chunk_cnt must be zero on entry.
__device__ __forceinline__ float4 ldg_stream4(const float* p) {
  float4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}

template <int UN>
__global__ void __launch_bounds__(256) k_local_scan_v(const float* __restrict__ cms, int H, int W, int C,
                                                      int rows_per_chunk, int chunk_cap, float threshold,
                                                      int* __restrict__ chunk_cnt, uint2* __restrict__ chunk_items) {
  const int chunk = blockIdx.x, b = blockIdx.y, n_chunks = gridDim.x;
  const int y0 = chunk * rows_per_chunk;
  const int y1 = min(H, y0 + rows_per_chunk);
  const int rowlen = W * C;
  const float* base = cms + (size_t)b * H * rowlen;
  const int f0 = y0 * rowlen, f1 = y1 * rowlen;          // multiples of 4 (host-checked)
  uint2* items = chunk_items + ((size_t)b * n_chunks + chunk) * chunk_cap;
  int* cnt = chunk_cnt + b * n_chunks + chunk;
  for (int fb = f0 + 4 * (int)threadIdx.x; fb < f1; fb += 4 * 256 * UN) {
    float4 q[UN];
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      const int f = fb + u * 1024;
      q[u] = (f < f1) ? ldg_stream4(base + f) : make_float4(threshold, threshold, threshold, threshold);
    }
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      if (!(fmaxf(fmaxf(q[u].x, q[u].y), fmaxf(q[u].z, q[u].w)) > threshold)) continue;
      const float vv[4] = {q[u].x, q[u].y, q[u].z, q[u].w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float v = vv[k];
        if (!(v > threshold)) continue;
        const int fk = fb + u * 1024 + k;
        const int y = fk / rowlen;
        const int r = fk - y * rowlen;
        const int x = r / C;
        float m = v - 1.0f;                             // centre tap: v + (-1)
        const bool up = y > 0, dn = y < H - 1, lf = x > 0, rt = x < W - 1;
        const float* p = base + fk;
        if (up) {
          if (lf) m = fmaxf(m, __ldg(p - rowlen - C));
          m = fmaxf(m, __ldg(p - rowlen));
          if (rt) m = fmaxf(m, __ldg(p - rowlen + C));
        }
        if (lf) m = fmaxf(m, __ldg(p - C));
        if (rt) m = fmaxf(m, __ldg(p + C));
        if (dn) {
          if (lf) m = fmaxf(m, __ldg(p + rowlen - C));
          m = fmaxf(m, __ldg(p + rowlen));
          if (rt) m = fmaxf(m, __ldg(p + rowlen + C));
        }
        if (v > m) {
          const int pos = atomicAdd(cnt, 1);
          if (pos < chunk_cap) items[pos] = make_uint2((unsigned)fk, __float_as_uint(v));
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Warp-cooperative form of refine_offset: lane s computes patch sample s (the four bilinear taps are its only
// memory traffic, so the 4 x p*p dependent-looking loads of the scalar routine become one round of independent
// loads), then every lane replays the SAME sequential accumulation over the samples (shuffle broadcast), i.e. the
// float operations and their order are those of refine_offset -- results are bit-identical to it.
// ------------------------------------------------------------------------------------------
__device__ void refine_offset_warp(const float* __restrict__ plane, int H, int W, int C, float px, float py, int mode, int p,
                                   int lane, float* dx, float* dy) {
  const float Hm1 = (float)(H - 1), Wm1 = (float)(W - 1);
  const float half = (float)(p - 1) * 0.5f;
  const float y1 = (py + (float)(-p + 1) * 0.5f) / Hm1;
  const float x1 = (px + (float)(-p + 1) * 0.5f) / Wm1;
  const float y2 = (py + (float)(p - 1) * 0.5f) / Hm1;
  const float x2 = (px + (float)(p - 1) * 0.5f) / Wm1;
  const float hs = (p > 1) ? ((y2 - y1) * Hm1) / (float)(p - 1) : 0.f;
  const float wsx = (p > 1) ? ((x2 - x1) * Wm1) / (float)(p - 1) : 0.f;
  const int n = p * p;
  float vals[4] = {0.f, 0.f, 0.f, 0.f};                 // samples lane, lane+32, lane+64, lane+96 (p <= 11)
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const int sidx = r * 32 + lane;
    if (sidx >= n) continue;
    const int i = sidx / p, j = sidx - i * p;
    const float in_y = (p > 1) ? (y1 * Hm1 + (float)i * hs) : (0.5f * (y1 + y2) * Hm1);
    const float in_x = (p > 1) ? (x1 * Wm1 + (float)j * wsx) : (0.5f * (x1 + x2) * Wm1);
    float v = 0.f;
    if (!(in_y < 0.f || in_y > Hm1) && !(in_x < 0.f || in_x > Wm1)) {
      const int ty = (int)floorf(in_y), by = (int)ceilf(in_y);
      const float ly = in_y - (float)ty;
      const int lx = (int)floorf(in_x), rx = (int)ceilf(in_x);
      const float xl = in_x - (float)lx;
      const float tl = ldf(plane + ((size_t)ty * W + lx) * C);
      const float tr = ldf(plane + ((size_t)ty * W + rx) * C);
      const float bl = ldf(plane + ((size_t)by * W + lx) * C);
      const float br = ldf(plane + ((size_t)by * W + rx) * C);
      const float t = tl + (tr - tl) * xl;
      const float bt = bl + (br - bl) * xl;
      v = t + (bt - t) * ly;
    }
    vals[r] = v;
  }
  if (mode == SB_REFINE_INTEGRAL) {
    float z = 0.f, sx = 0.f, sy = 0.f;
    for (int i = 0; i < p; ++i)
      for (int j = 0; j < p; ++j) {
        const int sidx = i * p + j;
        const int r = sidx >> 5;
        const float mine = r == 0 ? vals[0] : (r == 1 ? vals[1] : (r == 2 ? vals[2] : vals[3]));
        const float v = __shfl_sync(0xffffffffu, mine, sidx & 31);
        z += v;
        sx += ((float)j - half) * v;
        sy += ((float)i - half) * v;
      }
    *dx = sx / z;
    *dy = sy / z;
  } else {                                              // 3x3: left (1,0), right (1,2), top (0,1), bottom (2,1)
    const float left = __shfl_sync(0xffffffffu, vals[0], 3), right = __shfl_sync(0xffffffffu, vals[0], 5);
    const float top = __shfl_sync(0xffffffffu, vals[0], 1), bottom = __shfl_sync(0xffffffffu, vals[0], 7);
    const float gx = right - left, gy = bottom - top;
    *dx = (gx > 0.f ? 0.25f : (gx < 0.f ? -0.25f : gx * 0.f));
    *dy = (gy > 0.f ? 0.25f : (gy < 0.f ? -0.25f : gy * 0.f));
  }
}

// ------------------------------------------------------------------------------------------
// Local peaks, pass B: one CTA per sample.  (1) block scan of the chunk counts; (2) every scanned item finds its
// place in tf.where order -- chunks are row ranges (ordered), inside a chunk the rank of its (unique) flat index --
// and the first max_peaks of them are kept; (3) one warp per kept peak refines it (refine_offset_warp), scales it and
// stores it; (4) the per-node (channel) ascending peak lists that PAF candidate enumeration needs (stable argsort by
// channel, paf_grouping.py:106-109): the slot of peak i in its node's list is the number of earlier peaks of that
// channel.
// ------------------------------------------------------------------------------------------
constexpr int EMIT_THREADS = 512;

__global__ void __launch_bounds__(EMIT_THREADS) k_local_emit(
    const float* __restrict__ cms, const float* __restrict__ offsets, int H, int W, int C, int n_chunks,
    int chunk_cap, int refinement, int patch, float scale, float input_scale, int max_peaks,
    int max_node_peaks, const int* __restrict__ chunk_cnt, const uint2* __restrict__ chunk_items,
    uint2* __restrict__ sorted_items /*[B][max_peaks]*/, float* __restrict__ peaks, float* __restrict__ peak_vals,
    int* __restrict__ peak_ch, int* __restrict__ n_peaks, int* __restrict__ total_peaks, int* __restrict__ node_cnt,
    int* __restrict__ node_peaks, int* __restrict__ flags) {
  extern __shared__ int s_prefix[];  // n_chunks + 1
  const int b = blockIdx.x;
  __shared__ int s_warp[EMIT_THREADS / 32];
  __shared__ int s_carry;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (threadIdx.x == 0) s_carry = 0;
  __syncthreads();
  for (int k0 = 0; k0 < n_chunks; k0 += EMIT_THREADS) {         // exclusive block scan of min(cnt, cap)
    const int k = k0 + threadIdx.x;
    const int mine = k < n_chunks ? min(chunk_cnt[b * n_chunks + k], chunk_cap) : 0;
    int incl = mine;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, d);
      if (lane >= d) incl += t;
    }
    if (lane == 31) s_warp[wid] = incl;
    __syncthreads();
    int off = s_carry;
    for (int w = 0; w < wid; ++w) off += s_warp[w];
    if (k < n_chunks) s_prefix[k] = off + incl - mine;
    __syncthreads();
    if (threadIdx.x == EMIT_THREADS - 1) s_carry = off + incl;
    __syncthreads();
  }
  if (threadIdx.x == 0) s_prefix[n_chunks] = s_carry;
  __syncthreads();
  const int total = s_prefix[n_chunks];
  const int n = min(total, max_peaks);
  int flag = (total > max_peaks) ? SB_FLAG_PEAKS_TRUNCATED : 0;
  const int rowlen = W * C;
  const float* base = cms + (size_t)b * H * rowlen;
  float* pk = peaks + (size_t)b * max_peaks * 2;
  float* pv = peak_vals + (size_t)b * max_peaks;
  int* pc = peak_ch + (size_t)b * max_peaks;
  uint2* srt = sorted_items + (size_t)b * max_peaks;
  // (2) place every item
  for (int t = threadIdx.x; t < total; t += EMIT_THREADS) {
    int lo = 0, hi = n_chunks - 1;  // largest k with prefix[k] <= t
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (s_prefix[mid] <= t) lo = mid; else hi = mid - 1;
    }
    const uint2* lst = chunk_items + ((size_t)b * n_chunks + lo) * chunk_cap;
    const int cnt = s_prefix[lo + 1] - s_prefix[lo];
    const uint2 it = lst[t - s_prefix[lo]];
    int rank = 0;
    for (int q = 0; q < cnt; ++q) rank += (lst[q].x < it.x) ? 1 : 0;
    const int pos = s_prefix[lo] + rank;
    if (pos < n) {
      srt[pos] = it;
      const int r = (int)it.x % rowlen;
      pc[pos] = r % C;
    }
  }
  __syncthreads();                  // srt / pc written by this CTA are visible to it
  // (3) one warp per kept peak
  for (int i = wid; i < n; i += EMIT_THREADS / 32) {
    const uint2 it = srt[i];
    const int f = (int)it.x;
    const int y = f / rowlen;
    const int r = f - y * rowlen;
    const int x = r / C;
    const int c = r - x * C;
    float fx = (float)x, fy = (float)y;
    if (offsets != nullptr) {
      // learned offsets (B,H,W,C,2): refined = rough + offsets[b, y, x, c, :]
      const float* o = offsets + (((size_t)b * H + y) * W + x) * (size_t)(2 * C) + 2 * c;
      fx = fx + o[0];
      fy = fy + o[1];
    } else if (refinement != SB_REFINE_NONE) {
      float dx, dy;
      const int pp = refinement == SB_REFINE_INTEGRAL ? patch : 3;
      if (pp * pp <= 128) refine_offset_warp(base + c, H, W, C, fx, fy, refinement, pp, lane, &dx, &dy);
      else refine_offset(base + c, H, W, C, fx, fy, refinement, pp, &dx, &dy);
      fx = fx + dx;
      fy = fy + dy;
    }
    fx = fx * scale;
    fy = fy * scale;
    if (input_scale != 1.0f) {  // CentroidCrop: /input_scale + 0.5 (inference.py:1828-1833)
      fx = fx / input_scale + 0.5f;
      fy = fy / input_scale + 0.5f;
    }
    if (lane == 0) {
      pk[2 * i] = fx;
      pk[2 * i + 1] = fy;
      pv[i] = __uint_as_float(it.y);
    }
  }
  // (4) per-node ascending lists
  if (node_cnt != nullptr) {
    for (int i = threadIdx.x; i < n; i += EMIT_THREADS) {
      const int c = pc[i];
      int slot = 0;
      for (int j = 0; j < i; ++j) slot += (pc[j] == c) ? 1 : 0;
      if (slot < max_node_peaks) node_peaks[((size_t)b * C + c) * max_node_peaks + slot] = i;
    }
    for (int c = threadIdx.x; c < C; c += EMIT_THREADS) {
      int cnt = 0;
      for (int j = 0; j < n; ++j) cnt += (pc[j] == c) ? 1 : 0;
      node_cnt[b * C + c] = cnt;
      if (cnt > max_node_peaks) atomicOr(&flags[b], SB_FLAG_NODE_PEAKS_TRUNCATED);
    }
  }
  if (threadIdx.x == 0) {
    n_peaks[b] = n;
    total_peaks[b] = total;
    if (flag) atomicOr(&flags[b], flag);
  }
}

// ------------------------------------------------------------------------------------------
// Global peaks.  argmax_y(max_x) / argmax_x(max_y) with first-index ties == (first row, first
// column) that contain the global maximum, so one lexicographic (max, min y, min x) reduction.
// Pass 1: CTA per (row chunk, sample); each thread owns one channel (stride multiple of C) and
// walks the chunk coalesced.  Pass 2: CTA per sample finishes, thresholds, refines, fixes up.
// ------------------------------------------------------------------------------------------
struct GMax {
  float v;
  int y, x;
};
__device__ __forceinline__ void gmax_merge(GMax& a, float v, int y, int x) {
  if (v > a.v) {
    a.v = v; a.y = y; a.x = x;
  } else if (v == a.v) {
    a.y = min(a.y, y);
    a.x = min(a.x, x);
  }
}

__global__ void __launch_bounds__(256) k_global_partial(const float* __restrict__ cms, int H, int W,
                                                        int C, int rows_per_chunk,
                                                        float* __restrict__ part /*[B][chunks][C][3]*/) {
  const int chunk = blockIdx.x, b = blockIdx.y, n_chunks = gridDim.x;
  const int y0 = chunk * rows_per_chunk, y1 = min(H, y0 + rows_per_chunk);
  const int rowlen = W * C;
  const float* base = cms + (size_t)b * H * rowlen;
  const int per = max(1, 256 / C);           // pixels handled per sweep
  const int active = per * C;                // threads that own a (pixel slot, channel)
  extern __shared__ float s_red[];           // [active][3]
  GMax g;
  g.v = -CUDART_INF_F; g.y = 0x7fffffff; g.x = 0x7fffffff;
  if (threadIdx.x < active && C <= 256) {
    const int c = threadIdx.x % C;
    const int f0 = y0 * rowlen, f1 = y1 * rowlen;
    for (int f = f0 + threadIdx.x; f < f1; f += active) {
      const float v = ldf(base + f);
      const int y = f / rowlen;
      const int x = (f - y * rowlen) / C;
      gmax_merge(g, v, y, x);
      (void)c;
    }
    s_red[threadIdx.x * 3 + 0] = g.v;
    s_red[threadIdx.x * 3 + 1] = __int_as_float(g.y);
    s_red[threadIdx.x * 3 + 2] = __int_as_float(g.x);
  }
  __syncthreads();
  if (threadIdx.x < C && C <= 256) {
    GMax a;
    a.v = -CUDART_INF_F; a.y = 0x7fffffff; a.x = 0x7fffffff;
    for (int s = 0; s < per; ++s) {
      const int t = s * C + threadIdx.x;
      gmax_merge(a, s_red[t * 3], __float_as_int(s_red[t * 3 + 1]), __float_as_int(s_red[t * 3 + 2]));
    }
    float* o = part + (((size_t)b * n_chunks + chunk) * C + threadIdx.x) * 3;
    o[0] = a.v; o[1] = __int_as_float(a.y); o[2] = __int_as_float(a.x);
  }
}

struct GlobalFix {
  float scale;        // output stride
  float input_scale;  // != 1 -> /input_scale + 0.5
  int has_crop_off;   // + crop_offsets[b] / input_scale
};

__global__ void k_global_final(const float* __restrict__ cms, const float* __restrict__ offsets, int H,
                               int W, int C, int n_chunks, const float* __restrict__ part,
                               float threshold, int refinement, int patch, GlobalFix fix,
                               const float* __restrict__ crop_off, float* __restrict__ out_points,
                               float* __restrict__ out_vals) {
  const int b = blockIdx.x;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    GMax a;
    a.v = -CUDART_INF_F; a.y = 0x7fffffff; a.x = 0x7fffffff;
    for (int k = 0; k < n_chunks; ++k) {
      const float* o = part + (((size_t)b * n_chunks + k) * C + c) * 3;
      gmax_merge(a, o[0], __float_as_int(o[1]), __float_as_int(o[2]));
    }
    const int row = min(max(a.y, 0), H - 1), col = min(max(a.x, 0), W - 1);
    const float* plane = cms + (size_t)b * H * W * C + c;
    const float val = ldf(plane + ((size_t)row * W + col) * C);
    float fx = (float)col, fy = (float)row;
    if (val < threshold) {
      fx = CUDART_NAN_F; fy = CUDART_NAN_F;
    } else {
      if (offsets != nullptr) {
        const float* o = offsets + (((size_t)b * H + row) * W + col) * (size_t)(2 * C) + 2 * c;
        fx = fx + o[0]; fy = fy + o[1];
      } else if (refinement != SB_REFINE_NONE) {
        float dx, dy;
        refine_offset(plane, H, W, C, fx, fy, refinement, refinement == SB_REFINE_INTEGRAL ? patch : 3, &dx, &dy);
        fx = fx + dx; fy = fy + dy;
      }
      fx = fx * fix.scale; fy = fy * fix.scale;
      if (fix.input_scale != 1.0f) {
        fx = fx / fix.input_scale + 0.5f; fy = fy / fix.input_scale + 0.5f;
      }
      if (fix.has_crop_off) {
        fx = fx + crop_off[2 * b] / fix.input_scale;
        fy = fy + crop_off[2 * b + 1] / fix.input_scale;
      }
    }
    out_points[((size_t)b * C + c) * 2] = fx;
    out_points[((size_t)b * C + c) * 2 + 1] = fy;
    out_vals[(size_t)b * C + c] = val;
  }
}

// SciPy's linear_sum_assignment on one score matrix: cost = isnan ? +inf : -score, in double as SciPy does
// (the solver is sb_lsap.cuh).
__device__ int lsap_solve(const float* __restrict__ scores, int n_src, int n_dst, LsapScratch s,
                          int* out_rows, int* out_cols) {
  auto cost = [&](int i, int j) -> double {
    const float sc = scores[i * n_dst + j];
    return (sc != sc) ? (double)CUDART_INF_F : -(double)sc;
  };
  return lsap_solve_cost(cost, n_src, n_dst, s, out_rows, out_cols);
}

// ------------------------------------------------------------------------------------------
// PAF line scoring + matching: one CTA per (edge, sample).  One warp per candidate pair, lanes
// over the line points (warp-shuffle reduction of the dot products); then thread 0 solves the
// assignment for this edge.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_score_match(
    const float* __restrict__ pafs, int Hp, int Wp, int C2, int C, int K, int max_peaks,
    const int* __restrict__ edges, const float* __restrict__ peaks, const int* __restrict__ node_cnt,
    const int* __restrict__ node_peaks, int n_points, float pafs_stride, float max_edge_length,
    float dist_w, float* __restrict__ score_mat, int* __restrict__ match_cnt,
    int* __restrict__ match_src, int* __restrict__ match_dst, float* __restrict__ match_score) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int e = blockIdx.x, b = blockIdx.y, E = gridDim.x;
  const int src_node = edges[2 * e], dst_node = edges[2 * e + 1];
  const int ns = min(node_cnt[b * C + src_node], K), nd = min(node_cnt[b * C + dst_node], K);
  float* s_scores = reinterpret_cast<float*>(smem_raw);                 // K*K
  unsigned char* s_lsap = smem_raw + (((size_t)K * K * sizeof(float) + 15) & ~(size_t)15);
  const int* src_list = node_peaks + ((size_t)b * C + src_node) * K;
  const int* dst_list = node_peaks + ((size_t)b * C + dst_node) * K;
  const float* pk = peaks + (size_t)b * max_peaks * 2;
  const float* paf_b = pafs + (size_t)b * Hp * Wp * C2;
  float* gmat = score_mat + ((size_t)b * E + e) * K * K;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int p = wid; p < ns * nd; p += nw) {
    const int i = p / nd, j = p - i * nd;
    const int si = src_list[i], di = dst_list[j];
    const float sx = pk[2 * si], sy = pk[2 * si + 1];
    const float dx = pk[2 * di], dy = pk[2 * di + 1];
    const float vx = dx - sx, vy = dy - sy;
    const float len = sqrtf(vx * vx + vy * vy);
    const float ux = vx / len, uy = vy / len;
    const float stepx = (n_points > 1) ? (dx - sx) / (float)(n_points - 1) : 0.f;
    const float stepy = (n_points > 1) ? (dy - sy) / (float)(n_points - 1) : 0.f;
    float acc = 0.f;
    for (int q = lane; q < n_points; q += 32) {
      float X, Y;
      if (q == n_points - 1 && n_points > 1) { X = dx; Y = dy; }
      else { X = sx + stepx * (float)q; Y = sy + stepy * (float)q; }
      const int col = (int)rintf(X / pafs_stride);   // tf.round: half to even
      const int row = (int)rintf(Y / pafs_stride);
      float px = 0.f, py = 0.f;
      if (row >= 0 && row < Hp && col >= 0 && col < Wp) {
        const float2 pv = *reinterpret_cast<const float2*>(paf_b + ((size_t)row * Wp + col) * C2 + 2 * e);
        px = pv.x; py = pv.y;
      }
      acc += px * ux + py * uy;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) {
      const float mean = acc / (float)n_points;
      const float pen = fminf(max_edge_length / len - 1.0f, 0.f) * dist_w;
      const float sc = mean + pen;
      s_scores[p] = sc;
      gmat[p] = sc;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    LsapScratch s = carve_lsap(s_lsap, K);
    int* rows = match_src + ((size_t)b * E + e) * K;
    int* cols = match_dst + ((size_t)b * E + e) * K;
    const int n = lsap_solve(s_scores, ns, nd, s, rows, cols);
    float* ms = match_score + ((size_t)b * E + e) * K;
    for (int k = 0; k < n; ++k) ms[k] = s_scores[rows[k] * nd + cols[k]];
    match_cnt[b * E + e] = n;
  }
}

// Generic batched LSAP (stage-level API): one CTA (thread 0) per problem.
__global__ void k_lsap_batch(const float* __restrict__ scores, const int* __restrict__ n_src,
                             const int* __restrict__ n_dst, const int* __restrict__ offsets, int K,
                             int* __restrict__ out_rows, int* __restrict__ out_cols,
                             float* __restrict__ out_scores, int* __restrict__ out_counts) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int p = blockIdx.x;
  if (threadIdx.x != 0) return;
  LsapScratch s = carve_lsap(smem_raw, K);
  const int ns = n_src[p], nd = n_dst[p];
  const float* sc = scores + offsets[p];
  int n = 0;
  if (ns <= K && nd <= K) n = lsap_solve(sc, ns, nd, s, out_rows + (size_t)p * K, out_cols + (size_t)p * K);
  for (int k = 0; k < n; ++k)
    out_scores[(size_t)p * K + k] = sc[out_rows[(size_t)p * K + k] * nd + out_cols[(size_t)p * K + k]];
  out_counts[p] = n;
}

// ------------------------------------------------------------------------------------------
// Greedy instance grouping: one CTA per sample; thread 0 replays the reference's sequential
// dict algorithm on an array (node, local peak) -> instance id; the CTA fills outputs.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_group(
    int C, int E, int K, int max_peaks, int max_inst, const int* __restrict__ edges,
    const int* __restrict__ sorted_edges, int n_sorted, const float* __restrict__ peaks,
    const float* __restrict__ peak_vals, const int* __restrict__ g_node_cnt,
    const int* __restrict__ node_peaks, const int* __restrict__ g_match_cnt,
    const int* __restrict__ g_match_src, const int* __restrict__ g_match_dst,
    const float* __restrict__ g_match_score, int min_instance_peaks, float min_line_scores,
    float input_scale, float* __restrict__ inst_peaks, float* __restrict__ inst_vals,
    float* __restrict__ inst_scores, int* __restrict__ n_inst, int* __restrict__ flags,
    float* __restrict__ records /* [B][max_inst*C*3 + max_inst + 2] or null */, const SbGatherDev gx) {
  extern __shared__ int s_assign[];  // [C*K] instance id or -1; then [C*K] rank map scratch
  const int b = blockIdx.x;
  int* assign = s_assign;
  int* idrank = s_assign + C * K;    // instance id -> rank (ids < C*K)
  int* order = s_assign + 2 * C * K; // dict insertion sequence of each (node, peak) key
  // the sequential replay below runs on ONE thread: everything it reads is staged in shared memory first
  // (round 1 read the match tables from global memory, ~50 us per launch of dependent-load latency)
  int* node_cnt = s_assign + 3 * C * K;            // [C]
  int* match_cnt = node_cnt + C;                   // [E]
  int* match_src = match_cnt + E;                  // [E*K]
  int* match_dst = match_src + E * K;              // [E*K]
  float* match_score = reinterpret_cast<float*>(match_dst + E * K);   // [E*K]
  int* s_edges = reinterpret_cast<int*>(match_score + E * K);         // [2*E]
  int* s_sorted = s_edges + 2 * E;                                    // [n_sorted <= E]
  __shared__ int s_ninst;
  for (int t = threadIdx.x; t < C * K; t += blockDim.x) { assign[t] = -1; idrank[t] = -1; order[t] = -1; }
  for (int t = threadIdx.x; t < C; t += blockDim.x) node_cnt[t] = g_node_cnt[b * C + t];
  for (int t = threadIdx.x; t < E; t += blockDim.x) match_cnt[t] = g_match_cnt[b * E + t];
  for (int t = threadIdx.x; t < E * K; t += blockDim.x) {
    match_src[t] = g_match_src[(size_t)b * E * K + t];
    match_dst[t] = g_match_dst[(size_t)b * E * K + t];
    match_score[t] = g_match_score[(size_t)b * E * K + t];
  }
  for (int t = threadIdx.x; t < 2 * E; t += blockDim.x) s_edges[t] = edges[t];
  for (int t = threadIdx.x; t < n_sorted; t += blockDim.x) s_sorted[t] = sorted_edges[t];
  float* op = inst_peaks + (size_t)b * max_inst * C * 2;
  float* ov = inst_vals + (size_t)b * max_inst * C;
  float* os = inst_scores + (size_t)b * max_inst;
  for (int t = threadIdx.x; t < max_inst * C * 2; t += blockDim.x) op[t] = CUDART_NAN_F;
  for (int t = threadIdx.x; t < max_inst * C; t += blockDim.x) ov[t] = CUDART_NAN_F;
  for (int t = threadIdx.x; t < max_inst; t += blockDim.x) os[t] = CUDART_NAN_F;
  __syncthreads();
  if (threadIdx.x == 0) {
    const int n_slots = C * K;
    int seq = 0, cur_max = -1;
    for (int se = 0; se < n_sorted; ++se) {
      const int e = s_sorted[se];
      const int sn = s_edges[2 * e], dn = s_edges[2 * e + 1];
      const int cnt = match_cnt[e];
      const int mo = e * K;
      for (int m = 0; m < cnt; ++m) {
        if (!(match_score[mo + m] >= min_line_scores)) continue;
        const int sid = sn * K + match_src[mo + m], did = dn * K + match_dst[mo + m];
        const int si = assign[sid], di = assign[did];
        if (si < 0 && di < 0) {
          assign[sid] = cur_max + 1;          // max(instance_assignments.values()) + 1, tracked incrementally
          assign[did] = cur_max + 1;
          ++cur_max;
          order[sid] = seq++;                 // src key is inserted before dst (paf_grouping.py:853-854)
          order[did] = seq++;
        } else if (si >= 0 && di < 0) {
          assign[did] = si;
          order[did] = seq++;
        } else if (si >= 0 && di >= 0) {
          assign[did] = si;
          // node-type sets of both instances AFTER the re-assignment of dst
          bool share = false;
          for (int node = 0; node < C && !share; ++node) {
            bool in_s = false, in_d = false;
            const int kn = min(node_cnt[node], K);
            for (int k = 0; k < kn; ++k) {
              const int a = assign[node * K + k];
              in_s |= (a == si);
              in_d |= (a == di);
            }
            share = in_s && in_d;
          }
          if (!share)
            for (int node = 0; node < C; ++node) {
              const int kn = min(node_cnt[node], K);
              for (int k = 0; k < kn; ++k)
                if (assign[node * K + k] == di) assign[node * K + k] = si;
            }
          // instance ids can disappear through merges / steals: recompute the running maximum
          cur_max = -1;
          for (int node = 0; node < C; ++node) {
            const int kn = min(node_cnt[node], K);
            for (int k = 0; k < kn; ++k) cur_max = max(cur_max, assign[node * K + k]);
          }
        }
      }
    }
    if (min_instance_peaks > 0) {
      // instance ids are < n_slots; count peaks per id in idrank (reused as counter)
      for (int t = 0; t < n_slots; ++t) idrank[t] = 0;
      for (int t = 0; t < n_slots; ++t) if (assign[t] >= 0) idrank[assign[t]]++;
      for (int t = 0; t < n_slots; ++t)
        if (assign[t] >= 0 && idrank[assign[t]] < min_instance_peaks) assign[t] = -2;  // removed
      for (int t = 0; t < n_slots; ++t) { if (assign[t] == -2) assign[t] = -1; }
      for (int t = 0; t < n_slots; ++t) idrank[t] = -1;
    }
    // np.unique(return_inverse): rank of each id among the sorted unique ids
    for (int t = 0; t < n_slots; ++t) if (assign[t] >= 0) idrank[assign[t]] = 0;
    int r = 0;
    for (int t = 0; t < n_slots; ++t) if (idrank[t] == 0) idrank[t] = r++;
    s_ninst = r;
    int fl = 0;
    if (r > max_inst) fl = SB_FLAG_INSTANCES_TRUNCATED;
    const int keep = min(r, max_inst);
    for (int t = 0; t < keep; ++t) os[t] = 0.f;
    for (int se = 0; se < n_sorted; ++se) {
      const int e = s_sorted[se];
      const int sn = s_edges[2 * e];
      const int cnt = match_cnt[e];
      const int mo = e * K;
      for (int m = 0; m < cnt; ++m) {
        const float sc = match_score[mo + m];
        if (!(sc >= min_line_scores)) continue;
        const int a = assign[sn * K + match_src[mo + m]];
        if (a >= 0) {
          const int rk = idrank[a];
          if (rk < keep) os[rk] = os[rk] + sc;
        }
      }
    }
    n_inst[b] = keep;
    if (fl) flags[b] |= fl;
  }
  __syncthreads();
  const int keep = min(s_ninst, max_inst);
  const float* pk = peaks + (size_t)b * max_peaks * 2;
  const float* pv = peak_vals + (size_t)b * max_peaks;
  for (int t = threadIdx.x; t < C * K; t += blockDim.x) {
    const int a = assign[t];
    if (a < 0) continue;
    const int rk = idrank[a];
    if (rk >= keep) continue;
    const int node = t / K, k = t - node * K;
    if (k >= min(node_cnt[node], K)) continue;
    // two peaks of one node type can land in the same instance (skeletons where a node is the
    // destination of several edges); the reference fills the output in dict insertion order, so the
    // key inserted last wins (paf_grouping.py:973-979)
    bool later = false;
    for (int k2 = 0; k2 < K; ++k2)
      later |= (assign[node * K + k2] == a && order[node * K + k2] > order[t]);
    if (later) continue;
    const int pi = node_peaks[((size_t)b * C + node) * K + k];
    float x = pk[2 * pi], y = pk[2 * pi + 1];
    if (input_scale != 1.0f) {  // inference.py:2980-2984
      x = x / input_scale + 0.5f;
      y = y / input_scale + 0.5f;
    }
    op[((size_t)rk * C + node) * 2] = x;
    op[((size_t)rk * C + node) * 2 + 1] = y;
    ov[(size_t)rk * C + node] = pv[pi];
  }
  if (records == nullptr) return;
  // Epilogue: this frame's fixed-size result record, contiguous -- the ONE thing that leaves the GPU per frame
  // (single D2H copy) and the unit of the multi-GPU exchange (sb_gather_*): peaks | peak values | instance scores |
  // n_valid | flags, all float32 (the two counters are small integers, exact in float).
  __syncthreads();                       // this CTA's op / ov / os writes are visible to all its threads
  const int n2 = max_inst * C * 2, n1 = max_inst * C;
  const int w = (int)sb_record_width(max_inst, C);
  float* rec = records + (size_t)b * w;
  for (int t = threadIdx.x; t < n2; t += blockDim.x) rec[t] = op[t];
  for (int t = threadIdx.x; t < n1; t += blockDim.x) rec[n2 + t] = ov[t];
  for (int t = threadIdx.x; t < max_inst; t += blockDim.x) rec[n2 + n1 + t] = os[t];
  if (threadIdx.x == 0) {
    rec[n2 + n1 + max_inst] = (float)keep;
    rec[n2 + n1 + max_inst + 1] = (float)flags[b];
    for (int t = n2 + n1 + max_inst + 2; t < w; ++t) rec[t] = 0.f;   // padding
  }
  if (!gx.on) return;
  // ---- fused exchange: this frame's record goes straight into every rank's gather window over NVLink peer memory.
  // Generation gen of a window may be overwritten only when every consumer has acknowledged step - G (flow control:
  // only a producer G steps ahead of the slowest consumer ever waits here).
  __shared__ int s_go;
  const int gen = (int)(gx.step % (unsigned long long)gx.G);
  if (threadIdx.x == 0) {
    int go = 1;
    if (gx.step >= (unsigned long long)gx.G) {
      const unsigned long long need = gx.step - gx.G + 1;
      unsigned long long t0;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
      for (int r = 0; r < gx.world && go; ++r) {
        const volatile unsigned long long* a = gx.ack[gx.rank] + r;
        while (*a < need) {
          unsigned long long t1;
          asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
          if (t1 - t0 > gx.timeout_ns) { go = 0; atomicExch(gx.status, SB_GATHER_TIMEOUT_ACK); break; }
          __nanosleep(200);
        }
      }
      __threadfence_system();
    }
    s_go = go;
  }
  __syncthreads();                       // also: rec[] of this CTA is complete
  if (s_go) {
    const float4* src4 = reinterpret_cast<const float4*>(rec);
    for (int r = 0; r < gx.world; ++r) {  // record width is a multiple of 4 floats: 16-byte peer stores
      float4* dst4 = reinterpret_cast<float4*>(gx.data[r] + (((size_t)gen * gx.world + gx.rank) * gx.Bmax + b) * (size_t)w);
      for (int t = threadIdx.x; t < w / 4; t += blockDim.x) dst4[t] = src4[t];
    }
  }
  __threadfence_system();                // this thread's peer stores are ordered before the arrival word below
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int prev = atomicAdd(gx.done, 1u);
    if (prev == gridDim.x - 1) {         // last CTA of the launch: every frame's record is on its way / visible
      *gx.done = 0;
      __threadfence_system();
      const unsigned long long word = ((gx.step + 1) << 8) | (unsigned long long)gridDim.x;
      for (int r = 0; r < gx.world; ++r)
        asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(gx.arrive[r] + (size_t)gen * gx.world + gx.rank), "l"(word) : "memory");
    }
  }
}

// ------------------------------------------------------------------------------------------
// Identity grouping of the bottom-up multi-class step: one CTA per (node, sample).  The threads read the class-map
// logits of the node's peaks (k_local_emit's per-node list, tf.where order) at the rounded class-map cell, apply the
// sigmoid to those values only, and NaN-fill the node's cells of the frame's record; thread 0 then solves SciPy's
// assignment on -probability (rows: peaks, columns: classes) and keeps a match only where its probability is the
// peak's best over all classes.  The CTA of node 0 writes the frame's flags and padding.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128) k_class_group(
    const float* __restrict__ class_maps /*[B][Hc][Wc][NC] logits*/, int Hc, int Wc, int NC, float class_stride,
    float input_scale, int C, int K, int max_peaks, const float* __restrict__ peaks, const float* __restrict__ peak_vals,
    const int* __restrict__ node_cnt, const int* __restrict__ node_peaks, const int* __restrict__ flags,
    float* __restrict__ records /*[B][sb_class_record_width(NC, C)]*/) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int c = blockIdx.x, b = blockIdx.y;
  const int n = min(node_cnt[b * C + c], K);
  const int L = max(K, NC), M = min(K, NC);
  unsigned char* s_lsap = smem_raw;                                                        // LSAP scratch for max(K, NC)
  float* s_prob = reinterpret_cast<float*>(smem_raw + ((lsap_scratch_bytes(L) + 15) & ~(size_t)15));   // [K][NC]
  float* s_pt = s_prob + K * NC;                                                           // [K][2] output points
  int* s_cell = reinterpret_cast<int*>(s_pt + 2 * K);                                      // [K] class-map cell or -1
  int* s_rows = s_cell + K;                                                                // [M]
  int* s_cols = s_rows + M;                                                                // [M]
  const int* lst = node_peaks + ((size_t)b * C + c) * K;
  const float* pk = peaks + (size_t)b * max_peaks * 2;
  const float* pv = peak_vals + (size_t)b * max_peaks;
  const float* cmap = class_maps + (size_t)b * Hc * Wc * NC;
  // (1) per peak: its class-map cell and its output point, ((peak / cs) * cs) [/ input_scale + 0.5] in separate fp32 ops
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int pi = lst[i];
    const float xs = pk[2 * pi] / class_stride, ys = pk[2 * pi + 1] / class_stride;
    const float col = rintf(xs), row = rintf(ys);            // tf.round: half to even
    // a cell outside the class map reads 0 (gather_nd on the GPU), not sigmoid(0)
    s_cell[i] = (row >= 0.f && row < (float)Hc && col >= 0.f && col < (float)Wc) ? (int)row * Wc + (int)col : -1;
    float x = xs * class_stride, y = ys * class_stride;
    if (input_scale != 1.0f) {           // inference.py:3555-3577
      x = x / input_scale + 0.5f;
      y = y / input_scale + 0.5f;
    }
    s_pt[2 * i] = x;
    s_pt[2 * i + 1] = y;
  }
  const int n1 = NC * C;
  const int w = (int)sb_class_record_width(NC, C);
  float* rec = records + (size_t)b * w;
  for (int k = threadIdx.x; k < NC; k += blockDim.x) {
    const int cell = k * C + c;
    rec[2 * cell] = CUDART_NAN_F;
    rec[2 * cell + 1] = CUDART_NAN_F;
    rec[2 * n1 + cell] = CUDART_NAN_F;
    rec[3 * n1 + cell] = CUDART_NAN_F;
  }
  if (c == 0 && threadIdx.x == 0) {
    rec[4 * n1] = (float)flags[b];
    for (int t = 4 * n1 + 1; t < w; ++t) rec[t] = 0.f;   // padding
  }
  __syncthreads();
  // (2) the class probabilities of the node's peaks: the sigmoid of the sampled logits only
  for (int t = threadIdx.x; t < n * NC; t += blockDim.x) {
    const int i = t / NC;
    const int cell = s_cell[i];
    float p = 0.f;
    if (cell >= 0) {
      const double z = (double)cmap[(size_t)cell * NC + (t - i * NC)];
      p = (float)(1.0 / (1.0 + exp(-z)));                   // identity.class_probabilities
    }
    s_prob[t] = p;
  }
  __syncthreads();                       // probabilities staged; this CTA's NaN fill ordered before thread 0's stores
  if (threadIdx.x != 0 || n == 0) return;
  // (3) SciPy's assignment on -p, then the keep rule
  LsapScratch s = carve_lsap(s_lsap, L);
  const int nm = lsap_solve_cost([s_prob, NC](int i, int k) { return -(double)s_prob[i * NC + k]; }, n, NC, s, s_rows, s_cols);
  for (int q = 0; q < nm; ++q) {
    const int i = s_rows[q], k = s_cols[q];
    const float p = s_prob[i * NC + k];
    float best = s_prob[i * NC];
    for (int j = 1; j < NC; ++j) {       // np.max: a NaN propagates
      const float v = s_prob[i * NC + j];
      best = (v > best || v != v) ? v : best;
    }
    if (!(p == best)) continue;
    const int cell = k * C + c;
    rec[2 * cell] = s_pt[2 * i];
    rec[2 * cell + 1] = s_pt[2 * i + 1];
    rec[2 * n1 + cell] = pv[lst[i]];
    rec[3 * n1 + cell] = p;
  }
}

// ------------------------------------------------------------------------------------------
// Centred bilinear crops (top-down): crop_bboxes(make_centered_bboxes(centroid, h, w)) of the H x W frames a texel
// source reads: the frames themselves, or the frames resized on the fly (resize_image before the crop, for instance
// models trained at an input scale != 1), which is never stored.
// ------------------------------------------------------------------------------------------
template <typename TI>
struct SbFrameTexels {                      // channel c of pixel (y, x) of frame b
  const TI* __restrict__ img;
  int H, W, C;
  __device__ __forceinline__ float operator()(int b, int y, int x, int c) const {
    return (float)img[(size_t)b * H * W * C + ((size_t)y * W + x) * C + c];
  }
};
template <typename TI, bool TRUNC_U8>
struct SbResizedTexels {                    // channel c of pixel (y, x) of frame b resized from H x W to Hr x Wr
  const TI* __restrict__ img;
  int H, W, C, Hr, Wr;
  __device__ __forceinline__ float operator()(int b, int y, int x, int c) const {
    const TI* f = img + (size_t)b * H * W * C + c;
    const float v = sb_resize_sample([&](int sy, int sx) { return (float)f[((size_t)sy * W + sx) * C]; }, y, x, H, W, Hr, Wr);
    return TRUNC_U8 ? truncf(fminf(fmaxf(v, 0.f), 255.f)) : v;    // tf.cast back to the frame dtype
  }
};

template <typename Src, typename TO, bool TRUNC_U8>
__global__ void k_crop(Src img, int H, int W, int C,
                       const float* __restrict__ centroids, const int* __restrict__ sample_inds,
                       int crop_h, int crop_w, TO* __restrict__ out) {
  const int n = blockIdx.y;
  const float cx = centroids[2 * n], cy = centroids[2 * n + 1];
  const int b = sample_inds[n];
  const float Hm1 = (float)(H - 1), Wm1 = (float)(W - 1);
  const float y1 = (cy + (float)(-crop_h + 1) * 0.5f) / Hm1;
  const float x1 = (cx + (float)(-crop_w + 1) * 0.5f) / Wm1;
  const float y2 = (cy + (float)(crop_h - 1) * 0.5f) / Hm1;
  const float x2 = (cx + (float)(crop_w - 1) * 0.5f) / Wm1;
  const float hs = (crop_h > 1) ? ((y2 - y1) * Hm1) / (float)(crop_h - 1) : 0.f;
  const float wsx = (crop_w > 1) ? ((x2 - x1) * Wm1) / (float)(crop_w - 1) : 0.f;
  const int total = crop_h * crop_w * C;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
    const int c = t % C;
    const int j = (t / C) % crop_w;
    const int i = t / (C * crop_w);
    const float in_y = (crop_h > 1) ? (y1 * Hm1 + (float)i * hs) : (0.5f * (y1 + y2) * Hm1);
    const float in_x = (crop_w > 1) ? (x1 * Wm1 + (float)j * wsx) : (0.5f * (x1 + x2) * Wm1);
    float v = 0.f;
    if (!(in_y < 0.f || in_y > Hm1) && !(in_x < 0.f || in_x > Wm1)) {
      const int ty = (int)floorf(in_y), by = (int)ceilf(in_y);
      const int lx = (int)floorf(in_x), rx = (int)ceilf(in_x);
      const float ly = in_y - (float)ty, xl = in_x - (float)lx;
      const float tl = img(b, ty, lx, c), tr = img(b, ty, rx, c), bl = img(b, by, lx, c), br = img(b, by, rx, c);
      const float tp = tl + (tr - tl) * xl;
      const float bt = bl + (br - bl) * xl;
      v = tp + (bt - tp) * ly;
    }
    if (TRUNC_U8) out[(size_t)n * total + t] = (TO)(unsigned char)truncf(fminf(fmaxf(v, 0.f), 255.f));
    else out[(size_t)n * total + t] = (TO)v;
  }
}


// ------------------------------------------------------------------------------------------
// Function-level helpers kept for the reference's unit-test surface:
//   k_lines     : make_line_subs + get_paf_lines + score_paf_lines for explicit candidate lists
//                 (paf_grouping.py:145-222, :225-275, :325-403); one warp per candidate.
//   k_integral  : integral_regression (peak_finding.py:311-334); one warp per (sample, channel).
//   k_local_dir : find_offsets_local_direction (peak_finding.py:78-132).
// ------------------------------------------------------------------------------------------
__global__ void k_lines(const float* __restrict__ pafs /*(Hp,Wp,C2) or null*/, int Hp, int Wp, int C2,
                        const float* __restrict__ lines_in /*(n,P,2) or null*/,
                        const float* __restrict__ peaks, const int* __restrict__ edge_peak_inds,
                        const int* __restrict__ edge_inds, int n, int P, float pafs_stride,
                        float max_edge_length, float dist_w, int* __restrict__ out_subs /*(n,P,2)*/,
                        float* __restrict__ out_lines /*(n,P,2)*/, float* __restrict__ out_scores) {
  const int lane = threadIdx.x & 31;
  const int cand = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (cand >= n) return;
  const int si = edge_peak_inds[2 * cand], di = edge_peak_inds[2 * cand + 1];
  const int e = edge_inds ? edge_inds[cand] : 0;
  const float sx = peaks[2 * si], sy = peaks[2 * si + 1];
  const float dx = peaks[2 * di], dy = peaks[2 * di + 1];
  const float vx = dx - sx, vy = dy - sy;
  const float len = sqrtf(vx * vx + vy * vy);
  const float ux = vx / len, uy = vy / len;
  const float stepx = (P > 1) ? (dx - sx) / (float)(P - 1) : 0.f;
  const float stepy = (P > 1) ? (dy - sy) / (float)(P - 1) : 0.f;
  float acc = 0.f;
  for (int q = lane; q < P; q += 32) {
    float px = 0.f, py = 0.f;
    if (lines_in != nullptr) {
      px = lines_in[((size_t)cand * P + q) * 2];
      py = lines_in[((size_t)cand * P + q) * 2 + 1];
    } else {
      float X, Y;
      if (q == P - 1 && P > 1) { X = dx; Y = dy; }
      else { X = sx + stepx * (float)q; Y = sy + stepy * (float)q; }
      const int col = (int)rintf(X / pafs_stride);
      const int row = (int)rintf(Y / pafs_stride);
      if (out_subs) {
        out_subs[((size_t)cand * P + q) * 2] = row;
        out_subs[((size_t)cand * P + q) * 2 + 1] = col;
      }
      if (pafs != nullptr && row >= 0 && row < Hp && col >= 0 && col < Wp && 2 * e + 1 < C2) {
        px = pafs[((size_t)row * Wp + col) * C2 + 2 * e];
        py = pafs[((size_t)row * Wp + col) * C2 + 2 * e + 1];
      }
    }
    if (out_lines) {
      out_lines[((size_t)cand * P + q) * 2] = px;
      out_lines[((size_t)cand * P + q) * 2 + 1] = py;
    }
    acc += px * ux + py * uy;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0 && out_scores) {
    const float mean = acc / (float)P;
    const float pen = fminf(max_edge_length / len - 1.0f, 0.f) * dist_w;
    out_scores[cand] = mean + pen;
  }
}

__global__ void k_integral(const float* __restrict__ cms, int N, int Hh, int Ww, int C,
                           const float* __restrict__ xv, const float* __restrict__ yv,
                           float* __restrict__ x_hat, float* __restrict__ y_hat) {
  const int lane = threadIdx.x & 31;
  const int item = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (item >= N * C) return;
  const int nidx = item / C, c = item - nidx * C;
  const float* base = cms + (size_t)nidx * Hh * Ww * C + c;
  float z = 0.f, sx = 0.f, sy = 0.f;
  for (int t = lane; t < Hh * Ww; t += 32) {
    const int i = t / Ww, j = t - i * Ww;
    const float v = base[(size_t)t * C];
    z += v; sx += xv[j] * v; sy += yv[i] * v;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    z += __shfl_xor_sync(0xffffffffu, z, o);
    sx += __shfl_xor_sync(0xffffffffu, sx, o);
    sy += __shfl_xor_sync(0xffffffffu, sy, o);
  }
  if (lane == 0) { x_hat[item] = sx / z; y_hat[item] = sy / z; }
}

__global__ void k_local_dir(const float* __restrict__ patches /*(N,3,3,1)*/, int N, float delta,
                            float* __restrict__ out /*(N,2)*/) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const float* p = patches + (size_t)i * 9;
  const float gx = p[5] - p[3], gy = p[7] - p[1];
  out[2 * i] = (gx > 0.f ? 1.f : (gx < 0.f ? -1.f : gx * 0.f)) * delta;
  out[2 * i + 1] = (gy > 0.f ? 1.f : (gy < 0.f ? -1.f : gy * 0.f)) * delta;
}

}  // namespace

// =================================== host launchers =========================================

int sb_post_ws_alloc(sb_handle_s* h, SbPostWs& ws, int B, int H, int W, int C, int max_peaks,
                     int max_node_peaks, int max_instances, int n_edges) {
  ws.B = B; ws.H = H; ws.W = W; ws.C = C;
  ws.max_peaks = max_peaks; ws.max_node_peaks = max_node_peaks; ws.max_instances = max_instances;
  ws.n_edges = n_edges;
  ws.node_lists = n_edges > 0;
  // streaming scan: ~8 CTAs of 256 threads per SM over the batch, each with >= ~16 KB of map to walk
  int target_chunks = (8 * h->sm_count + B - 1) / B;
  int rpc = (H + target_chunks - 1) / target_chunks;
  if (rpc < 1) rpc = 1;
  while ((long long)rpc * W * C < 4096 && rpc < H) ++rpc;
  while ((long long)rpc * W * C > 65536 && rpc > 1) rpc = (rpc + 1) / 2;
  ws.rows_per_chunk = rpc;
  ws.n_chunks = (H + rpc - 1) / rpc;
  ws.chunk_cap = ((rpc + 1) / 2) * ((W + 1) / 2) * C;
  const int E = n_edges > 0 ? n_edges : 1, K = max_node_peaks > 0 ? max_node_peaks : 1;
  int rc = 0;
#define A(ptr, n) do { if ((rc = sb_dev_alloc(h, &ptr, (size_t)(n))) != 0) return rc; ws.bytes += sizeof(*ptr) * (size_t)(n); } while (0)
  A(ws.chunk_cnt, (size_t)B * ws.n_chunks);
  A(ws.chunk_items, (size_t)B * ws.n_chunks * ws.chunk_cap);
  A(ws.sorted_items, (size_t)B * max_peaks);
  A(ws.peaks, (size_t)B * max_peaks * 2);
  A(ws.peak_vals, (size_t)B * max_peaks);
  A(ws.peak_ch, (size_t)B * max_peaks);
  A(ws.n_peaks, B); A(ws.total_peaks, B); A(ws.flags, B);
  A(ws.node_cnt, (size_t)B * C);
  A(ws.node_peaks, (size_t)B * C * K);
  if (n_edges > 0) {
    A(ws.score_mat, (size_t)B * E * K * K);
    A(ws.match_cnt, (size_t)B * E);
    A(ws.match_src, (size_t)B * E * K);
    A(ws.match_dst, (size_t)B * E * K);
    A(ws.match_score, (size_t)B * E * K);
    A(ws.inst_peaks, (size_t)B * max_instances * C * 2);
    A(ws.inst_vals, (size_t)B * max_instances * C);
    A(ws.inst_scores, (size_t)B * max_instances);
    A(ws.n_inst, B);
    A(ws.records, (size_t)B * sb_record_width(max_instances, C));
    A(ws.edges_dev, (size_t)E * 2);
    A(ws.sorted_edges_dev, (size_t)E);
  }
#undef A
  return 0;
}

void sb_post_ws_free(SbPostWs& ws) {
  void* ptrs[] = {ws.chunk_cnt, ws.chunk_items, ws.peaks, ws.peak_vals, ws.peak_ch, ws.n_peaks,
                  ws.total_peaks, ws.flags, ws.node_cnt, ws.node_peaks, ws.score_mat, ws.match_cnt,
                  ws.match_src, ws.match_dst, ws.match_score, ws.inst_peaks, ws.inst_vals,
                  ws.inst_scores, ws.n_inst, ws.edges_dev, ws.sorted_edges_dev, ws.sorted_items, ws.records};
  for (void* p : ptrs) if (p) cudaFree(p);
  ws = SbPostWs();
}

int sbk_local_peaks(sb_handle_s* h, const float* cms, const float* offsets, int B, int H, int W, int C,
                    const SbPeakParams& p, SbPostWs& ws) {
  if (B > ws.B || H != ws.H || W != ws.W || C != ws.C)
    return sb_fail(h, SB_ERR_INVALID, "local peaks: workspace shape mismatch");
  dim3 g(ws.n_chunks, B);
  // zero the per-chunk append counters and the per-frame overflow flags (one memset node each, same stream)
  SB_CUDA(h, cudaMemsetAsync(ws.chunk_cnt, 0, (size_t)ws.B * ws.n_chunks * sizeof(int), h->stream));
  SB_CUDA(h, cudaMemsetAsync(ws.flags, 0, (size_t)ws.B * sizeof(int), h->stream));
  const bool vec_ok = ((W * C) % 4 == 0) && ((reinterpret_cast<uintptr_t>(cms) & 15) == 0) && !getenv("SB_DISABLE_SCAN_V");
  if (vec_ok)
    k_local_scan_v<4><<<g, 256, 0, h->stream>>>(cms, H, W, C, ws.rows_per_chunk, ws.chunk_cap, p.threshold,
                                                ws.chunk_cnt, ws.chunk_items);
  else
    k_local_scan<<<g, 256, 0, h->stream>>>(cms, H, W, C, ws.rows_per_chunk, ws.chunk_cap, p.threshold, ws.chunk_cnt,
                                           ws.chunk_items);
  SB_CHECK_LAUNCH(h);
  const size_t sm = (size_t)(ws.n_chunks + 1) * sizeof(int);
  int* ncnt = ws.node_lists ? ws.node_cnt : nullptr;
  k_local_emit<<<B, EMIT_THREADS, sm, h->stream>>>(
      cms, offsets, H, W, C, ws.n_chunks, ws.chunk_cap, p.refinement, p.patch,
      p.scale, p.input_scale, ws.max_peaks, ws.max_node_peaks, ws.chunk_cnt, ws.chunk_items, ws.sorted_items, ws.peaks,
      ws.peak_vals, ws.peak_ch, ws.n_peaks, ws.total_peaks, ncnt, ws.node_peaks, ws.flags);
  SB_CHECK_LAUNCH(h);
  return 0;
}

int sbk_global_peaks(sb_handle_s* h, const float* cms, const float* offsets, int B, int H, int W, int C, const SbPeakParams& p,
                     const float* crop_off_dev, float* part_buf, int n_chunks, int rows_per_chunk,
                     float* out_points, float* out_vals) {
  if (C > 256) return sb_fail(h, SB_ERR_UNSUPPORTED, "global peaks: C > 256");
  dim3 g(n_chunks, B);
  const int per = 256 / C > 0 ? 256 / C : 1;
  const size_t sm = (size_t)per * C * 3 * sizeof(float);
  GlobalFix fix;
  fix.scale = p.scale; fix.input_scale = p.input_scale; fix.has_crop_off = crop_off_dev != nullptr;
  k_global_partial<<<g, 256, sm, h->stream>>>(cms, H, W, C, rows_per_chunk, part_buf);
  SB_CHECK_LAUNCH(h);
  k_global_final<<<B, 64, 0, h->stream>>>(cms, offsets, H, W, C, n_chunks, part_buf, p.threshold, p.refinement, p.patch, fix,
                                          crop_off_dev, out_points, out_vals);
  SB_CHECK_LAUNCH(h);
  return 0;
}

size_t sb_score_match_smem(int K) { return (((size_t)K * K * sizeof(float) + 15) & ~(size_t)15) + lsap_scratch_bytes(K); }

size_t sb_group_smem(int n_nodes, int n_edges, int K) {
  return ((size_t)3 * n_nodes * K + n_nodes + n_edges + 3 * (size_t)n_edges * K + 3 * (size_t)n_edges) * sizeof(int);
}

size_t sb_class_group_smem(int K, int n_classes) {
  const int L = std::max(K, n_classes), M = std::min(K, n_classes);
  return ((lsap_scratch_bytes(L) + 15) & ~(size_t)15) + ((size_t)K * n_classes + 2 * (size_t)K) * sizeof(float) +
         ((size_t)K + 2 * (size_t)M) * sizeof(int);
}

// SB_ERR_UNSUPPORTED unless `kernel` can be launched with `bytes` of dynamic shared memory on the handle's device: the
// opt-in limit per block less the kernel's static shared memory
template <typename Kern>
static int smem_fits(sb_handle_s* h, Kern* kernel, const char* what, const char* cap, size_t bytes) {
  int optin = 0;
  SB_CUDA(h, cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, h->device));
  cudaFuncAttributes a;
  SB_CUDA(h, cudaFuncGetAttributes(&a, kernel));
  const size_t limit = (size_t)optin > a.sharedSizeBytes ? (size_t)optin - a.sharedSizeBytes : 0;
  if (bytes > limit)
    return sb_fail(h, SB_ERR_UNSUPPORTED, "%s: %s needs %zu B of shared memory per block, above the device's limit of %zu B",
                   cap, what, bytes, limit);
  return 0;
}

int sb_check_paf_smem(sb_handle_s* h, int n_nodes, int n_edges, int K) {
  char cap[64];
  snprintf(cap, sizeof(cap), "max_node_peaks %d", K);
  if (int rc = smem_fits(h, k_score_match, "PAF scoring and matching", cap, sb_score_match_smem(K))) return rc;
  return smem_fits(h, k_group, "grouping", cap, sb_group_smem(n_nodes, n_edges, K));
}

int sb_check_class_smem(sb_handle_s* h, int K, int n_classes) {
  char cap[64];
  snprintf(cap, sizeof(cap), "max_node_peaks %d with %d classes", K, n_classes);
  return smem_fits(h, k_class_group, "class grouping", cap, sb_class_group_smem(K, n_classes));
}

int sbk_score_match(sb_handle_s* h, const float* pafs, int B, int Hp, int Wp, int C2, int n_points,
                    int pafs_stride, float max_edge_length, float dist_penalty_weight, SbPostWs& ws) {
  const int K = ws.max_node_peaks, E = ws.n_edges;
  const size_t sm = sb_score_match_smem(K);
  if (sm > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(k_score_match, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    if (e != cudaSuccess) return sb_fail(h, SB_ERR_CUDA, "score_match smem %zu: %s", sm, cudaGetErrorString(e));
  }
  dim3 g(E, B);
  k_score_match<<<g, 128, sm, h->stream>>>(pafs, Hp, Wp, C2, ws.C, K, ws.max_peaks, ws.edges_dev, ws.peaks,
                                           ws.node_cnt, ws.node_peaks, n_points, (float)pafs_stride,
                                           max_edge_length, dist_penalty_weight, ws.score_mat, ws.match_cnt,
                                           ws.match_src, ws.match_dst, ws.match_score);
  SB_CHECK_LAUNCH(h);
  return 0;
}

int sbk_group(sb_handle_s* h, int B, int n_nodes, int min_instance_peaks, float min_line_scores,
              float input_scale, SbPostWs& ws, const SbGatherDev* gather) {
  SbGatherDev gx;
  if (gather) gx = *gather; else memset(&gx, 0, sizeof(gx));
  const int K = ws.max_node_peaks;
  const int E = ws.n_edges;
  const size_t sm = sb_group_smem(n_nodes, E, K);
  if (sm > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(k_group, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    if (e != cudaSuccess) return sb_fail(h, SB_ERR_CUDA, "group smem %zu: %s", sm, cudaGetErrorString(e));
  }
  k_group<<<B, 128, sm, h->stream>>>(n_nodes, ws.n_edges, K, ws.max_peaks, ws.max_instances, ws.edges_dev,
                                     ws.sorted_edges_dev, ws.n_sorted, ws.peaks, ws.peak_vals, ws.node_cnt,
                                     ws.node_peaks, ws.match_cnt, ws.match_src, ws.match_dst, ws.match_score,
                                     min_instance_peaks, min_line_scores, input_scale, ws.inst_peaks,
                                     ws.inst_vals, ws.inst_scores, ws.n_inst, ws.flags, ws.records, gx);
  SB_CHECK_LAUNCH(h);
  return 0;
}

int sbk_class_group(sb_handle_s* h, const float* class_maps, int B, int Hc, int Wc, int n_classes, float class_stride,
                    float input_scale, SbPostWs& ws) {
  if (!ws.node_lists || !ws.records || B > ws.B) return sb_fail(h, SB_ERR_INVALID, "class grouping: workspace not sized for it");
  const int K = ws.max_node_peaks;
  const size_t sm = sb_class_group_smem(K, n_classes);
  if (sm > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(k_class_group, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    if (e != cudaSuccess) return sb_fail(h, SB_ERR_CUDA, "class group smem %zu: %s", sm, cudaGetErrorString(e));
  }
  k_class_group<<<dim3(ws.C, B), 128, sm, h->stream>>>(class_maps, Hc, Wc, n_classes, class_stride, input_scale, ws.C, K,
                                                        ws.max_peaks, ws.peaks, ws.peak_vals, ws.node_cnt, ws.node_peaks,
                                                        ws.flags, ws.records);
  SB_CHECK_LAUNCH(h);
  return 0;
}

int sbk_lsap_batch(sb_handle_s* h, const float* scores, const int* n_src, const int* n_dst,
                   const int* offsets, int n_problems, int max_k, int* out_rows, int* out_cols,
                   float* out_scores, int* out_counts) {
  if (n_problems <= 0) return 0;
  const size_t sm = lsap_scratch_bytes(max_k);
  if (sm > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(k_lsap_batch, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm);
    if (e != cudaSuccess) return sb_fail(h, SB_ERR_CUDA, "lsap smem %zu: %s", sm, cudaGetErrorString(e));
  }
  k_lsap_batch<<<n_problems, 32, sm, h->stream>>>(scores, n_src, n_dst, offsets, max_k, out_rows, out_cols,
                                                  out_scores, out_counts);
  SB_CHECK_LAUNCH(h);
  return 0;
}

// k_crop of n crops of the H x W frames `src` reads: uint8 frames give uint8 crops (float -> uint8 truncation, as tf.cast in
// crop_bboxes), float frames float crops
template <template <typename> class Src>
static int launch_crop(sb_handle_s* h, Src<unsigned char> src_u8, Src<float> src_f32, int img_is_u8, int H, int W, int C,
                       const float* centroids, const int* sample_inds, int n, int crop_h, int crop_w, void* out) {
  if (n <= 0) return 0;
  const int total = crop_h * crop_w * C;
  dim3 g((total + 255) / 256, n);
  if (g.x > 64) g.x = 64;
  if (img_is_u8)
    k_crop<Src<unsigned char>, unsigned char, true><<<g, 256, 0, h->stream>>>(src_u8, H, W, C, centroids, sample_inds, crop_h,
                                                                             crop_w, (unsigned char*)out);
  else
    k_crop<Src<float>, float, false><<<g, 256, 0, h->stream>>>(src_f32, H, W, C, centroids, sample_inds, crop_h, crop_w,
                                                               (float*)out);
  SB_CHECK_LAUNCH(h);
  return 0;
}

template <typename TI>
using SbResizedFrameTexels = SbResizedTexels<TI, sizeof(TI) == 1>;

int sbk_crop(sb_handle_s* h, const void* images, int img_is_u8, int B, int H, int W, int C,
             const float* centroids, const int* sample_inds, int n, int crop_h, int crop_w, void* out,
             int out_is_u8_trunc) {
  return launch_crop<SbFrameTexels>(h, {(const unsigned char*)images, H, W, C}, {(const float*)images, H, W, C}, img_is_u8, H, W,
                                    C, centroids, sample_inds, n, crop_h, crop_w, out);
}

int sbk_crop_resized(sb_handle_s* h, const void* images, int img_is_u8, int B, int H, int W, int C, int Hr, int Wr,
                     const float* centroids, const int* sample_inds, int n, int crop_h, int crop_w, void* out) {
  return launch_crop<SbResizedFrameTexels>(h, {(const unsigned char*)images, H, W, C, Hr, Wr}, {(const float*)images, H, W, C, Hr, Wr},
                                           img_is_u8, Hr, Wr, C, centroids, sample_inds, n, crop_h, crop_w, out);
}

int sbk_lines(sb_handle_s* h, const float* pafs, int Hp, int Wp, int C2, const float* lines_in,
              const float* peaks, const int* edge_peak_inds, const int* edge_inds, int n, int P,
              float pafs_stride, float max_edge_length, float dist_w, int* out_subs, float* out_lines,
              float* out_scores) {
  if (n <= 0) return 0;
  k_lines<<<(n + 3) / 4, 128, 0, h->stream>>>(pafs, Hp, Wp, C2, lines_in, peaks, edge_peak_inds, edge_inds, n, P,
                                              pafs_stride, max_edge_length, dist_w, out_subs, out_lines, out_scores);
  SB_CHECK_LAUNCH(h);
  return 0;
}

int sbk_integral(sb_handle_s* h, const float* cms, int N, int Hh, int Ww, int C, const float* xv,
                 const float* yv, float* x_hat, float* y_hat) {
  if (N * C <= 0) return 0;
  k_integral<<<(N * C + 3) / 4, 128, 0, h->stream>>>(cms, N, Hh, Ww, C, xv, yv, x_hat, y_hat);
  SB_CHECK_LAUNCH(h);
  return 0;
}

int sbk_local_dir(sb_handle_s* h, const float* patches, int N, float delta, float* out) {
  if (N <= 0) return 0;
  k_local_dir<<<(N + 127) / 128, 128, 0, h->stream>>>(patches, N, delta, out);
  SB_CHECK_LAUNCH(h);
  return 0;
}
