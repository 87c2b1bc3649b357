// Identity tracker on the device (sleap/nn/tracking.py:542-844 Tracker.track with the simple and simple-max-tracks
// candidate makers; the similarities, matchers and culling of sleap/nn/tracker/components.py).
//
// k_track runs as one CTA per call and walks the call's frames in order, as the host calls Tracker.track once per
// frame.  Per frame:
//   1. one thread per instance: visible-node count, nanmedian centroid and nanmin / nanmax box;
//   2. thread 0: pre-cull (cull_frame_instances / nms_fast), then the candidate pool and its tracks in first-appearance
//      order (FrameMatches.from_candidate_instances' by_track);
//   3. one warp per (instance, track) pair, one lane per candidate: the similarities in float64, then max (NaN
//      propagates, as np.max) or np.quantile's linear interpolation (numpy's _lerp, both branches); cost = -sim, NaN
//      -> +inf;
//   4. greedy matching by warp 0 (every pair, infinite ones included, cheapest first, ties by ascending flat index --
//      np.argsort(kind="stable")), or thread 0 solving SciPy's linear_sum_assignment (sb_lsap.cuh);
//   5. thread 0: the tracked list (matches in matching order, then new tracks), then the queue update.
// The sums restate numpy's: np.nansum is the pairwise sum (8 accumulators from 8 elements on), np.linalg.norm of a
// 2-vector is sqrt(fma(y, y, x * x)) (OpenBLAS ddot).  Built with -fmad=false so that no other product is contracted.
// The queues live in device memory between calls: the simple maker keeps a ring of the last track_window frames'
// tracked instances; the max-tracks maker keeps, per track in queue-table insertion order, a ring of its last
// track_window instances.
#include <algorithm>
#include <cmath>

#include "sb_common.cuh"
#include "sb_lsap.cuh"

namespace {

constexpr int kTrackThreads = 256;
constexpr int kTrackWarps = kTrackThreads / 32;
constexpr int kTrackMaxInstances = 128;
constexpr int kTrackMaxNodes = 64;
constexpr int kTrackMaxWindow = 64;
constexpr int kTrackMaxTable = 65536;
constexpr int kGeo = 7;                         // per instance: centroid x, y | box y1, x1, y2, x2 | visible nodes

struct TrackCfg {
  int maker, sim, match, W, max_tracks, max_tracking, min_match_points, min_new_track_points;
  double robust;
  int cull_target, cull_use_iou;
  double cull_iou;
  int oks_weight, oks_norm;
  int C, I, T;                                  // nodes, instances per frame, queue-table capacity
  int NE, NT;                                   // queue entries, most tracks in one frame's pool
};

struct TrackState {
  long long next_t;
  int n_spawned, head, len, n_table;            // head / len: the simple maker's ring of frames
  int status, n_done;                           // status: 0, SB_TRACK_INFEASIBLE, 2 = queue table full, or
                                                // SB_TRACK_OVER_CAPACITY
};

struct TrackBufs {
  TrackState* st;
  const double* prec;                           // [C] OKS precision fitted to the skeleton
  // queue entries (simple: frame slot * I + k; max-tracks: table row * W + ring position)
  double* e_pts; double* e_conf; double* e_geo; int* e_tid; long long* e_t;
  int* ring_cnt; long long* ring_t;             // simple: per frame slot
  int* tab_tid; int* tab_len; int* tab_head;    // max-tracks: per table row
  // the call
  const double* pts; const double* conf; const double* score; const int* count; const double* hw; const long long* t_in;
  int* o_idx; int* o_tid; double* o_score; int* o_matched; int* o_n; long long* o_t;
  // per-frame scratch
  double* u_geo; int* live; int* order; int* dropped; int* kept;
  int* cand; int* trk_tid; int* trk_start; int* trk_mem;
  double* cost; int* m_row; int* m_col; unsigned char* used; unsigned char* lsap;
};

__device__ __forceinline__ bool isnan_d(double x) { return x != x; }
__device__ __forceinline__ double qnan() { return __longlong_as_double(0x7ff8000000000000ll); }
// np.maximum / np.minimum: NaN propagates
__device__ __forceinline__ double np_max(double a, double b) { return isnan_d(a) ? a : (isnan_d(b) ? b : (a > b ? a : b)); }
__device__ __forceinline__ double np_min(double a, double b) { return isnan_d(a) ? a : (isnan_d(b) ? b : (a < b ? a : b)); }
// Python's max(a, b) / min(a, b) on floats: the second argument only replaces the first when it compares larger / smaller
__device__ __forceinline__ double py_max(double a, double b) { return b > a ? b : a; }
__device__ __forceinline__ double py_min(double a, double b) { return b < a ? b : a; }

// numpy's pairwise summation of n <= 128 terms (np.add.reduce on a contiguous float64 array); NaN terms count as 0
// (np.nansum)
template <typename F>
__device__ double np_nansum(F term, int n) {
  auto v = [&](int k) { const double x = term(k); return isnan_d(x) ? 0.0 : x; };
  if (n < 8) {
    double res = 0.0;
    for (int k = 0; k < n; ++k) res += v(k);
    return res;
  }
  double r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = v(j);
  int i = 8;
  for (; i < n - (n % 8); i += 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) r[j] += v(i + j);
  }
  double res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]));
  for (; i < n; ++i) res += v(i);
  return res;
}

// centroid (np.nanmedian, i.e. np.ma.median: (low + high) / 2 of the sorted visible values), box ([y1, x1, y2, x2]:
// nanmin / nanmax; NaN when no node is visible) and visible-node count of one instance
__device__ void instance_geo(const double* p, int C, double* g) {
  int nvis = 0;
  for (int k = 0; k < C; ++k) nvis += !(isnan_d(p[2 * k]) || isnan_d(p[2 * k + 1]));
  for (int a = 0; a < 2; ++a) {
    int m = 0;
    double lo = qnan(), hi = qnan();
    for (int k = 0; k < C; ++k) {
      const double x = p[2 * k + a];
      if (isnan_d(x)) continue;
      ++m;
      lo = isnan_d(lo) || x < lo ? x : lo;
      hi = isnan_d(hi) || x > hi ? x : hi;
    }
    double med = qnan();
    if (m > 0) {                                 // the values of rank (m - 1) / 2 and m / 2, ties by index
      double low = 0.0, high = 0.0;
      for (int k = 0; k < C; ++k) {
        const double x = p[2 * k + a];
        if (isnan_d(x)) continue;
        int rank = 0;
        for (int j = 0; j < C; ++j) {
          const double y = p[2 * j + a];
          rank += !isnan_d(y) && (y < x || (y == x && j < k));
        }
        if (rank == (m - 1) / 2) low = x;
        if (rank == m / 2) high = x;
      }
      med = (low + high) / 2.0;
    }
    g[a] = med;
    g[3 - a] = lo;                               // g = [cx, cy, y1, x1, y2, x2, visible nodes]
    g[5 - a] = hi;
  }
  g[6] = (double)nvis;
}

// similarity_function(ref = untracked instance, query = candidate)
__device__ double similarity(const TrackCfg& c, const double* __restrict__ prec, const double* r, const double* rc,
                             const double* rg, const double* q, const double* qc, const double* qg, double sw, double sh) {
  const int C = c.C;
  switch (c.sim) {
    case SB_TRACK_SIM_INSTANCE:
    case SB_TRACK_SIM_NORMALIZED_INSTANCE: {
      const bool nz = c.sim == SB_TRACK_SIM_NORMALIZED_INSTANCE;
      int n_ref = 0;
      for (int k = 0; k < C; ++k) {
        const double x = nz ? r[2 * k] / sw : r[2 * k], y = nz ? r[2 * k + 1] / sh : r[2 * k + 1];
        n_ref += !(isnan_d(x) || isnan_d(y));
      }
      const double s = np_nansum([&](int k) {
        const double dx = nz ? q[2 * k] / sw - r[2 * k] / sw : q[2 * k] - r[2 * k];
        const double dy = nz ? q[2 * k + 1] / sh - r[2 * k + 1] / sh : q[2 * k + 1] - r[2 * k + 1];
        return exp(-(dx * dx + dy * dy));
      }, C);
      return s / (double)n_ref;
    }
    case SB_TRACK_SIM_OBJECT_KEYPOINT: {
      int denom = C;
      if (c.oks_norm != SB_TRACK_OKS_ALL) {
        denom = 0;
        for (int k = 0; k < C; ++k) {
          const bool vr = !(isnan_d(r[2 * k]) || isnan_d(r[2 * k + 1]));
          const bool vq = !(isnan_d(q[2 * k]) || isnan_d(q[2 * k + 1]));
          denom += c.oks_norm == SB_TRACK_OKS_REF ? vr : (vr && vq);
        }
      }
      if (denom == 0) return 0.0;
      const double s = np_nansum([&](int k) {
        const double dx = q[2 * k] - r[2 * k], dy = q[2 * k + 1] - r[2 * k + 1];
        const double e = exp(-((dx * dx + dy * dy) * prec[k]));
        return c.oks_weight ? (rc[k] * qc[k]) * e : e;
      }, C);
      return s / (double)denom;
    }
    case SB_TRACK_SIM_CENTROID: {
      const double dx = rg[0] - qg[0], dy = rg[1] - qg[1];
      return -sqrt(__fma_rn(dy, dy, dx * dx));
    }
    default: {                                   // IoU: compute_iou(box(ref), box(query)), inclusive pixels
      const double iy1 = py_max(rg[2], qg[2]), ix1 = py_max(rg[3], qg[3]);
      const double iy2 = py_min(rg[4], qg[4]), ix2 = py_min(rg[5], qg[5]);
      const double inter = py_max(ix2 - ix1 + 1.0, 0.0) * py_max(iy2 - iy1 + 1.0, 0.0);
      const double area_a = (rg[5] - rg[3] + 1.0) * (rg[4] - rg[2] + 1.0);
      const double area_b = (qg[5] - qg[3] + 1.0) * (qg[4] - qg[2] + 1.0);
      return inter / (area_a + area_b - inter);
    }
  }
}

// cull_frame_instances(instances, cull_target, iou_threshold) on live[0..n): returns the survivors' count, in order
__device__ int pre_cull(const TrackCfg& c, const TrackBufs& bf, const double* sc, int n) {
  int* live = bf.live;
  for (int i = 0; i < n; ++i) live[i] = i;
  const int cnt = c.cull_target;
  if (cnt <= 0 || n <= cnt) return n;            // pre-cull off, or nothing to cull
  int nkeep = n;
  if (c.cull_use_iou) {                          // nms_fast on the boxes (as [x1, y1, x2, y2] columns of [y1, x1, y2, x2])
    int* alive = bf.order;
    for (int i = 0; i < n; ++i) {                // stable ascending argsort of the scores
      int j = i;
      while (j > 0 && sc[alive[j - 1]] > sc[i]) { alive[j] = alive[j - 1]; --j; }
      alive[j] = i;
    }
    const double* g = bf.u_geo;
    auto col = [&](int i, int k) { return g[i * kGeo + 2 + k]; };
    int na = n, nk = 0, nd = 0;
    while (na > 0) {
      const int top = alive[--na];
      bf.kept[nk++] = top;
      int nn = 0;
      for (int j = 0; j < na; ++j) {
        const int r = alive[j];
        const double area = (col(r, 2) - col(r, 0) + 1.0) * (col(r, 3) - col(r, 1) + 1.0);
        const double w = np_max(0.0, np_min(col(top, 2), col(r, 2)) - np_max(col(top, 0), col(r, 0)) + 1.0);
        const double h = np_max(0.0, np_min(col(top, 3), col(r, 3)) - np_max(col(top, 1), col(r, 1)) + 1.0);
        if ((w * h) / area > c.cull_iou) bf.dropped[nd++] = r; else alive[nn++] = r;
      }
      na = nn;
    }
    if (nd > 0 && nk < cnt) {                   // hand-back: dropped[:min(nd, nk - cnt)], a negative slice end
      for (int i = 1; i < nd; ++i) {             // stable sort by descending score
        const int x = bf.dropped[i];
        int j = i;
        while (j > 0 && sc[bf.dropped[j - 1]] < sc[x]) { bf.dropped[j] = bf.dropped[j - 1]; --j; }
        bf.dropped[j] = x;
      }
      const int take = max(0, nd + nk - cnt);
      for (int i = 0; i < take; ++i) bf.kept[nk++] = bf.dropped[i];
    }
    unsigned char* picked = bf.used;
    for (int i = 0; i < n; ++i) picked[i] = 0;
    for (int i = 0; i < nk; ++i) picked[bf.kept[i]] = 1;
    nkeep = 0;
    for (int i = 0; i < n; ++i)
      if (picked[i]) live[nkeep++] = i;
  }
  if (nkeep > cnt) {                             // drop the nkeep - cnt lowest scores (stable sort of the kept list)
    int* o = bf.order;
    for (int i = 0; i < nkeep; ++i) {
      int j = i;
      while (j > 0 && sc[o[j - 1]] > sc[live[i]]) { o[j] = o[j - 1]; --j; }
      o[j] = live[i];
    }
    unsigned char* gone = bf.used;
    for (int i = 0; i < n; ++i) gone[i] = 0;
    for (int i = 0; i < nkeep - cnt; ++i) gone[o[i]] = 1;
    int m = 0;
    for (int i = 0; i < nkeep; ++i)
      if (!gone[live[i]]) live[m++] = live[i];
    nkeep = m;
  }
  return nkeep;
}

__device__ __forceinline__ void copy_entry(const TrackCfg& c, const TrackBufs& bf, int e, const double* p,
                                           const double* pc, const double* g, int tid, long long t, int lane, int nl) {
  for (int k = lane; k < 2 * c.C; k += nl) bf.e_pts[(size_t)e * 2 * c.C + k] = p[k];
  for (int k = lane; k < c.C; k += nl) bf.e_conf[(size_t)e * c.C + k] = pc[k];
  for (int k = lane; k < kGeo; k += nl) bf.e_geo[(size_t)e * kGeo + k] = g[k];
  if (lane == 0) { bf.e_tid[e] = tid; bf.e_t[e] = t; }
}

__global__ void __launch_bounds__(kTrackThreads) k_track(TrackCfg c, TrackBufs bf, int B) {
  __shared__ double s_vals[kTrackWarps][kTrackMaxWindow];
  __shared__ int s_n[4];                         // live instances, candidates, tracks, tracked
  __shared__ int s_nm;                           // matches
  __shared__ long long s_t;
  __shared__ int s_dst[kTrackMaxInstances];      // queue entry of each tracked instance (-1: not queued)
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  TrackState* st = bf.st;
  const int C = c.C, I = c.I, W = c.W;
  if (tid == 0) st->n_done = 0;
  if (st->status) return;                        // a full queue table stays an error until sb_tracker_reset
  for (int b = 0; b < B; ++b) {
    const int n = bf.count[b];
    if (n > I) {                                 // a list longer than the capacity: frames b.. stay untracked
      if (tid == 0) { st->status = SB_TRACK_OVER_CAPACITY; st->n_done = b; }
      return;
    }
    const double* P = bf.pts + (size_t)b * I * C * 2;
    const double* PC = bf.conf + (size_t)b * I * C;
    const double* SC = bf.score + (size_t)b * I;
    const double sw = bf.hw ? bf.hw[2 * b + 1] : 1.0, sh = bf.hw ? bf.hw[2 * b] : 1.0;
    for (int i = tid; i < n; i += kTrackThreads) {
      double g[kGeo];
      instance_geo(P + (size_t)i * C * 2, C, g);
      for (int k = 0; k < kGeo; ++k) bf.u_geo[i * kGeo + k] = g[k];
    }
    __syncthreads();
    if (tid == 0) {
      s_t = bf.t_in[b] >= 0 ? bf.t_in[b] : st->next_t;
      const int nl = n > 0 ? pre_cull(c, bf, SC, n) : 0;
      int nc = 0, nt = 0;
      if (nl > 0) {
        if (c.maker == SB_TRACK_SIMPLE) {
          for (int f = 0; f < st->len; ++f) {
            const int slot = (st->head + f) % W;
            for (int k = 0; k < bf.ring_cnt[slot]; ++k) {
              const int e = slot * I + k;
              if (bf.e_geo[(size_t)e * kGeo + 6] < c.min_match_points) continue;
              bf.cand[nc++] = e;
              int j = 0;
              while (j < nt && bf.trk_tid[j] != bf.e_tid[e]) ++j;
              if (j == nt) bf.trk_tid[nt++] = bf.e_tid[e];
            }
          }
        } else {
          int counted = 0;
          for (int r = 0; r < st->n_table; ++r) {
            if (c.max_tracking && counted >= c.max_tracks) continue;
            ++counted;
            const int before = nc;
            for (int h = 0; h < bf.tab_len[r]; ++h) {
              const int e = r * W + (bf.tab_head[r] + h) % W;
              if (bf.e_geo[(size_t)e * kGeo + 6] >= c.min_match_points) bf.cand[nc++] = e;
            }
            if (nc > before) bf.trk_tid[nt++] = bf.tab_tid[r];
          }
        }
        // members of each track, in candidate order
        int m = 0;
        for (int j = 0; j < nt; ++j) {
          bf.trk_start[j] = m;
          for (int k = 0; k < nc; ++k)
            if (bf.e_tid[bf.cand[k]] == bf.trk_tid[j]) bf.trk_mem[m++] = bf.cand[k];
        }
        bf.trk_start[nt] = m;
      }
      s_n[0] = nl; s_n[1] = nc; s_n[2] = nt;
    }
    __syncthreads();
    const int nl = s_n[0], nt = s_n[2];
    // similarity matrix: one warp per (instance, track), one lane per candidate
    const bool quant = c.robust > 0.0 && c.robust < 1.0;
    for (int p = warp; p < nl * nt; p += kTrackWarps) {
      const int i = p / nt, j = p - i * nt;
      const int u = bf.live[i];
      const double* r = P + (size_t)u * C * 2;
      const double* rc = PC + (size_t)u * C;
      const double* rg = bf.u_geo + u * kGeo;
      const int m0 = bf.trk_start[j], mn = bf.trk_start[j + 1] - m0;
      double best = -(double)CUDART_INF_F;
      bool any_nan = false;
      for (int k = lane; k < mn; k += 32) {
        const int e = bf.trk_mem[m0 + k];
        const double s = similarity(c, bf.prec, r, rc, rg, bf.e_pts + (size_t)e * 2 * C, bf.e_conf + (size_t)e * C,
                                    bf.e_geo + (size_t)e * kGeo, sw, sh);
        if (isnan_d(s)) any_nan = true; else best = s > best ? s : best;
        if (quant) s_vals[warp][k] = s;
      }
      any_nan = __any_sync(0xffffffffu, any_nan);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) best = fmax(best, __shfl_xor_sync(0xffffffffu, best, o));
      __syncwarp();
      if (lane == 0) {
        double sim;
        if (any_nan) {
          sim = qnan();
        } else if (!quant) {
          sim = best;
        } else {                                 // np.quantile(s, robust), method "linear"
          double* v = s_vals[warp];
          for (int a = 1; a < mn; ++a) {
            const double x = v[a];
            int z = a;
            while (z > 0 && v[z - 1] > x) { v[z] = v[z - 1]; --z; }
            v[z] = x;
          }
          const double vi = (double)(mn - 1) * c.robust;
          double lo, hi, gamma;
          if (vi >= (double)(mn - 1)) { lo = hi = v[mn - 1]; gamma = vi + 1.0; }
          else if (vi < 0.0) { lo = hi = v[0]; gamma = vi; }
          else { const int f = (int)floor(vi); lo = v[f]; hi = v[f + 1]; gamma = vi - (double)f; }
          const double d = hi - lo;
          sim = gamma >= 0.5 ? hi - d * (1.0 - gamma) : lo + d * gamma;
        }
        const double cst = -sim;
        bf.cost[i * nt + j] = isnan_d(cst) ? (double)CUDART_INF_F : cst;
      }
      __syncwarp();
    }
    __syncthreads();
    // matching
    if (nl > 0 && nt > 0) {
      if (c.match == SB_TRACK_MATCH_GREEDY) {
        if (warp == 0) {
          unsigned char* ur = bf.used;
          unsigned char* uc = bf.used + I;
          for (int k = lane; k < nl; k += 32) ur[k] = 0;
          for (int k = lane; k < nt; k += 32) uc[k] = 0;
          __syncwarp();
          const int steps = min(nl, nt);
          for (int s = 0; s < steps; ++s) {
            double bv = (double)CUDART_INF_F;
            int bi = 0x7fffffff;
            for (int f = lane; f < nl * nt; f += 32) {
              const int i = f / nt, j = f - i * nt;
              if (ur[i] || uc[j]) continue;
              const double v = bf.cost[f];
              if (v < bv || (v == bv && f < bi)) { bv = v; bi = f; }
            }
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
              const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
              const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
              if (ov < bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
            }
            if (lane == 0) {
              const int i = bi / nt, j = bi - i * nt;
              ur[i] = 1; uc[j] = 1;
              bf.m_row[s] = i; bf.m_col[s] = j;
            }
            __syncwarp();
          }
          if (lane == 0) s_nm = steps;
        }
      } else if (tid == 0) {
        const int K = max(nl, nt);
        LsapScratch ls = carve_lsap(bf.lsap, K);
        const double* cm = bf.cost;
        const int nm = lsap_solve_cost([&](int i, int j) { return cm[i * nt + j]; }, nl, nt, ls, bf.m_row, bf.m_col);
        s_nm = nm;
        if (nm == 0) st->status = SB_TRACK_INFEASIBLE;
      }
    } else if (tid == 0) {
      s_nm = 0;
    }
    __syncthreads();
    if (st->status) return;                      // frame b stays untracked; nothing of it reaches the state
    // tracked list and queue slots
    if (tid == 0) {
      const long long t = s_t;
      int* oi = bf.o_idx + (size_t)b * I;
      int* ot = bf.o_tid + (size_t)b * I;
      double* os = bf.o_score + (size_t)b * I;
      int* om = bf.o_matched + (size_t)b * I;
      int no = 0;
      unsigned char* taken = bf.used + I + c.NT;
      for (int i = 0; i < nl; ++i) taken[i] = 0;
      for (int s = 0; s < s_nm; ++s) {
        const int i = bf.m_row[s], j = bf.m_col[s];
        taken[i] = 1;
        oi[no] = bf.live[i]; ot[no] = bf.trk_tid[j]; os[no] = -bf.cost[i * nt + j]; om[no] = 1; ++no;
      }
      for (int i = 0; i < nl; ++i) {
        if (taken[i]) continue;
        const int u = bf.live[i];
        if (bf.u_geo[u * kGeo + 6] < c.min_new_track_points) continue;
        if (c.maker == SB_TRACK_SIMPLE_MAX_TRACKS && c.max_tracking && st->n_table >= c.max_tracks) break;
        oi[no] = u; ot[no] = st->n_spawned++; os[no] = 0.0; om[no] = 0; ++no;
      }
      bf.o_n[b] = no;
      bf.o_t[b] = t;
      if (c.maker == SB_TRACK_SIMPLE) {
        int slot;
        if (st->len == W) { slot = st->head; st->head = (st->head + 1) % W; }
        else { slot = (st->head + st->len) % W; ++st->len; }
        bf.ring_cnt[slot] = no; bf.ring_t[slot] = t;
        for (int k = 0; k < no; ++k) s_dst[k] = slot * I + k;
        st->next_t = t + 1;
      } else {
        for (int k = 0; k < no; ++k) {
          int r = 0;
          while (r < st->n_table && bf.tab_tid[r] != ot[k]) ++r;
          if (r == st->n_table) {
            if (c.max_tracking && st->n_table >= c.max_tracks) { s_dst[k] = -1; continue; }
            if (st->n_table == c.T) { st->status = 2; break; }
            bf.tab_tid[r] = ot[k]; bf.tab_len[r] = 0; bf.tab_head[r] = 0; ++st->n_table;
          }
          int pos;
          if (bf.tab_len[r] == W) { pos = bf.tab_head[r]; bf.tab_head[r] = (bf.tab_head[r] + 1) % W; }
          else { pos = (bf.tab_head[r] + bf.tab_len[r]) % W; ++bf.tab_len[r]; }
          s_dst[k] = r * W + pos;
        }
      }
      s_n[3] = no;
    }
    __syncthreads();
    if (st->status) return;
    // copy the tracked instances into their queue entries, one warp per instance
    for (int k = warp; k < s_n[3]; k += kTrackWarps) {
      const int e = s_dst[k];
      if (e < 0) continue;
      const int u = bf.o_idx[(size_t)b * I + k];
      copy_entry(c, bf, e, P + (size_t)u * C * 2, PC + (size_t)u * C, bf.u_geo + u * kGeo, bf.o_tid[(size_t)b * I + k],
                 s_t, lane, 32);
    }
    __syncthreads();
    if (tid == 0) {
      if (c.maker == SB_TRACK_SIMPLE_MAX_TRACKS) {  // _next_t: last frame of the first longest queue, + 1
        int best = -1;
        for (int r = 0; r < st->n_table; ++r)
          if (best < 0 || bf.tab_len[r] > bf.tab_len[best]) best = r;
        st->next_t = best < 0 ? 0 : bf.e_t[best * W + (bf.tab_head[best] + bf.tab_len[best] - 1) % W] + 1;
      }
      st->n_done = b + 1;
    }
    __syncthreads();
  }
}

// The instance list the predictors build from one frame's grouping output (Predictor._frames_from_example): rows with
// every point NaN are skipped; with max_instances >= 0 only the highest scores stay, in sorted(..., reverse=True)
// order (stable).  One CTA per frame.
__global__ void k_track_prep(const float* __restrict__ ip, const float* __restrict__ iv, const float* __restrict__ isc,
                             const int* __restrict__ n_inst, int I_src, int C, int max_instances, double img_h,
                             double img_w, int I, double* pts, double* conf, double* score, int* count, double* hw,
                             long long* t) {
  __shared__ int s_keep[kTrackMaxInstances];
  __shared__ int s_n;
  const int b = blockIdx.x;
  const float* P = ip + (size_t)b * I_src * C * 2;
  const float* S = isc + (size_t)b * I_src;
  if (threadIdx.x == 0) {
    const int n = min(n_inst[b], I_src);
    int k = 0;
    for (int j = 0; j < n; ++j) {
      bool all_nan = true;
      for (int q = 0; q < 2 * C && all_nan; ++q) all_nan = P[(size_t)j * C * 2 + q] != P[(size_t)j * C * 2 + q];
      if (!all_nan) s_keep[k++] = j;
    }
    if (max_instances >= 0 && k > max_instances) {
      for (int a = 1; a < k; ++a) {              // stable sort by descending score
        const int x = s_keep[a];
        int z = a;
        while (z > 0 && S[s_keep[z - 1]] < S[x]) { s_keep[z] = s_keep[z - 1]; --z; }
        s_keep[z] = x;
      }
      k = max_instances;
    }
    s_n = k;
    count[b] = k; hw[2 * b] = img_h; hw[2 * b + 1] = img_w; t[b] = -1;
  }
  __syncthreads();
  const int k = s_n;
  for (int e = threadIdx.x; e < k * C; e += blockDim.x) {
    const int i = e / C, q = e - i * C, j = s_keep[i];
    pts[((size_t)b * I + i) * C * 2 + 2 * q] = (double)P[((size_t)j * C + q) * 2];
    pts[((size_t)b * I + i) * C * 2 + 2 * q + 1] = (double)P[((size_t)j * C + q) * 2 + 1];
    conf[((size_t)b * I + i) * C + q] = (double)iv[((size_t)b * I_src + j) * C + q];
  }
  for (int i = threadIdx.x; i < k; i += blockDim.x) score[(size_t)b * I + i] = (double)S[s_keep[i]];
}

// The instance list the predictors build from one frame of a top-down batch: the frame's crops offsets[b] + j,
// j < sel_count[b], in crop order, rows with every point NaN skipped; score = the centroid value sel_val[b * K + j].  No
// max_instances cut (top-down caps centroids only).  count[b] is the full length of the list, which may exceed I: only
// the first I rows are written, and k_track stops at such a frame.  One CTA per frame.
__global__ void k_track_prep_td(const float* __restrict__ ipts, const float* __restrict__ ivals, const float* __restrict__ sel_val,
                                const int* __restrict__ sel_count, const int* __restrict__ offsets, int K, int C, double img_h,
                                double img_w, int I, double* pts, double* conf, double* score, int* count, double* hw,
                                long long* t) {
  __shared__ int s_keep[kTrackMaxInstances];
  __shared__ int s_n;
  const int b = blockIdx.x;
  const int o = offsets[b];
  if (threadIdx.x == 0) {
    const int n = sel_count[b];
    int k = 0;
    for (int j = 0; j < n; ++j) {
      const float* p = ipts + (size_t)(o + j) * C * 2;
      bool all_nan = true;
      for (int q = 0; q < 2 * C && all_nan; ++q) all_nan = p[q] != p[q];
      if (all_nan) continue;
      if (k < I) s_keep[k] = j;                  // I <= kTrackMaxInstances
      ++k;
    }
    s_n = min(k, I);
    count[b] = k; hw[2 * b] = img_h; hw[2 * b + 1] = img_w; t[b] = -1;
  }
  __syncthreads();
  const int k = s_n;
  for (int e = threadIdx.x; e < k * C; e += blockDim.x) {
    const int i = e / C, q = e - i * C;
    const size_t src = (size_t)(o + s_keep[i]) * C + q;
    pts[((size_t)b * I + i) * C * 2 + 2 * q] = (double)ipts[src * 2];
    pts[((size_t)b * I + i) * C * 2 + 2 * q + 1] = (double)ipts[src * 2 + 1];
    conf[((size_t)b * I + i) * C + q] = (double)ivals[src];
  }
  for (int i = threadIdx.x; i < k; i += blockDim.x) score[(size_t)b * I + i] = (double)sel_val[(size_t)b * K + s_keep[i]];
}

// Per-frame track record: [n, flag, order[I], track id[I], tracking score[I]] (doubles; flag 0 = tracked, else the
// tracker's status: SB_TRACK_INFEASIBLE, 2 = queue table full, SB_TRACK_OVER_CAPACITY).  One CTA per frame.
__global__ void k_track_pack(const TrackState* st, const int* on, const int* oidx, const int* otid,
                             const double* oscore, int I, double* rec) {
  const int b = blockIdx.x;
  double* r = rec + (size_t)b * (2 + 3 * (size_t)I);
  const bool done = b < st->n_done;
  const int n = done ? on[b] : 0;
  if (threadIdx.x == 0) { r[0] = n; r[1] = done ? 0 : (st->status ? st->status : SB_TRACK_INFEASIBLE); }
  for (int k = threadIdx.x; k < I; k += blockDim.x) {
    r[2 + k] = k < n ? oidx[(size_t)b * I + k] : -1;
    r[2 + I + k] = k < n ? otid[(size_t)b * I + k] : -1;
    r[2 + 2 * I + k] = k < n ? oscore[(size_t)b * I + k] : 0.0;
  }
}

}  // namespace

struct SbTracker {
  TrackCfg cfg{};
  TrackBufs bf{};
  std::vector<void*> allocs;
  int cap_B = 0;
  void* io = nullptr;                           // per-call inputs / outputs, sized for cap_B frames
  ~SbTracker() {
    for (void* p : allocs) cudaFree(p);
    cudaFree(io);
  }
};

void sb_trackers_free(sb_handle_s* h) {
  for (SbTracker* t : h->trackers) delete t;
  h->trackers.clear();
}

SbTracker* sb_tracker_get(sb_handle_s* h, int id) {
  return (id >= 0 && id < (int)h->trackers.size()) ? h->trackers[id] : nullptr;
}
int sb_tracker_max_instances(const SbTracker* t) { return t->cfg.I; }
int sb_tracker_nodes(const SbTracker* t) { return t->cfg.C; }


namespace {

SbTracker* get_tracker(sb_handle_s* h, int id) { return sb_tracker_get(h, id); }

template <typename T>
int tr_alloc(sb_handle_s* h, SbTracker* t, T** p, size_t n) {
  int rc = sb_dev_alloc(h, p, std::max<size_t>(n, 1));
  if (rc == 0) t->allocs.push_back(*p);
  return rc;
}

// per-call inputs / outputs of cap frames, carved from one allocation (doubles, then 64-bit, then 32-bit ints)
struct TrackIo {
  double *pts, *conf, *score, *oscore, *hw;
  long long *t, *ot;
  int *count, *on, *oidx, *otid, *om;
};

int tracker_io(sb_handle_s* h, SbTracker* tr, int B, TrackIo& io) {
  const TrackCfg& c = tr->cfg;
  if (B > tr->cap_B) {
    cudaFree(tr->io);
    tr->io = nullptr; tr->cap_B = 0;
    const int cap = std::max(B, 64);
    const size_t per = (size_t)c.I * c.C * 3 * sizeof(double) + (size_t)c.I * (sizeof(double) * 2 + sizeof(int) * 3) +
                       sizeof(int) * 2 + sizeof(double) * 2 + sizeof(long long) * 2;
    int rc;
    if ((rc = sb_dev_alloc(h, (unsigned char**)&tr->io, per * cap + 256))) return rc;
    tr->cap_B = cap;
  }
  const int cap = tr->cap_B;
  double* dp = (double*)tr->io;
  io.pts = dp; dp += (size_t)cap * c.I * c.C * 2;
  io.conf = dp; dp += (size_t)cap * c.I * c.C;
  io.score = dp; dp += (size_t)cap * c.I;
  io.oscore = dp; dp += (size_t)cap * c.I;
  io.hw = dp; dp += (size_t)cap * 2;
  long long* lp = (long long*)dp;
  io.t = lp; lp += cap;
  io.ot = lp; lp += cap;
  int* ip = (int*)lp;
  io.count = ip; ip += cap;
  io.on = ip; ip += cap;
  io.oidx = ip; ip += (size_t)cap * c.I;
  io.otid = ip; ip += (size_t)cap * c.I;
  io.om = ip;
  return SB_OK;
}

TrackBufs call_bufs(const SbTracker* tr, const TrackIo& io, bool with_hw) {
  TrackBufs b = tr->bf;
  b.pts = io.pts; b.conf = io.conf; b.score = io.score; b.count = io.count; b.hw = with_hw ? io.hw : nullptr; b.t_in = io.t;
  b.o_idx = io.oidx; b.o_tid = io.otid; b.o_score = io.oscore; b.o_matched = io.om; b.o_n = io.on; b.o_t = io.ot;
  return b;
}

int tracker_clear(sb_handle_s* h, SbTracker* t) {
  SB_CUDA(h, cudaMemsetAsync(t->bf.st, 0, sizeof(TrackState), h->stream));
  SB_CUDA(h, cudaMemsetAsync(t->bf.ring_cnt, 0, sizeof(int) * t->cfg.W, h->stream));
  return SB_OK;
}

// k_track on the B instance lists a step's prep wrote into io, then one track record per frame into out_records
int track_and_pack(sb_handle_s* h, SbTracker* tr, int B, const TrackIo& io, double* out_records) {
  const TrackCfg& c = tr->cfg;
  k_track<<<1, kTrackThreads, 0, h->stream>>>(c, call_bufs(tr, io, true), B);
  SB_CHECK_LAUNCH(h);
  k_track_pack<<<B, 128, 0, h->stream>>>(tr->bf.st, io.on, io.oidx, io.otid, io.oscore, c.I, out_records);
  SB_CHECK_LAUNCH(h);
  return SB_OK;
}

}  // namespace

int sbk_track_step(sb_handle_s* h, SbTracker* tr, int B, const float* inst_peaks, const float* inst_vals,
                   const float* inst_scores, const int* n_inst, int I_src, int max_instances, double img_h, double img_w,
                   double* out_records) {
  TrackIo io;
  int rc;
  if ((rc = tracker_io(h, tr, B, io))) return rc;
  const TrackCfg& c = tr->cfg;
  k_track_prep<<<B, 128, 0, h->stream>>>(inst_peaks, inst_vals, inst_scores, n_inst, I_src, c.C, max_instances, img_h,
                                         img_w, c.I, io.pts, io.conf, io.score, io.count, io.hw, io.t);
  SB_CHECK_LAUNCH(h);
  return track_and_pack(h, tr, B, io, out_records);
}

int sbk_track_topdown(sb_handle_s* h, SbTracker* tr, int B, const float* ipts, const float* ivals, const float* sel_val,
                      const int* sel_count, const int* offsets, int K, double img_h, double img_w, double* out_records) {
  TrackIo io;
  int rc;
  if ((rc = tracker_io(h, tr, B, io))) return rc;
  const TrackCfg& c = tr->cfg;
  k_track_prep_td<<<B, 128, 0, h->stream>>>(ipts, ivals, sel_val, sel_count, offsets, K, c.C, img_h, img_w, c.I, io.pts, io.conf,
                                            io.score, io.count, io.hw, io.t);
  SB_CHECK_LAUNCH(h);
  return track_and_pack(h, tr, B, io, out_records);
}

extern "C" {

int sb_tracker_create(sb_handle_t h, const sb_tracker_params* p, int* out_tracker_id) {
  if (!h || !p || !out_tracker_id) return sb_fail(h, SB_ERR_INVALID, "sb_tracker_create: null argument");
  if (p->maker != SB_TRACK_SIMPLE && p->maker != SB_TRACK_SIMPLE_MAX_TRACKS)
    return sb_fail(h, SB_ERR_INVALID, "sb_tracker_create: candidate maker %d", p->maker);
  if (p->similarity < SB_TRACK_SIM_INSTANCE || p->similarity > SB_TRACK_SIM_IOU)
    return sb_fail(h, SB_ERR_INVALID, "sb_tracker_create: similarity %d", p->similarity);
  if (p->match != SB_TRACK_MATCH_GREEDY && p->match != SB_TRACK_MATCH_HUNGARIAN)
    return sb_fail(h, SB_ERR_INVALID, "sb_tracker_create: matcher %d", p->match);
  if (p->oks_normalization < SB_TRACK_OKS_ALL || p->oks_normalization > SB_TRACK_OKS_UNION)
    return sb_fail(h, SB_ERR_INVALID, "sb_tracker_create: oks normalization %d", p->oks_normalization);
  if (p->track_window < 1 || p->track_window > kTrackMaxWindow)
    return sb_fail(h, SB_ERR_INVALID, "sb_tracker_create: track_window %d outside 1..%d", p->track_window, kTrackMaxWindow);
  if (p->n_nodes < 1 || p->n_nodes > kTrackMaxNodes)
    return sb_fail(h, SB_ERR_INVALID, "sb_tracker_create: %d nodes outside 1..%d", p->n_nodes, kTrackMaxNodes);
  if (p->max_instances < 1 || p->max_instances > kTrackMaxInstances)
    return sb_fail(h, SB_ERR_INVALID, "sb_tracker_create: max_instances %d outside 1..%d", p->max_instances, kTrackMaxInstances);
  if (p->track_table < 1 || p->track_table > kTrackMaxTable)
    return sb_fail(h, SB_ERR_INVALID, "sb_tracker_create: track_table %d outside 1..%d", p->track_table, kTrackMaxTable);
  const bool capped = p->maker == SB_TRACK_SIMPLE_MAX_TRACKS && p->max_tracking && p->max_tracks > 0;
  if (capped && p->track_table < p->max_tracks)
    return sb_fail(h, SB_ERR_INVALID, "sb_tracker_create: track_table %d < max_tracks %d", p->track_table, p->max_tracks);
  if (p->cull_target < 0) return sb_fail(h, SB_ERR_INVALID, "sb_tracker_create: cull target %d", p->cull_target);
  if (p->n_oks_errors < 0 || (p->n_oks_errors > 0 && !p->oks_errors))
    return sb_fail(h, SB_ERR_INVALID, "sb_tracker_create: %d OKS errors", p->n_oks_errors);
  SB_CUDA(h, cudaSetDevice(h->device));
  SbTracker* t = new SbTracker();
  TrackCfg& c = t->cfg;
  c.maker = p->maker; c.sim = p->similarity; c.match = p->match; c.W = p->track_window;
  c.max_tracks = p->max_tracks; c.max_tracking = capped ? 1 : 0;
  c.min_match_points = p->min_match_points; c.min_new_track_points = p->min_new_track_points;
  c.robust = p->robust;
  c.cull_target = p->cull_target; c.cull_use_iou = p->cull_use_iou ? 1 : 0; c.cull_iou = p->cull_iou_threshold;
  c.oks_weight = p->oks_score_weighting ? 1 : 0; c.oks_norm = p->oks_normalization;
  c.C = p->n_nodes; c.I = p->max_instances;
  c.T = c.maker == SB_TRACK_SIMPLE ? 0 : p->track_table;
  c.NE = c.maker == SB_TRACK_SIMPLE ? c.W * c.I : c.T * c.W;
  c.NT = c.maker == SB_TRACK_SIMPLE ? c.W * c.I : c.T;
  // precision = 1 / (2 e^2), fitted to the skeleton: one value broadcasts, more are cut or edge-padded to n_nodes
  std::vector<double> prec(c.C);
  const int ne = p->n_oks_errors;
  for (int k = 0; k < c.C; ++k) {
    const double e = ne == 0 ? 1.0 : p->oks_errors[ne == 1 ? 0 : std::min(k, ne - 1)];
    prec[k] = 1.0 / (2.0 * (e * e));
  }
  TrackBufs& b = t->bf;
  const int K = std::max(c.I, c.NT);
  int rc = 0;
  double* prec_dev = nullptr;
  if ((rc = tr_alloc(h, t, &b.st, 1)) || (rc = tr_alloc(h, t, &prec_dev, c.C)) ||
      (rc = tr_alloc(h, t, &b.e_pts, (size_t)c.NE * 2 * c.C)) || (rc = tr_alloc(h, t, &b.e_conf, (size_t)c.NE * c.C)) ||
      (rc = tr_alloc(h, t, &b.e_geo, (size_t)c.NE * kGeo)) || (rc = tr_alloc(h, t, &b.e_tid, c.NE)) ||
      (rc = tr_alloc(h, t, &b.e_t, c.NE)) || (rc = tr_alloc(h, t, &b.ring_cnt, c.W)) || (rc = tr_alloc(h, t, &b.ring_t, c.W)) ||
      (rc = tr_alloc(h, t, &b.tab_tid, c.T)) || (rc = tr_alloc(h, t, &b.tab_len, c.T)) || (rc = tr_alloc(h, t, &b.tab_head, c.T)) ||
      (rc = tr_alloc(h, t, &b.u_geo, (size_t)c.I * kGeo)) || (rc = tr_alloc(h, t, &b.live, c.I)) ||
      (rc = tr_alloc(h, t, &b.order, c.I)) || (rc = tr_alloc(h, t, &b.dropped, c.I)) || (rc = tr_alloc(h, t, &b.kept, c.I)) ||
      (rc = tr_alloc(h, t, &b.cand, c.NE)) || (rc = tr_alloc(h, t, &b.trk_tid, c.NT)) ||
      (rc = tr_alloc(h, t, &b.trk_start, c.NT + 1)) || (rc = tr_alloc(h, t, &b.trk_mem, c.NE)) ||
      (rc = tr_alloc(h, t, &b.cost, (size_t)c.I * c.NT)) || (rc = tr_alloc(h, t, &b.m_row, K)) ||
      (rc = tr_alloc(h, t, &b.m_col, K)) || (rc = tr_alloc(h, t, &b.used, 2 * (size_t)c.I + c.NT)) ||
      (rc = tr_alloc(h, t, &b.lsap, lsap_scratch_bytes(K)))) {
    delete t;
    return rc;
  }
  b.prec = prec_dev;
  cudaError_t e = cudaMemcpyAsync(prec_dev, prec.data(), sizeof(double) * c.C, cudaMemcpyHostToDevice, h->stream);
  if (e != cudaSuccess || (rc = tracker_clear(h, t)) || (e = cudaStreamSynchronize(h->stream)) != cudaSuccess) {
    delete t;
    return rc ? rc : sb_fail(h, SB_ERR_CUDA, "sb_tracker_create: %s", cudaGetErrorString(e));
  }
  h->trackers.push_back(t);
  *out_tracker_id = (int)h->trackers.size() - 1;
  return SB_OK;
}

int sb_tracker_reset(sb_handle_t h, int tracker_id) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  SbTracker* t = get_tracker(h, tracker_id);
  if (!t) return sb_fail(h, SB_ERR_INVALID, "sb_tracker_reset: no tracker %d", tracker_id);
  SB_CUDA(h, cudaSetDevice(h->device));
  int rc;
  if ((rc = tracker_clear(h, t))) return rc;
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  return SB_OK;
}

int sb_tracker_destroy(sb_handle_t h, int tracker_id) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  SbTracker* t = get_tracker(h, tracker_id);
  if (!t) return sb_fail(h, SB_ERR_INVALID, "sb_tracker_destroy: no tracker %d", tracker_id);
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->stream);
  delete t;
  h->trackers[tracker_id] = nullptr;
  return SB_OK;
}

int sb_track_instances(sb_handle_t h, int tracker_id, int B, int I, const double* points, const double* point_conf,
                       const double* scores, const int32_t* counts, const double* img_hw, const int64_t* t_in,
                       int32_t* out_index, int32_t* out_track, double* out_score, int32_t* out_matched,
                       int32_t* out_n, int64_t* out_t, int32_t* out_n_done, int32_t* out_flag) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  SbTracker* tr = get_tracker(h, tracker_id);
  if (!tr) return sb_fail(h, SB_ERR_INVALID, "sb_track_instances: no tracker %d", tracker_id);
  if (!out_n_done || !out_flag) return sb_fail(h, SB_ERR_INVALID, "sb_track_instances: null status outputs");
  *out_n_done = 0; *out_flag = 0;
  if (B < 0 || I < 0) return sb_fail(h, SB_ERR_INVALID, "sb_track_instances: B = %d, I = %d", B, I);
  if (B == 0) return SB_OK;
  if (!points || !point_conf || !scores || !counts || !t_in || !out_index || !out_track || !out_score || !out_matched ||
      !out_n || !out_t)
    return sb_fail(h, SB_ERR_INVALID, "sb_track_instances: null buffer");
  TrackCfg& c = tr->cfg;
  if (c.sim == SB_TRACK_SIM_NORMALIZED_INSTANCE && !img_hw)
    return sb_fail(h, SB_ERR_INVALID, "sb_track_instances: normalized_instance needs img_hw");
  int B_ok = B;                                  // frames up to the first over-full one are tracked, then the error
  for (int b = 0; b < B; ++b)
    if (counts[b] < 0 || counts[b] > c.I || counts[b] > I) { B_ok = b; break; }
  SB_CUDA(h, cudaSetDevice(h->device));
  if (B_ok > 0) {
    TrackIo io;
    int rc;
    if ((rc = tracker_io(h, tr, B_ok, io))) return rc;
    double *d_pts = io.pts, *d_conf = io.conf, *d_score = io.score, *d_oscore = io.oscore, *d_hw = io.hw;
    long long *d_t = io.t, *d_ot = io.ot;
    int *d_count = io.count, *d_on = io.on, *d_oidx = io.oidx, *d_otid = io.otid, *d_om = io.om;
    // inputs: (B, I, ...) host rows -> (B, c.I, ...) device rows
    const size_t Iw = (size_t)std::min(I, c.I), ds = sizeof(double);
    SB_CUDA(h, cudaMemcpy2DAsync(d_pts, (size_t)c.I * c.C * 2 * ds, points, (size_t)I * c.C * 2 * ds, Iw * c.C * 2 * ds, B_ok,
                                 cudaMemcpyHostToDevice, h->stream));
    SB_CUDA(h, cudaMemcpy2DAsync(d_conf, (size_t)c.I * c.C * ds, point_conf, (size_t)I * c.C * ds, Iw * c.C * ds, B_ok,
                                 cudaMemcpyHostToDevice, h->stream));
    SB_CUDA(h, cudaMemcpy2DAsync(d_score, (size_t)c.I * ds, scores, (size_t)I * ds, Iw * ds, B_ok, cudaMemcpyHostToDevice,
                                 h->stream));
    if (img_hw) SB_CUDA(h, cudaMemcpyAsync(d_hw, img_hw, sizeof(double) * 2 * B_ok, cudaMemcpyHostToDevice, h->stream));
    SB_CUDA(h, cudaMemcpyAsync(d_t, t_in, sizeof(long long) * B_ok, cudaMemcpyHostToDevice, h->stream));
    SB_CUDA(h, cudaMemcpyAsync(d_count, counts, sizeof(int) * B_ok, cudaMemcpyHostToDevice, h->stream));
    k_track<<<1, kTrackThreads, 0, h->stream>>>(c, call_bufs(tr, io, img_hw != nullptr), B_ok);
    SB_CHECK_LAUNCH(h);
    TrackState st;
    SB_CUDA(h, cudaMemcpyAsync(&st, tr->bf.st, sizeof(TrackState), cudaMemcpyDeviceToHost, h->stream));
    SB_CUDA(h, cudaStreamSynchronize(h->stream));
    const int done = st.n_done;
    if (done > 0) {
      auto rows = [&](void* dst, const void* src, size_t elem) {
        return cudaMemcpy2DAsync(dst, (size_t)I * elem, src, (size_t)c.I * elem, (size_t)std::min(I, c.I) * elem, done,
                                 cudaMemcpyDeviceToHost, h->stream);
      };
      SB_CUDA(h, rows(out_index, d_oidx, sizeof(int)));
      SB_CUDA(h, rows(out_track, d_otid, sizeof(int)));
      SB_CUDA(h, rows(out_score, d_oscore, sizeof(double)));
      SB_CUDA(h, rows(out_matched, d_om, sizeof(int)));
      SB_CUDA(h, cudaMemcpyAsync(out_n, d_on, sizeof(int) * done, cudaMemcpyDeviceToHost, h->stream));
      SB_CUDA(h, cudaMemcpyAsync(out_t, d_ot, sizeof(long long) * done, cudaMemcpyDeviceToHost, h->stream));
      SB_CUDA(h, cudaStreamSynchronize(h->stream));
    }
    *out_n_done = done;
    if (st.status == SB_TRACK_INFEASIBLE) {
      *out_flag = SB_TRACK_INFEASIBLE;
      SB_CUDA(h, cudaMemsetAsync(&tr->bf.st->status, 0, sizeof(int), h->stream));
      SB_CUDA(h, cudaStreamSynchronize(h->stream));
      return SB_OK;
    }
    if (st.status)
      return sb_fail(h, SB_ERR_INVALID, "sb_track_instances: frame %d would grow the track queue table past %d tracks",
                     done, c.T);
  }
  if (B_ok < B)
    return sb_fail(h, SB_ERR_INVALID, "sb_track_instances: frame %d has %d instances (capacity %d, row length %d)", B_ok,
                   counts[B_ok], c.I, I);
  return SB_OK;
}

}  // extern "C"
