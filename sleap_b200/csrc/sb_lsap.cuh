// SciPy rectangular linear-sum-assignment (Crouse's shortest augmenting path), restated for one thread.  Shared by the
// PAF matching (sb_post.cu, float scores) and the identity tracker (sb_track.cu, float64 costs); each caller supplies
// cost(src, dst) as a double, +inf for a forbidden pair.  Returns the number of assignments (0 when SciPy would raise:
// a -inf entry or an infeasible matrix); rows ascending.
#pragma once
#include <math_constants.h>

struct LsapScratch {
  double* u; double* v; double* spc;
  int* path; int* col4row; int* row4col; int* remaining;
  unsigned char* SR; unsigned char* SC;
};

template <typename CostFn>
__device__ int lsap_solve_cost(CostFn cost_of, int n_src, int n_dst, LsapScratch s, int* out_rows, int* out_cols) {
  if (n_src == 0 || n_dst == 0) return 0;
  const bool transpose = n_dst < n_src;
  const int nr = transpose ? n_dst : n_src, nc = transpose ? n_src : n_dst;
  auto cost = [&](int i, int j) -> double { return transpose ? cost_of(j, i) : cost_of(i, j); };
  for (int i = 0; i < nr; ++i)
    for (int j = 0; j < nc; ++j)
      if (cost(i, j) == -(double)CUDART_INF_F) return 0;  // SciPy: invalid (-inf) entries raise
  for (int i = 0; i < nr; ++i) { s.u[i] = 0.0; s.col4row[i] = -1; }
  for (int j = 0; j < nc; ++j) { s.v[j] = 0.0; s.path[j] = -1; s.row4col[j] = -1; }
  for (int cur = 0; cur < nr; ++cur) {
    double minVal = 0.0;
    int i = cur;
    int num_remaining = nc;
    for (int it = 0; it < nc; ++it) s.remaining[it] = nc - it - 1;
    for (int k = 0; k < nr; ++k) s.SR[k] = 0;
    for (int k = 0; k < nc; ++k) { s.SC[k] = 0; s.spc[k] = (double)CUDART_INF_F; }
    int sink = -1;
    while (sink == -1) {
      int index = -1;
      double lowest = (double)CUDART_INF_F;
      s.SR[i] = 1;
      for (int it = 0; it < num_remaining; ++it) {
        const int j = s.remaining[it];
        const double r = minVal + cost(i, j) - s.u[i] - s.v[j];
        if (r < s.spc[j]) { s.path[j] = i; s.spc[j] = r; }
        if (s.spc[j] < lowest || (s.spc[j] == lowest && s.row4col[j] == -1)) {
          lowest = s.spc[j];
          index = it;
        }
      }
      minVal = lowest;
      if (minVal == (double)CUDART_INF_F) return 0;  // infeasible
      const int j = s.remaining[index];
      if (s.row4col[j] == -1) sink = j; else i = s.row4col[j];
      s.SC[j] = 1;
      s.remaining[index] = s.remaining[--num_remaining];
    }
    s.u[cur] += minVal;
    for (int k = 0; k < nr; ++k)
      if (s.SR[k] && k != cur) s.u[k] += minVal - s.spc[s.col4row[k]];
    for (int k = 0; k < nc; ++k)
      if (s.SC[k]) s.v[k] -= minVal - s.spc[k];
    int j = sink;
    while (true) {
      const int ii = s.path[j];
      s.row4col[j] = ii;
      const int tmp = s.col4row[ii];
      s.col4row[ii] = j;
      j = tmp;
      if (ii == cur) break;
    }
  }
  if (!transpose) {
    for (int i = 0; i < nr; ++i) { out_rows[i] = i; out_cols[i] = s.col4row[i]; }
  } else {
    // rows of the transposed problem are dst; emit sorted by src (= col4row value), stable
    // argsort by insertion (values are distinct).
    int cnt = 0;
    for (int srci = 0; srci < nc; ++srci) {
      const int d = s.row4col[srci];
      if (d >= 0) { out_rows[cnt] = srci; out_cols[cnt] = d; ++cnt; }
    }
  }
  return nr;
}

__device__ __forceinline__ LsapScratch carve_lsap(unsigned char* raw, int K) {
  LsapScratch s;
  double* d = reinterpret_cast<double*>(raw);
  s.u = d; s.v = d + K; s.spc = d + 2 * K;
  int* ip = reinterpret_cast<int*>(d + 3 * K);
  s.path = ip; s.col4row = ip + K; s.row4col = ip + 2 * K; s.remaining = ip + 3 * K;
  s.SR = reinterpret_cast<unsigned char*>(ip + 4 * K);
  s.SC = s.SR + K;
  return s;
}
__host__ __device__ inline size_t lsap_scratch_bytes(int K) {
  return (size_t)K * (3 * sizeof(double) + 4 * sizeof(int) + 2) + 16;
}
