// wgmma implicit-GEMM convolution for sm_90a: NHWC fp16 activations, fp32 accumulation in registers.
//
// Replaces cuDNN's Conv2D / Conv2DTranspose as dispatched by the reference's Keras graph
// (sleap/nn/architectures/encoder_decoder.py:117-131, 304-310, 369-389; hourglass.py:36-45;
// heads.py:55-63).
//
// Mapping (one CTA = one 8x16-pixel output tile x one N tile of output channels):
//   GEMM M = 128 output pixels, N = C_out tile (16..256), K = taps x C_in.
//   A operand: TMA (cp.async.bulk.tensor.4d) loads an NHWC box [KC ch, 16 px, 8+halo rows] with
//     hardware zero fill outside the image (= TF "SAME" padding) into 128B/64B/32B-swizzled
//     shared memory, one pixel per row, i.e. exactly the canonical K-major wgmma layout.  The
//     x shift of a filter tap is baked into the TMA coordinate (one load per distinct dx); the
//     y shift is a whole number of 16-pixel rows = a swizzle-atom-aligned start-address offset,
//     so the three ky taps of one dx share one staged tile.
//   B operand: weights pre-arranged [tap][C_out][C_in] fp16 (K-major), TMA box [KC, N, 1].
//   D: two warpgroups, each m64nNk16 wgmma over 64 of the 128 pixels; epilogue through a shared-memory
//     staging tile -> bias / ReLU / BN affine -> fp16 (or fp32 for head outputs) NHWC stores into the
//     consumer's channel slice.
//   Conv2DTranspose(k3 / k4, s2) = four sub-pixel phase GEMMs over the input grid with strided stores: four launches, or
//     one persistent k_tconv_wg_hw launch over all four.
//   1x1 stride-2 convs (ResNet) = 1x1 stride-1 convs over a subsampled view of the input: the A tensor map gets the
//     output's H / W and doubled pixel / row pitches (TMA takes any 16-byte-multiple global strides).
//   Residual blocks (ResNet, add skips): the epilogue adds the shortcut tensor after the bias and applies the ADD's
//     ReLU, storing into the ADD's output slice.
#include <cuda.h>

#include <algorithm>

#include "sb_model.h"

namespace {

constexpr int TW = 16, TH = 8;          // output tile (pixels); M = 128
constexpr int MAX_GROUPS = 7, MAX_TAPS = 7;   // filter columns / rows of the widest kernel taken (7x7)
// dynamic shared memory every kernel here is opted in for (cudaFuncAttributeMaxDynamicSharedMemorySize); more than
// half of the SM's 227 KB, so a launch padded to this size is guaranteed to run one CTA per SM
constexpr size_t kMaxDynSmem = 225 * 1024;

struct TcTap { int row_off, w_tap; };
struct TcGroup { int dx, n_taps; TcTap taps[MAX_TAPS]; };

struct TcParams {
  int H, W;                    // iteration grid (input grid for tconv phases, output grid for convs)
  int tiles_x;
  int n_chunks, KC;
  int n_groups;
  TcGroup groups[MAX_GROUPS];
  int dy0, box_rows;
  int N, Cout;                 // wgmma N of this launch, valid output channels
  void* out;
  int out_f32, out_H, out_W, out_Ctot, out_coff;
  int oy_mul, oy_add, ox_mul, ox_add;
  const float* bias;
  const float* bn_scale;
  const float* bn_shift;
  int relu;
  void* pool_out;               // optional fused MaxPool2D(2,2) output (same dtype as out)
  int pool_H, pool_W, pool_Ctot, pool_coff;
  // optional residual shortcut (fp16 NHWC slice, same pixel grid as out): added after the bias, before the ReLU;
  // precision 2: its [lo | hi | hi] planes, Cout channels apart, are summed first
  const void* res;
  int res_Ctot, res_coff;
  int a_slot_bytes, b_slot_bytes, n_a_slots, n_b_slots;
  int a_tx_bytes, b_tx_bytes;
  int layout_type;             // wgmma descriptor layout: 1 = SW128, 2 = SW64, 3 = SW32
  int row_bytes;               // KC * 2
  // 1: the common epilogue shape (fp16 NHWC output, no BN affine, C_out a multiple of 16 covering the whole
  //    channel tile, 32-byte aligned channel slices for the output and the fused pool) runs tc_epilogue_cols_fast
  int epi_mode;
  // 1: the full-resolution output of this conv has no reader (only its fused 2x2 max-pool is consumed): skip the stores
  int skip_out;
  // precision 2 (split-fp16 activations): the C_out logical channels are stored as three fp16 planes [lo | hi | hi],
  // Cout channels apart, from out_coff / pool_coff (sb_kernels_direct.cuh: st_split); 0 for fp32 head outputs
  int split;
  // programmatic dependent launch: 1 = call griddepcontrol.launch_dependents after the prologue (host: only for launches
  // that own their SMs, so that the successor's CTAs wait for free SMs instead of sharing them)
  int pdl_trigger;
  // persistent form (k_conv_wg_p): output tiles of the launch, frames
  int n_tiles, batch;
  // halo form (k_conv_wg_h): the input slice (fp16 NHWC, H x W of the iteration grid), its pixel pitch and channel count
  const void* in;
  int in_Ctot, in_C;
};

#include "sb_tc_prims.cuh"

// bias / BN scale / BN shift of output channels [n0, n0 + N) -> shared memory (zeros / ones beyond Cout)
__device__ __forceinline__ void stage_params(const TcParams& P, float* s_par, int n0) {
  for (int i = threadIdx.x; i < P.N; i += blockDim.x) {
    const int co = n0 + i;
    const bool ok = co < P.Cout;
    s_par[i] = (ok && P.bias) ? P.bias[co] : 0.f;
    s_par[P.N + i] = (ok && P.bn_scale) ? P.bn_scale[co] : 1.f;
    s_par[2 * P.N + i] = (ok && P.bn_shift) ? P.bn_shift[co] : 0.f;
  }
}

// Shared epilogue: 16 accumulator columns of this thread's pixel -> bias / ReLU / BN -> stores
// (+ fused 2x2 max-pool).  q = warp of the epilogue: it holds tile pixels 32q .. 32q+31, one per lane.
template <int TWC = 0>   // TWC: tile width known at compile time (0 = P.tw)
__device__ __forceinline__ void tc_epilogue_cols(const TcParams& P, const float* __restrict__ s_par, const uint32_t (&r)[16],
                                                 int n0, int c0, bool valid, size_t pix, int b, int x0, int y0, int q, int lane) {
  // s_par: [3][N] = bias | bn_scale | bn_shift of this N tile, staged in shared memory once per CTA
  float v[16];
  const float4* pb = reinterpret_cast<const float4*>(s_par + c0);
  const float4* ps = reinterpret_cast<const float4*>(s_par + P.N + c0);
  const float4* ph = reinterpret_cast<const float4*>(s_par + 2 * P.N + c0);
#pragma unroll
  for (int j4 = 0; j4 < 4; ++j4) {
    const float4 bb = pb[j4];
    v[4 * j4 + 0] = __uint_as_float(r[4 * j4 + 0]) + bb.x;
    v[4 * j4 + 1] = __uint_as_float(r[4 * j4 + 1]) + bb.y;
    v[4 * j4 + 2] = __uint_as_float(r[4 * j4 + 2]) + bb.z;
    v[4 * j4 + 3] = __uint_as_float(r[4 * j4 + 3]) + bb.w;
  }
  if (P.relu) {
#pragma unroll
    for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], 0.f);
  }
  if (P.bn_scale != nullptr) {
#pragma unroll
    for (int j4 = 0; j4 < 4; ++j4) {
      const float4 sc = ps[j4], sh = ph[j4];
      v[4 * j4 + 0] = v[4 * j4 + 0] * sc.x + sh.x;
      v[4 * j4 + 1] = v[4 * j4 + 1] * sc.y + sh.y;
      v[4 * j4 + 2] = v[4 * j4 + 2] * sc.z + sh.z;
      v[4 * j4 + 3] = v[4 * j4 + 3] * sc.w + sh.w;
    }
  }
  if (P.split) {
    // v = hi + lo: both planes (and the second copy of hi that pairs with the consumer's Wl rows) are written; the fused
    // 2x2 max-pool takes the maximum of the fp32 values BEFORE they are split (max is not separable over hi / lo)
    const bool full = n0 + c0 + 16 <= P.Cout;
    auto store3 = [&](__half* base, int Ctot, int coff, const float (&x)[16]) {
      __align__(16) __half hh[16], ll[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        hh[j] = __float2half_rn(x[j]);
        ll[j] = __float2half_rn(x[j] - __half2float(hh[j]));
      }
      __half* p0 = base + coff + n0 + c0;
      if (full) {
        const bool wide = ((Ctot | (coff + n0) | P.Cout) & 15) == 0;
#pragma unroll
        for (int pl = 0; pl < 3; ++pl) {
          __half* pd = p0 + pl * P.Cout;
          const __half* src = pl == 0 ? ll : hh;
          if (wide) st_global_256(pd, *reinterpret_cast<const __half2 (*)[8]>(src));
          else {
            reinterpret_cast<uint4*>(pd)[0] = *reinterpret_cast<const uint4*>(src);
            reinterpret_cast<uint4*>(pd)[1] = *reinterpret_cast<const uint4*>(src + 8);
          }
        }
      } else {
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (n0 + c0 + j < P.Cout) { p0[j] = ll[j]; p0[P.Cout + j] = hh[j]; p0[2 * P.Cout + j] = hh[j]; }
      }
    };
    if (valid && !(P.pool_out != nullptr && P.skip_out))
      store3(reinterpret_cast<__half*>(P.out) + pix * P.out_Ctot, P.out_Ctot, P.out_coff, v);
    if (P.pool_out != nullptr) {
      const int tw = TWC ? TWC : TW;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        v[j] = fmaxf(v[j], __shfl_xor_sync(0xffffffffu, v[j], 1));
        v[j] = fmaxf(v[j], __shfl_xor_sync(0xffffffffu, v[j], tw));
      }
      const int lr = lane / tw, lc = lane % tw;
      if (valid && ((lc | lr) & 1) == 0) {
        const int py = (y0 >> 1) + ((q * (32 / tw) + lr) >> 1), px = (x0 >> 1) + (lc >> 1);
        store3(reinterpret_cast<__half*>(P.pool_out) + (((size_t)b * P.pool_H + py) * P.pool_W + px) * P.pool_Ctot, P.pool_Ctot, P.pool_coff, v);
      }
    }
    return;
  }
  if (P.pool_out != nullptr) {
    // fused MaxPool2D(2, strides=2) (fp16 outputs only): lanes of a warp hold tile pixels
    // (ty = q*(32/tw) + lane/tw, tx = lane%tw); the 2x2 partners are lane^1 (x) and lane^tw (y); lanes with
    // even tx and even ty store.  The max runs on the already rounded, packed halves: rounding is
    // monotonic, so max(round(a), round(b)) == round(max(a, b)) and this equals pooling the stored tensor.
    const int tw = TWC ? TWC : TW;
    __align__(16) __half2 h[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) h[j] = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
    if (valid && !P.skip_out) {
      __half* po = reinterpret_cast<__half*>(P.out) + pix * P.out_Ctot + P.out_coff + n0 + c0;
      if (n0 + c0 + 16 <= P.Cout) {
        if (((P.out_Ctot | (P.out_coff + n0)) & 15) == 0) st_global_256(po, h);
        else {
          reinterpret_cast<uint4*>(po)[0] = *reinterpret_cast<uint4*>(&h[0]);
          reinterpret_cast<uint4*>(po)[1] = *reinterpret_cast<uint4*>(&h[4]);
        }
      } else {
        const __half* hs = reinterpret_cast<const __half*>(h);
#pragma unroll
        for (int j = 0; j < 16; ++j)
          if (n0 + c0 + j < P.Cout) po[j] = hs[j];
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      uint32_t a = *reinterpret_cast<uint32_t*>(&h[j]);
      uint32_t o = __shfl_xor_sync(0xffffffffu, a, 1);
      __half2 m2 = __hmax2(*reinterpret_cast<__half2*>(&a), *reinterpret_cast<__half2*>(&o));
      a = *reinterpret_cast<uint32_t*>(&m2);
      o = __shfl_xor_sync(0xffffffffu, a, tw);
      h[j] = __hmax2(m2, *reinterpret_cast<__half2*>(&o));
    }
    const int lr = lane / tw, lc = lane % tw;
    if (valid && ((lc | lr) & 1) == 0 && n0 + c0 + 16 <= P.Cout) {
      const int py = (y0 >> 1) + ((q * (32 / tw) + lr) >> 1), px = (x0 >> 1) + (lc >> 1);
      __half* pp = reinterpret_cast<__half*>(P.pool_out) + (((size_t)b * P.pool_H + py) * P.pool_W + px) * P.pool_Ctot +
                   P.pool_coff + n0 + c0;
      if (((P.pool_Ctot | (P.pool_coff + n0)) & 15) == 0) st_global_256(pp, h);
      else {
        reinterpret_cast<uint4*>(pp)[0] = *reinterpret_cast<uint4*>(&h[0]);
        reinterpret_cast<uint4*>(pp)[1] = *reinterpret_cast<uint4*>(&h[4]);
      }
    }
    return;
  }
  if (!valid) return;
  if (P.out_f32) {
    float* po = reinterpret_cast<float*>(P.out) + pix * P.out_Ctot + P.out_coff + n0 + c0;
#pragma unroll
    for (int j = 0; j < 16; ++j)
      if (n0 + c0 + j < P.Cout) po[j] = v[j];
  } else {
    __half* po = reinterpret_cast<__half*>(P.out) + pix * P.out_Ctot + P.out_coff + n0 + c0;
    if (n0 + c0 + 16 <= P.Cout) {
      __align__(16) __half2 h[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) h[j] = __floats2half2_rn(v[2 * j], v[2 * j + 1]);
      if (((P.out_Ctot | (P.out_coff + n0)) & 15) == 0) st_global_256(po, h);
      else {
        reinterpret_cast<uint4*>(po)[0] = *reinterpret_cast<uint4*>(&h[0]);
        reinterpret_cast<uint4*>(po)[1] = *reinterpret_cast<uint4*>(&h[4]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < 16; ++j)
        if (n0 + c0 + j < P.Cout) po[j] = __float2half_rn(v[j]);
    }
  }
}

__device__ __forceinline__ float4 lds_f4(uint32_t saddr) {
  float4 v;
  asm("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(saddr));
  return v;
}

// Specialised form of tc_epilogue_cols for P.epi_mode == 1.  The generic routine re-derives, for every 16
// columns, facts that are fixed per launch (output dtype, BN, alignment, partial channel tiles), which makes the
// epilogue of the low-channel full-resolution layers instruction-issue bound.  Here the launch-invariant decisions are made on
// the host, the bias comes from shared memory through ld.shared (the generic path emitted generic LDs), ReLU
// is a branch-free max against 0 / -inf, and the output / pooled row pointers are computed once per tile.
template <int TWC, bool POOL>
__device__ __forceinline__ void tc_epilogue_cols_fast(uint32_t s_bias, const uint32_t (&r)[16], bool valid, __half* po, __half* pp,
                                                      bool pool_store, float lo, int tw_rt) {
  __align__(16) __half2 h[8];
#pragma unroll
  for (int j4 = 0; j4 < 4; ++j4) {
    const float4 bb = lds_f4(s_bias + 16u * j4);
    const float a0 = fmaxf(__uint_as_float(r[4 * j4 + 0]) + bb.x, lo), a1 = fmaxf(__uint_as_float(r[4 * j4 + 1]) + bb.y, lo);
    const float a2 = fmaxf(__uint_as_float(r[4 * j4 + 2]) + bb.z, lo), a3 = fmaxf(__uint_as_float(r[4 * j4 + 3]) + bb.w, lo);
    h[2 * j4] = __floats2half2_rn(a0, a1);
    h[2 * j4 + 1] = __floats2half2_rn(a2, a3);
  }
  if (valid) st_global_256(po, h);
  if (POOL) {
    const int tw = TWC ? TWC : tw_rt;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      uint32_t a = *reinterpret_cast<uint32_t*>(&h[j]);
      uint32_t o = __shfl_xor_sync(0xffffffffu, a, 1);
      __half2 m2 = __hmax2(*reinterpret_cast<__half2*>(&a), *reinterpret_cast<__half2*>(&o));
      a = *reinterpret_cast<uint32_t*>(&m2);
      o = __shfl_xor_sync(0xffffffffu, a, tw);
      h[j] = __hmax2(m2, *reinterpret_cast<__half2*>(&o));
    }
    if (pool_store) st_global_256(pp, h);
  }
}

constexpr int kConsumerThreads = 256;                 // two warpgroups: tile rows 0-63 / 64-127
constexpr int kConvThreads = kConsumerThreads + 32;   // + the TMA producer warp
// fp32 accumulator columns staged through shared memory per epilogue round (must divide N)
constexpr int stage_cols(int n) { return n % 32 == 0 ? 32 : 16; }

// Residual shortcut of output channels [n, n + 16) of pixel `pix`, added to the staged accumulators (before the bias; the
// epilogue then applies bias, the ADD's ReLU and the store): 16 contiguous fp16 channels of one pixel per thread, two
// 16-byte loads when the tile is full; precision 2: lo + hi of the [lo | hi | hi] planes, Cout channels apart.
__device__ __forceinline__ void tc_add_residual(const TcParams& P, uint32_t (&r)[16], size_t pix, int n) {
  const __half* pr = reinterpret_cast<const __half*>(P.res) + pix * P.res_Ctot + P.res_coff + n;
  if (!P.split && n + 16 <= P.Cout) {
    const uint4 q[2] = {reinterpret_cast<const uint4*>(pr)[0], reinterpret_cast<const uint4*>(pr)[1]};
    const __half2* hq = reinterpret_cast<const __half2*>(q);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float2 f = __half22float2(hq[j]);
      r[2 * j] = __float_as_uint(__uint_as_float(r[2 * j]) + f.x);
      r[2 * j + 1] = __float_as_uint(__uint_as_float(r[2 * j + 1]) + f.y);
    }
    return;
  }
#pragma unroll
  for (int j = 0; j < 16; ++j)
    if (n + j < P.Cout)
      r[j] = __float_as_uint(__uint_as_float(r[j]) + (P.split ? __half2float(pr[j]) + __half2float(pr[P.Cout + j]) : __half2float(pr[j])));
}

// Epilogue of 16 accumulator columns [c0, c0 + 16) of one tile pixel, read from the fp32 staging rows in shared memory
// (`src`: this pixel's 16 staged values).  Called by whole warps (the fused max-pool shuffles across lanes): lane l of
// warp q holds tile pixel 32 q + l.
__device__ __forceinline__ void tc_epilogue_chunk(const TcParams& P, const float* __restrict__ s_par, const float* src, int n0, int c0,
                                               bool valid, size_t pix, int b, int x0, int y0, int q, int lane) {
  uint32_t r[16];
#pragma unroll
  for (int j4 = 0; j4 < 4; ++j4) {
    const float4 v = reinterpret_cast<const float4*>(src)[j4];
    r[4 * j4 + 0] = __float_as_uint(v.x); r[4 * j4 + 1] = __float_as_uint(v.y);
    r[4 * j4 + 2] = __float_as_uint(v.z); r[4 * j4 + 3] = __float_as_uint(v.w);
  }
  if (P.res != nullptr && valid) tc_add_residual(P, r, pix, n0 + c0);
  if (P.epi_mode != 1) {
    tc_epilogue_cols<TW>(P, s_par, r, n0, c0, valid, pix, b, x0, y0, q, lane);
    return;
  }
  const float lo = P.relu ? 0.f : -INFINITY;
  __half* po = reinterpret_cast<__half*>(P.out) + pix * P.out_Ctot + P.out_coff + n0 + c0;
  if (P.pool_out == nullptr) {
    tc_epilogue_cols_fast<TW, false>(smem_u32(s_par + c0), r, valid, po, nullptr, false, lo, TW);
    return;
  }
  const int lr = lane / TW, lc = lane % TW;
  const bool pool_store = valid && ((lc | lr) & 1) == 0;
  const int py = (y0 >> 1) + ((q * (32 / TW) + lr) >> 1), px = (x0 >> 1) + (lc >> 1);
  __half* pp = reinterpret_cast<__half*>(P.pool_out) + (((size_t)b * P.pool_H + py) * P.pool_W + px) * P.pool_Ctot + P.pool_coff + n0 + c0;
  tc_epilogue_cols_fast<TW, true>(smem_u32(s_par + c0), r, valid && !P.skip_out, po, pp, pool_store, lo, TW);
}

__device__ __forceinline__ void consumer_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumerThreads) : "memory"); }

// Epilogue of one 128-pixel tile of k_conv_wg_p (all 256 consumer threads; warp / lane of the calling thread); k_conv_wg
// runs the same steps written out in its body.  Accumulators -> shared-memory
// staging, CW columns at a time -> one pixel per thread, 16 columns per call (bias / ReLU / BN / residual / fused max-pool /
// split planes).  Starts by writing the staging rows: a caller that ran an epilogue before must consumer_sync() first.
template <int N>
__device__ __forceinline__ void conv_epilogue(const TcParams& P, const float* __restrict__ s_par, float* s_stage, float (&acc)[N / 2],
                                              int x0, int y0, int n0, int b, int warp, int lane) {
  constexpr int CW = stage_cols(N), SP = CW + 4;   // staged columns per round, staging row pitch (floats)
  const int wg = warp >> 2;
  // fragment rows of this thread: 16 (warp % 4) + lane / 4 (+ 8) of its warpgroup's 64; columns 8 j + 2 (lane % 4) (+ 1)
  const int frow = wg * 64 + (warp & 3) * 16 + (lane >> 2), fcol = 2 * (lane & 3);
  // staging readers: pixel m = threadIdx.x % 128 (warp q = m / 32 as the fused pool expects), column half threadIdx.x / 128
  const int m = threadIdx.x & 127, half = threadIdx.x >> 7;
  const int iy = y0 + m / TW, ix = x0 + m % TW;
  const bool valid = (iy < P.H) && (ix < P.W);
  const size_t pix = ((size_t)b * P.out_H + (iy * P.oy_mul + P.oy_add)) * P.out_W + (ix * P.ox_mul + P.ox_add);
#pragma unroll
  for (int c0 = 0; c0 < N; c0 += CW) {
    if (c0 > 0) consumer_sync();     // the previous round's readers are done with the staging rows
#pragma unroll
    for (int jj = 0; jj < CW / 8; ++jj) {
      const int j = c0 / 8 + jj;
      *reinterpret_cast<float2*>(s_stage + frow * SP + 8 * jj + fcol) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(s_stage + (frow + 8) * SP + 8 * jj + fcol) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
    consumer_sync();
    const int cc = c0 + 16 * half;
    if (cc < c0 + CW && n0 + cc < P.Cout)     // warp-uniform
      tc_epilogue_chunk(P, s_par, s_stage + m * SP + 16 * half, n0, cc, valid, pix, b, x0, y0, warp & 3, lane);
  }
}

// Implicit-GEMM convolution on wgmma.  One CTA = one 16x8-pixel output tile x one N tile of output channels:
//   warp 8, lane 0: TMA producer -- per (input-channel chunk, filter column) one activation box into the A ring, per filter
//     tap one [N x KC] weight slice into the B ring (mbarrier full / empty pairs);
//   warps 0-7 (two warpgroups): warpgroup w multiplies tile rows [64 w, 64 w + 64) -- m64nNk16 wgmma, fp32 accumulators in
//     registers; a step's slots are released once the NEXT step's wgmma group has been issued and the step's own has
//     completed (wgmma.wait_group 1), so the tensor cores always have one group queued;
//   epilogue: accumulators -> shared-memory staging, CW columns at a time -> one pixel per thread, 16 columns per call
//     (bias / ReLU / BN / fused max-pool / split planes, as the scalar kernels do).
template <int KSTEPS, int N>
__global__ void __launch_bounds__(kConvThreads, 1) k_conv_wg(const __grid_constant__ CUtensorMap mapA,
                                                             const __grid_constant__ CUtensorMap mapB,
                                                             const __grid_constant__ TcParams P) {
  constexpr int CW = stage_cols(N), SP = CW + 4;   // staged columns per round, staging row pitch (floats)
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // carve shared memory (ring slots are 1024-aligned: required by the 128B swizzle atoms)
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* a_ring = base;
  uint8_t* b_ring = a_ring + (size_t)P.n_a_slots * P.a_slot_bytes;
  float* s_stage = reinterpret_cast<float*>(b_ring + (size_t)P.n_b_slots * P.b_slot_bytes);   // [128][SP]
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_stage + 128 * SP);
  uint64_t* fullA = bars;
  uint64_t* emptyA = fullA + P.n_a_slots;
  uint64_t* fullB = emptyA + P.n_a_slots;
  uint64_t* emptyB = fullB + P.n_b_slots;
  float* s_par = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(emptyB + P.n_b_slots) + 15) & ~(uintptr_t)15);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x;
  const int x0 = (tile % P.tiles_x) * TW, y0 = (tile / P.tiles_x) * TH;
  const int n0 = blockIdx.y * P.N;
  const int b = blockIdx.z;
  stage_params(P, s_par, n0);

  if (threadIdx.x == 0) {
    for (int i = 0; i < P.n_a_slots; ++i) { mbar_init(smem_u32(fullA + i), 1); mbar_init(smem_u32(emptyA + i), kConsumerThreads / 32); }
    for (int i = 0; i < P.n_b_slots; ++i) { mbar_init(smem_u32(fullB + i), 1); mbar_init(smem_u32(emptyB + i), kConsumerThreads / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapB) : "memory");
  }
  __syncthreads();

  if (P.pdl_trigger) griddep_launch();
  if (warp == kConsumerThreads / 32) {
    // ------------------------------ TMA producer ------------------------------
    if (lane == 0) {
      griddep_wait();                  // activations come from the previous kernel of the stream
      int sa = 0, sb = 0;
      uint32_t pha = 0, phb = 0;
      for (int ch = 0; ch < P.n_chunks; ++ch) {
        for (int g = 0; g < P.n_groups; ++g) {
          mbar_wait(smem_u32(emptyA + sa), pha ^ 1);
          mbar_expect_tx(smem_u32(fullA + sa), (uint32_t)P.a_tx_bytes);
          tma_load_4d(smem_u32(a_ring + (size_t)sa * P.a_slot_bytes), &mapA, smem_u32(fullA + sa), ch * P.KC,
                      x0 + P.groups[g].dx, y0 + P.dy0, b);
          for (int t = 0; t < P.groups[g].n_taps; ++t) {
            mbar_wait(smem_u32(emptyB + sb), phb ^ 1);
            mbar_expect_tx(smem_u32(fullB + sb), (uint32_t)P.b_tx_bytes);
            tma_load_3d(smem_u32(b_ring + (size_t)sb * P.b_slot_bytes), &mapB, smem_u32(fullB + sb), ch * P.KC, n0,
                        P.groups[g].taps[t].w_tap);
            if (++sb == P.n_b_slots) { sb = 0; phb ^= 1; }
          }
          if (++sa == P.n_a_slots) { sa = 0; pha ^= 1; }
        }
      }
    }
    return;
  }

  // ------------------------------ MMA (two warpgroups) ------------------------
  const int wg = warp >> 2;
  float acc[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  const uint64_t desc_hi = make_desc(0, P.row_bytes, P.layout_type);
  const uint32_t a_row0 = (uint32_t)(wg * 64 * P.row_bytes);
  int sa = 0, sb = 0, rel_a = -1, rel_b = -1;
  uint32_t pha = 0, phb = 0, scale_d = 0;
  for (int ch = 0; ch < P.n_chunks; ++ch) {
    for (int g = 0; g < P.n_groups; ++g) {
      mbar_wait(smem_u32(fullA + sa), pha);
      const uint32_t a_base = smem_u32(a_ring + (size_t)sa * P.a_slot_bytes) + a_row0;
      const int n_taps = P.groups[g].n_taps;
      for (int t = 0; t < n_taps; ++t) {
        mbar_wait(smem_u32(fullB + sb), phb);
        const uint64_t da = desc_hi + (uint64_t)((a_base + (uint32_t)(P.groups[g].taps[t].row_off * TW * P.row_bytes)) >> 4);
        const uint64_t db = desc_hi + (uint64_t)(smem_u32(b_ring + (size_t)sb * P.b_slot_bytes) >> 4);
        wgmma_fence();
        wgmma_reg_fence(acc);
#pragma unroll
        for (int k = 0; k < KSTEPS; ++k) {
          wgmma_f16<N>(acc, da + 2 * k, db + 2 * k, scale_d);
          scale_d = 1;
        }
        wgmma_commit();
        wgmma_reg_fence(acc);
        wgmma_wait<1>();               // the previous step's products are done: its slots may be refilled
        __syncwarp();
        if (lane == 0) {
          if (rel_b >= 0) mbar_arrive(smem_u32(emptyB + rel_b));
          if (rel_a >= 0) mbar_arrive(smem_u32(emptyA + rel_a));
        }
        rel_b = sb;
        rel_a = t == n_taps - 1 ? sa : -1;
        if (++sb == P.n_b_slots) { sb = 0; phb ^= 1; }
      }
      if (++sa == P.n_a_slots) { sa = 0; pha ^= 1; }
    }
  }
  wgmma_wait<0>();
  wgmma_reg_fence(acc);

  // ------------------------------ epilogue (all 256 consumer threads) ----------
  // (the same steps as conv_epilogue, written out: calling it, even force-inlined, changes this kernel's register allocation
  // and grows the N = 256 spills from 54 to 90 bytes)
  // fragment rows of this thread: 16 (warp % 4) + lane / 4 (+ 8) of its warpgroup's 64; columns 8 j + 2 (lane % 4) (+ 1)
  const int frow = wg * 64 + (warp & 3) * 16 + (lane >> 2), fcol = 2 * (lane & 3);
  // staging readers: pixel m = threadIdx.x % 128 (warp q = m / 32 as the fused pool expects), column half threadIdx.x / 128
  const int m = threadIdx.x & 127, half = threadIdx.x >> 7;
  const int iy = y0 + m / TW, ix = x0 + m % TW;
  const bool valid = (iy < P.H) && (ix < P.W);
  const size_t pix = ((size_t)b * P.out_H + (iy * P.oy_mul + P.oy_add)) * P.out_W + (ix * P.ox_mul + P.ox_add);
#pragma unroll
  for (int c0 = 0; c0 < N; c0 += CW) {
    if (c0 > 0) consumer_sync();     // the previous round's readers are done with the staging rows
#pragma unroll
    for (int jj = 0; jj < CW / 8; ++jj) {
      const int j = c0 / 8 + jj;
      *reinterpret_cast<float2*>(s_stage + frow * SP + 8 * jj + fcol) = make_float2(acc[4 * j], acc[4 * j + 1]);
      *reinterpret_cast<float2*>(s_stage + (frow + 8) * SP + 8 * jj + fcol) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
    }
    consumer_sync();
    const int cc = c0 + 16 * half;
    if (cc < c0 + CW && n0 + cc < P.Cout)     // warp-uniform
      tc_epilogue_chunk(P, s_par, s_stage + m * SP + 16 * half, n0, cc, valid, pix, b, x0, y0, warp & 3, lane);
  }
}

// Persistent form of k_conv_wg with resident weights (one N tile: C_out_pad <= 128).  The grid holds as many CTAs as fit on
// the GPU at once; each walks a static list of work items (pixel tile, frame): CTA u takes items u, u + gridDim.x, ...
// Barrier init, bias staging, descriptor prefetch and the weights happen once per CTA: the whole [chunk][step] bank of
// weight slices is loaded with the mapB boxes before the grid dependency is waited on, and there is no weight ring.  The
// activation ring runs on across items, so the producer stages the next tile's boxes while the consumers run the
// epilogue.  Every item issues exactly the wgmma sequence of k_conv_wg -- same (chunk, filter column, tap, k-step) order on
// the same operands -- so the outputs are bit-identical.
template <int KSTEPS, int N>
__global__ void __launch_bounds__(kConvThreads, N <= 64 ? 2 : 1) k_conv_wg_p(const __grid_constant__ CUtensorMap mapA,
                                                                          const __grid_constant__ CUtensorMap mapB,
                                                                          const __grid_constant__ TcParams P) {
  constexpr int SP = stage_cols(N) + 4;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* a_ring = base;
  uint8_t* bank = a_ring + (size_t)P.n_a_slots * P.a_slot_bytes;             // n_b_slots = n_chunks x steps weight slices
  float* s_stage = reinterpret_cast<float*>(bank + (size_t)P.n_b_slots * P.b_slot_bytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(s_stage + 128 * SP);
  uint64_t* fullA = bars;
  uint64_t* emptyA = fullA + P.n_a_slots;
  uint64_t* fullB = emptyA + P.n_a_slots;                                    // the bank has landed
  float* s_par = reinterpret_cast<float*>((reinterpret_cast<uintptr_t>(fullB + 1) + 15) & ~(uintptr_t)15);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_work = P.n_tiles * P.batch;
  stage_params(P, s_par, 0);

  if (threadIdx.x == 0) {
    for (int i = 0; i < P.n_a_slots; ++i) { mbar_init(smem_u32(fullA + i), 1); mbar_init(smem_u32(emptyA + i), kConsumerThreads / 32); }
    mbar_init(smem_u32(fullB), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapB) : "memory");
  }
  __syncthreads();

  if (warp == kConsumerThreads / 32) {
    // ------------------------------ TMA producer ------------------------------
    if (lane == 0) {
      // weights are static: load the bank while the predecessor drains
      mbar_expect_tx(smem_u32(fullB), (uint32_t)(P.n_b_slots * P.b_tx_bytes));
      int s = 0;
      for (int ch = 0; ch < P.n_chunks; ++ch)
        for (int g = 0; g < P.n_groups; ++g)
          for (int t = 0; t < P.groups[g].n_taps; ++t, ++s)
            tma_load_3d(smem_u32(bank + (size_t)s * P.b_slot_bytes), &mapB, smem_u32(fullB), ch * P.KC, 0, P.groups[g].taps[t].w_tap);
      griddep_wait();                                   // activations come from the previous kernel of the stream
      int sa = 0;
      uint32_t pha = 0;
      for (int w = blockIdx.x; w < n_work; w += gridDim.x) {
        if (w + (int)gridDim.x >= n_work) griddep_launch();   // last item of this CTA
        const int tile = w % P.n_tiles, b = w / P.n_tiles;
        const int x0 = (tile % P.tiles_x) * TW, y0 = (tile / P.tiles_x) * TH;
        for (int ch = 0; ch < P.n_chunks; ++ch) {
          for (int g = 0; g < P.n_groups; ++g) {
            mbar_wait(smem_u32(emptyA + sa), pha ^ 1);
            mbar_expect_tx(smem_u32(fullA + sa), (uint32_t)P.a_tx_bytes);
            tma_load_4d(smem_u32(a_ring + (size_t)sa * P.a_slot_bytes), &mapA, smem_u32(fullA + sa), ch * P.KC,
                        x0 + P.groups[g].dx, y0 + P.dy0, b);
            if (++sa == P.n_a_slots) { sa = 0; pha ^= 1; }
          }
        }
      }
    }
    return;
  }

  // ------------------------------ MMA (two warpgroups) + epilogue ------------------------
  const int wg = warp >> 2;
  float acc[N / 2];
  const uint64_t desc_hi = make_desc(0, P.row_bytes, P.layout_type);
  const uint32_t a_row0 = (uint32_t)(wg * 64 * P.row_bytes);
  const uint32_t b_base = smem_u32(bank);
  mbar_wait(smem_u32(fullB), 0);
  int sa = 0;
  uint32_t pha = 0;
  for (int w = blockIdx.x; w < n_work; w += gridDim.x) {
    const int tile = w % P.n_tiles, b = w / P.n_tiles;
    const int x0 = (tile % P.tiles_x) * TW, y0 = (tile / P.tiles_x) * TH;
#pragma unroll
    for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
    int rel_a = -1, s = 0;
    uint32_t scale_d = 0;
    for (int ch = 0; ch < P.n_chunks; ++ch) {
      for (int g = 0; g < P.n_groups; ++g) {
        mbar_wait(smem_u32(fullA + sa), pha);
        const uint32_t a_base = smem_u32(a_ring + (size_t)sa * P.a_slot_bytes) + a_row0;
        const int n_taps = P.groups[g].n_taps;
        for (int t = 0; t < n_taps; ++t, ++s) {
          const uint64_t da = desc_hi + (uint64_t)((a_base + (uint32_t)(P.groups[g].taps[t].row_off * TW * P.row_bytes)) >> 4);
          const uint64_t db = desc_hi + (uint64_t)((b_base + (uint32_t)(s * P.b_slot_bytes)) >> 4);
          wgmma_fence();
          wgmma_reg_fence(acc);
#pragma unroll
          for (int k = 0; k < KSTEPS; ++k) {
            wgmma_f16<N>(acc, da + 2 * k, db + 2 * k, scale_d);
            scale_d = 1;
          }
          wgmma_commit();
          wgmma_reg_fence(acc);
          wgmma_wait<1>();               // the previous step's products are done: its activation slot may be refilled
          __syncwarp();
          if (lane == 0 && rel_a >= 0) mbar_arrive(smem_u32(emptyA + rel_a));
          rel_a = t == n_taps - 1 ? sa : -1;
        }
        if (++sa == P.n_a_slots) { sa = 0; pha ^= 1; }
      }
    }
    wgmma_wait<0>();
    wgmma_reg_fence(acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(emptyA + rel_a));   // the item's last box: the producer is filling the next item's
    if (w != (int)blockIdx.x) consumer_sync();              // the previous item's epilogue readers are done with the staging rows
    conv_epilogue<N>(P, s_par, s_stage, acc, x0, y0, 0, b, warp, lane);
  }
}

// Halo form (form 2): persistent, weights resident, for 3x3 stride-1 convs with C_in <= 64 (one K chunk) and one N tile of
// <= 64 channels in the epi_mode == 1 shape (fp16 out, no BN, no residual).  A work item is a 16 x 8 BY-pixel tile of one
// frame, cut into 2 x BY blocks of 8x8 pixels (one m64 each).  Lane 0 of the producer warp (warp 8) loads the item's
// (8 BY + 2) x 18-pixel halo patch as one TMA box of the patch map (encode_patches) into a ring of patch slots: pixel rows
// [rows][18][KC ch] of KC * 2 bytes, swizzled at the row width (SW128 / SW64 / SW32 for KC 64 / 32 / 16; TMA zero fill
// outside the image and beyond C_in).  Every tap (ky, kx) of a block is then the same swizzled K-major operand at start
// offset (ky * 18 + kx) * KC * 2 bytes (SBO = one patch row): one load serves all nine taps.  Consumer warpgroups 0 and 1
// take alternate items
// (ping-pong), so one warpgroup's epilogue overlaps the other's wgmma.
// The epilogue runs from registers (halo_block_epilogue): a thread's two accumulator rows are vertically adjacent pixels.  Every
// output element gets the wgmma products of k_conv_wg -- the same m64nNk16 shape, (filter column, tap, k-step) order and
// operand values -- and the bias / ReLU / fp16 rounding / 2x2 max of tc_epilogue_cols_fast in the same order, so the
// outputs are bit-identical to forms 0 and 1.
constexpr int kHaloCols = 18;                                  // 16 output columns + 2
// 8x8 blocks along y per item: 16x16 px where N <= 32 and N x KC <= 1024, else 16x8 (ptxas: 16x16 at N = 32, KC = 64 spills)
constexpr int halo_by(int n, int kc) { return n <= 32 && n * kc <= 1024 ? 2 : 1; }
// A patch of `rows` x 18 pixels of KC channels (forms 2 and 3): the bytes of its TMA box, and its slot in a patch ring,
// rounded up to the swizzle pattern (8 rows of KC * 2 bytes) so that every slot starts on one.
constexpr int patch_box_bytes(int rows, int kc) { return rows * kHaloCols * kc * 2; }
constexpr int patch_slot_bytes(int rows, int kc) { return (patch_box_bytes(rows, kc) + 16 * kc - 1) / (16 * kc) * (16 * kc); }
constexpr int patch_layout(int kc) { return kc == 64 ? 1 : (kc == 32 ? 2 : 3); }   // wgmma descriptor: SW128 / SW64 / SW32

// lane t of each quad holds piece k of chunks 0..3 in v[k]; afterwards it holds pieces 0..3 of chunk t (two xor stages)
__device__ __forceinline__ void quad_transpose(uint32_t& v0, uint32_t& v1, uint32_t& v2, uint32_t& v3, int t) {
  const bool o1 = t & 1, o2 = t & 2;
  uint32_t r = __shfl_xor_sync(0xffffffffu, o1 ? v0 : v1, 1);
  if (o1) v0 = r; else v1 = r;
  r = __shfl_xor_sync(0xffffffffu, o1 ? v2 : v3, 1);
  if (o1) v2 = r; else v3 = r;
  r = __shfl_xor_sync(0xffffffffu, o2 ? v0 : v2, 2);
  if (o2) v0 = r; else v2 = r;
  r = __shfl_xor_sync(0xffffffffu, o2 ? v1 : v3, 2);
  if (o2) v1 = r; else v3 = r;
}

__device__ __forceinline__ uint32_t hmax2_u32(uint32_t a, uint32_t b) {
  const __half2 m = __hmax2(*reinterpret_cast<const __half2*>(&a), *reinterpret_cast<const __half2*>(&b));
  return *reinterpret_cast<const uint32_t*>(&m);
}

__device__ __forceinline__ float2 lds_f2(uint32_t saddr) {
  float2 v;
  asm("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(saddr));
  return v;
}

// Bias, ReLU and fp16 rounding of a thread's two wgmma fragment rows (columns 8 j + 2 t (+ 1), t = lane % 4), as in
// tc_epilogue_cols_fast: piece r * N / 8 + j of hv = channels 8 j + 2 t (+ 1) of row r, as half2 (s_bias: shared-memory
// address of the bias of the tile's first channel).
template <int N>
__device__ __forceinline__ void frag_rows_f16(const float (&acc)[N / 2], uint32_t s_bias, int t, float lo, uint32_t (&hv)[N / 4]) {
  constexpr int NJ = N / 8;                                    // 8-channel groups of the tile
#pragma unroll
  for (int j = 0; j < NJ; ++j) {
    const float2 bb = lds_f2(s_bias + 4u * (8 * j + 2 * t));
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const __half2 h2 = __floats2half2_rn(fmaxf(acc[4 * j + 2 * r] + bb.x, lo), fmaxf(acc[4 * j + 2 * r + 1] + bb.y, lo));
      hv[r * NJ + j] = *reinterpret_cast<const uint32_t*>(&h2);
    }
  }
}

// Stores of frag_rows_f16's pieces: a 4x4 transpose across the lanes of a quad turns the channel pairs into 16-byte stores of
// 8 contiguous channels; row r's channels [8 j, 8 j + 8) go to po + r * row_step + 8 j, where ok[r].
template <int N>
__device__ __forceinline__ void frag_rows_store(uint32_t (&hv)[N / 4], __half* po, size_t row_step, bool ok0, bool ok1, int t) {
  constexpr int NJ = N / 8;
#pragma unroll
  for (int c0 = 0; c0 < 2 * NJ; c0 += 4) {
    quad_transpose(hv[c0], hv[c0 + 1], hv[c0 + 2], hv[c0 + 3], t);
    const int c = c0 + t, r = c / NJ, j = c % NJ;
    if (r ? ok1 : ok0) *reinterpret_cast<uint4*>(po + r * row_step + 8 * j) = make_uint4(hv[c0], hv[c0 + 1], hv[c0 + 2], hv[c0 + 3]);
  }
}

// Register epilogue of one 8x8-pixel block of the halo-patch forms (2 and 3): output channels [n0, n0 + N) of this thread's
// two fragment rows, the vertically adjacent pixels (y, x) and (y + 1, x) of frame b (g = lane / 4, t = lane % 4; s_bias:
// shared-memory address of channel n0's bias).  Bias, ReLU and fp16 rounding as in tc_epilogue_cols_fast, then the 2x2 max
// on the rounded halves in the same order, max(max(h(y, x), h(y, x + 1)), max(h(y + 1, x), h(y + 1, x + 1))), on the
// even-column lane, which stores (its horizontal partner is lane ^ 4).
template <int N>
__device__ __forceinline__ void halo_block_epilogue(const TcParams& P, const float (&acc)[N / 2], uint32_t s_bias, int n0, int b,
                                                    int y, int x, int g, int t, float lo) {
  constexpr int NJ = N / 8;                                    // 8-channel groups of the tile
  uint32_t hv[2 * NJ];
  frag_rows_f16<N>(acc, s_bias, t, lo, hv);
  if (P.pool_out != nullptr) {
    constexpr int NJ4 = (NJ + 3) / 4 * 4;
    uint32_t pv[NJ4];
#pragma unroll
    for (int j = 0; j < NJ4; ++j) {
      if (j < NJ) {
        const uint32_t m0 = hmax2_u32(hv[j], __shfl_xor_sync(0xffffffffu, hv[j], 4));
        const uint32_t m1 = hmax2_u32(hv[NJ + j], __shfl_xor_sync(0xffffffffu, hv[NJ + j], 4));
        pv[j] = hmax2_u32(m0, m1);
      } else {
        pv[j] = 0u;
      }
    }
    __half* pp = reinterpret_cast<__half*>(P.pool_out) + (((size_t)b * P.pool_H + (y >> 1)) * P.pool_W + (x >> 1)) * P.pool_Ctot +
                 P.pool_coff + n0;
    const bool st = (g & 1) == 0 && y < P.H && x < P.W;
#pragma unroll
    for (int c0 = 0; c0 < NJ4; c0 += 4) {
      quad_transpose(pv[c0], pv[c0 + 1], pv[c0 + 2], pv[c0 + 3], t);
      if (st && c0 + t < NJ) *reinterpret_cast<uint4*>(pp + 8 * (c0 + t)) = make_uint4(pv[c0], pv[c0 + 1], pv[c0 + 2], pv[c0 + 3]);
    }
  }
  if (!P.skip_out) {
    __half* po = reinterpret_cast<__half*>(P.out) + (((size_t)b * P.out_H + y) * P.out_W + x) * P.out_Ctot + P.out_coff + n0;
    frag_rows_store<N>(hv, po, (size_t)P.out_W * P.out_Ctot, y < P.H && x < P.W, y + 1 < P.H && x < P.W, t);
  }
}

template <int KSTEPS, int N>
__global__ void __launch_bounds__(kConvThreads, 1) k_conv_wg_h(const __grid_constant__ CUtensorMap mapA,
                                                               const __grid_constant__ CUtensorMap mapB,
                                                               const __grid_constant__ TcParams P) {
  constexpr int KC = 16 * KSTEPS, BY = halo_by(N, KC), NB = 2 * BY;        // blocks per item: 2 along x, BY along y
  constexpr int PW = kHaloCols, RB = 2 * KC, BOX = patch_box_bytes(8 * BY + 2, KC), SLOT = patch_slot_bytes(8 * BY + 2, KC);
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* bank = base;                                        // 9 weight slices, swizzled as in k_conv_wg_p
  uint8_t* ring = bank + 9 * (size_t)P.b_slot_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(ring + (size_t)P.n_a_slots * SLOT);
  uint64_t* empty = full + P.n_a_slots;
  uint64_t* fullB = empty + P.n_a_slots;
  float* s_bias = reinterpret_cast<float*>(fullB + 1);          // [N]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_x = (P.W + 15) / 16, n_tiles = tiles_x * ((P.H + 8 * BY - 1) / (8 * BY));
  const int n_work = n_tiles * P.batch;
  for (int i = threadIdx.x; i < N; i += blockDim.x) s_bias[i] = (P.bias && i < P.Cout) ? P.bias[i] : 0.f;
  if (threadIdx.x == 0) {
    // full: the producer's expect_tx arrival + the box's bytes; empty: one arrival per warp of the consuming warpgroup
    for (int i = 0; i < P.n_a_slots; ++i) { mbar_init(smem_u32(full + i), 1); mbar_init(smem_u32(empty + i), 4); }
    mbar_init(smem_u32(fullB), 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapB) : "memory");
  }
  __syncthreads();

  if (warp == kConsumerThreads / 32) {
    // ------------------------------ producer warp ------------------------------
    if (lane == 0) {
      // weights are static: load the bank (slice kx * 3 + ky = filter tap (ky, kx)) while the predecessor drains
      mbar_expect_tx(smem_u32(fullB), (uint32_t)(9 * P.b_tx_bytes));
      for (int kx = 0; kx < 3; ++kx)
        for (int ky = 0; ky < 3; ++ky)
          tma_load_3d(smem_u32(bank + (size_t)(kx * 3 + ky) * P.b_slot_bytes), &mapB, smem_u32(fullB), 0, 0, ky * 3 + kx);
      griddep_wait();                                          // activations come from the previous kernel of the stream
      for (int i = 0, w = blockIdx.x; w < n_work; ++i, w += gridDim.x) {
        if (w + (int)gridDim.x >= n_work) griddep_launch();    // last item of this CTA
        const int s = i % P.n_a_slots;
        mbar_wait(smem_u32(empty + s), ((i / P.n_a_slots) & 1) ^ 1);
        const int tile = w % n_tiles, b = w / n_tiles;
        mbar_expect_tx(smem_u32(full + s), (uint32_t)BOX);       // zero-filled bytes count too
        tma_load_4d(smem_u32(ring + (size_t)s * SLOT), &mapA, smem_u32(full + s), 0, (tile % tiles_x) * 16 - 1,
                    (tile / tiles_x) * (8 * BY) - 1, b);
      }
    }
    return;
  }

  // ------------------------------ consumers: warpgroup wg takes the CTA's items wg, wg + 2, ... ------------------------------
  const int wg = warp >> 2, q = warp & 3, g = lane >> 2, t = lane & 3;
  const float lo = P.relu ? 0.f : -INFINITY;
  const uint64_t desc_a = make_desc(0, RB, patch_layout(KC), PW * RB);
  const uint64_t desc_b = make_desc(0, P.row_bytes, P.layout_type);
  const uint32_t b_base = smem_u32(bank);
  mbar_wait(smem_u32(fullB), 0);
  float acc[NB][N / 2];
  for (int i = wg, w = blockIdx.x + wg * (int)gridDim.x; w < n_work; i += 2, w += 2 * (int)gridDim.x) {
    const int s = i % P.n_a_slots;
    mbar_wait(smem_u32(full + s), (i / P.n_a_slots) & 1);
    const uint32_t a_base = smem_u32(ring + (size_t)s * SLOT);
    wgmma_fence();
#pragma unroll
    for (int bk = 0; bk < NB; ++bk) wgmma_reg_fence(acc[bk]);
#pragma unroll
    for (int kx = 0; kx < 3; ++kx)
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int k = 0; k < KSTEPS; ++k) {
          const uint64_t db = desc_b + (uint64_t)((b_base + (uint32_t)((kx * 3 + ky) * P.b_slot_bytes)) >> 4) + 2 * k;
#pragma unroll
          for (int bk = 0; bk < NB; ++bk) {
            const uint32_t a = a_base + (uint32_t)(((8 * (bk >> 1) + ky) * PW + 8 * (bk & 1) + kx) * RB + 32 * k);
            wgmma_f16<N>(acc[bk], desc_a + (uint64_t)(a >> 4), db, (kx | ky | k) ? 1u : 0u);
          }
        }
    wgmma_commit();
#pragma unroll
    for (int bk = 0; bk < NB; ++bk) wgmma_reg_fence(acc[bk]);
    wgmma_wait<0>();
#pragma unroll
    for (int bk = 0; bk < NB; ++bk) wgmma_reg_fence(acc[bk]);
    __syncwarp();
    if (lane == 0) mbar_arrive(smem_u32(empty + s));           // the patch slot may be refilled

    const int tile = w % n_tiles, b = w / n_tiles;
    const int x0 = (tile % tiles_x) * 16, y0 = (tile / tiles_x) * (8 * BY);
#pragma unroll
    for (int bk = 0; bk < NB; ++bk)
      halo_block_epilogue<N>(P, acc[bk], smem_u32(s_bias), 0, b, y0 + 8 * (bk >> 1) + 2 * q, x0 + 8 * (bk & 1) + g, g, t, lo);
  }
}

// Wide form (form 3): persistent, warp-specialized, for the 3x3 stride-1 convs of the 64-512-channel layers, whose weight
// banks do not fit in shared memory.  The streaming form re-reads every weight slice from L2 for each 128 output pixels;
// here a work item is 16 x 8 BY output pixels x one N tile (N <= 128) x one frame, cut into 2 x BY blocks of 8x8 pixels,
// and both consumer warpgroups (BY blocks each) read every weight slice, so one L2 read of a slice feeds 256 (N > 64) or
// 512 (N <= 64) pixels.  K = 9 taps x C_in runs in chunks of 64 input channels (the last zero-filled beyond C_in).
//   warpgroup 0 (registers cut to 56): lane 0 of warp 0 loads one halo patch per (item, chunk) in form 2's layout (128B-
//     swizzled 64-channel pixel rows [8 BY + 2][18][64], one TMA box of the patch map, zero outside the image and beyond
//     C_in) into a ring of patch slots; lane 0 of warp 1 streams the [N x 64] weight slices (SW128, TMA) in (chunk, filter
//     column, tap) order into a ring of weight slots.  The weights never wait on the grid dependency, so the first ring is
//     in flight while the predecessor drains.
//   warpgroups 1, 2 (registers raised to 224): per weight slice, m64nNk16 wgmma over all k-steps and the warpgroup's
//     blocks as one group; a slice's slot is released (one arrival per consumer warp, 8 in all) once the next slice's
//     group is issued and its own has completed, a patch slot after the chunk's last slice.  Then the register epilogue of
//     form 2 (halo_block_epilogue), for channels [n0, n0 + N).
// Every output element gets the wgmma products of k_conv_wg -- the (chunk, filter column, tap, k-step) order on the same
// operand values -- and form 2's epilogue arithmetic, so the outputs are bit-identical to forms 0, 1 and 2.
// The 128 accumulators of a consumer thread need more than the 168 registers per thread that any CTA of more than 8 warps
// gets at one CTA per SM (a quarter of the register file holds at most 3 warps of 170).  So the CTA is three warpgroups,
// and the consumers take what the producer warpgroup gives back: 128 x (168 - 56) = 256 x (224 - 168).
constexpr int kWideThreads = 384;
constexpr int wide_by(int n) { return n <= 64 ? 4 : 2; }       // 8x8 block rows per item: 128 accumulators per consumer thread
constexpr int wide_rows(int n) { return 8 * wide_by(n) + 2; }

template <int N>
__global__ void __launch_bounds__(kWideThreads, 1) k_conv_wg_hw(const __grid_constant__ CUtensorMap mapA,
                                                                const __grid_constant__ CUtensorMap mapB,
                                                                const __grid_constant__ TcParams P) {
  constexpr int BY = wide_by(N), PW = kHaloCols, RB = 128, BOX = patch_box_bytes(wide_rows(N), 64),
                SLOT = patch_slot_bytes(wide_rows(N), 64);
  constexpr int WSLOT = N * 128;                               // one [N x 64-channel] weight slice
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* wring = base;                                       // n_b_slots weight slices (1024-aligned: SW128 atoms)
  uint8_t* pring = wring + (size_t)P.n_b_slots * WSLOT;        // n_a_slots patches
  uint64_t* pfull = reinterpret_cast<uint64_t*>(pring + (size_t)P.n_a_slots * SLOT);
  uint64_t* pempty = pfull + P.n_a_slots;
  uint64_t* wfull = pempty + P.n_a_slots;
  uint64_t* wempty = wfull + P.n_b_slots;
  float* s_bias = reinterpret_cast<float*>(wempty + P.n_b_slots);   // [Cout]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // work item w = (N tile fastest, pixel tile, frame): the N tiles of one pixel tile run side by side and share its patches in L2
  const int tiles_x = (P.W + 15) / 16, n_pt = tiles_x * ((P.H + 8 * BY - 1) / (8 * BY));
  const int n_nt = P.Cout / N, n_work = n_nt * n_pt * P.batch;
  for (int i = threadIdx.x; i < P.Cout; i += blockDim.x) s_bias[i] = P.bias ? P.bias[i] : 0.f;
  if (threadIdx.x == 0) {
    // full: the producer's expect_tx arrival + the box's bytes; empty: one arrival per consumer warp
    for (int i = 0; i < P.n_a_slots; ++i) { mbar_init(smem_u32(pfull + i), 1); mbar_init(smem_u32(pempty + i), 8); }
    for (int i = 0; i < P.n_b_slots; ++i) { mbar_init(smem_u32(wfull + i), 1); mbar_init(smem_u32(wempty + i), 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapB) : "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------ producer warpgroup ------------------------------
    setmaxnreg_dec<56>();
    if (warp == 0 && lane == 0) {
      griddep_wait();                                          // activations come from the previous kernel of the stream
      for (int i = 0, w = blockIdx.x; w < n_work; w += gridDim.x) {
        if (w + (int)gridDim.x >= n_work) griddep_launch();    // last item of this CTA
        const int pt = (w / n_nt) % n_pt, b = w / (n_nt * n_pt);
        const int xs = (pt % tiles_x) * 16 - 1, ys = (pt / tiles_x) * (8 * BY) - 1;
        for (int ch = 0; ch < P.n_chunks; ++ch, ++i) {
          const int s = i % P.n_a_slots;
          mbar_wait(smem_u32(pempty + s), ((i / P.n_a_slots) & 1) ^ 1);
          mbar_expect_tx(smem_u32(pfull + s), (uint32_t)BOX);    // zero-filled bytes count too
          tma_load_4d(smem_u32(pring + (size_t)s * SLOT), &mapA, smem_u32(pfull + s), ch * 64, xs, ys, b);
        }
      }
    } else if (warp == 1 && lane == 0) {
      // weights are static: no grid-dependency wait
      for (int j = 0, w = blockIdx.x; w < n_work; w += gridDim.x) {
        const int n0 = (w % n_nt) * N;
        for (int ch = 0; ch < P.n_chunks; ++ch)
          for (int kx = 0; kx < 3; ++kx)
            for (int ky = 0; ky < 3; ++ky, ++j) {
              const int s = j % P.n_b_slots;
              mbar_wait(smem_u32(wempty + s), ((j / P.n_b_slots) & 1) ^ 1);
              mbar_expect_tx(smem_u32(wfull + s), (uint32_t)WSLOT);
              tma_load_3d(smem_u32(wring + (size_t)s * WSLOT), &mapB, smem_u32(wfull + s), ch * 64, n0, ky * 3 + kx);
            }
      }
    }
    return;
  }

  // ------------------------------ consumers: warpgroup cw multiplies block rows [cw BY / 2, (cw + 1) BY / 2) ----------------
  setmaxnreg_inc<224>();
  const int cw = (warp >> 2) - 1, q = warp & 3, g = lane >> 2, t = lane & 3;
  const float lo = P.relu ? 0.f : -INFINITY;
  const uint64_t desc_a = make_desc(0, RB, 1, PW * RB);
  const uint64_t desc_b = make_desc(0, 128, 1);
  const uint32_t p_base = smem_u32(pring) + (uint32_t)(cw * (BY / 2) * 8 * PW * RB), w_base = smem_u32(wring);
  float acc[BY][N / 2];
  int ps = 0, ws = 0;
  uint32_t pph = 0, wph = 0;
  for (int w = blockIdx.x; w < n_work; w += gridDim.x) {
    int rel_w = -1, rel_p = -1;
    for (int ch = 0; ch < P.n_chunks; ++ch) {
      mbar_wait(smem_u32(pfull + ps), pph);
      const uint32_t a_base = p_base + (uint32_t)(ps * SLOT);
#pragma unroll
      for (int kx = 0; kx < 3; ++kx)
#pragma unroll
        for (int ky = 0; ky < 3; ++ky) {
          mbar_wait(smem_u32(wfull + ws), wph);
          const uint64_t db = desc_b + (uint64_t)((w_base + (uint32_t)(ws * WSLOT)) >> 4);
          wgmma_fence();
#pragma unroll
          for (int i = 0; i < BY; ++i) wgmma_reg_fence(acc[i]);
#pragma unroll
          for (int k = 0; k < 4; ++k)
#pragma unroll
            for (int i = 0; i < BY; ++i) {
              const uint32_t a = a_base + (uint32_t)(((8 * (i >> 1) + ky) * PW + 8 * (i & 1) + kx) * RB + 32 * k);
              wgmma_f16<N>(acc[i], desc_a + (uint64_t)(a >> 4), db + 2 * k, (ch | kx | ky | k) ? 1u : 0u);
            }
          wgmma_commit();
#pragma unroll
          for (int i = 0; i < BY; ++i) wgmma_reg_fence(acc[i]);
          wgmma_wait<1>();               // the previous slice's products are done: its slots may be refilled
          __syncwarp();
          if (lane == 0) {
            if (rel_w >= 0) mbar_arrive(smem_u32(wempty + rel_w));
            if (rel_p >= 0) mbar_arrive(smem_u32(pempty + rel_p));
          }
          rel_w = ws;
          rel_p = (kx == 2 && ky == 2) ? ps : -1;
          if (++ws == P.n_b_slots) { ws = 0; wph ^= 1; }
        }
      if (++ps == P.n_a_slots) { ps = 0; pph ^= 1; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < BY; ++i) wgmma_reg_fence(acc[i]);
    __syncwarp();
    if (lane == 0) { mbar_arrive(smem_u32(wempty + rel_w)); mbar_arrive(smem_u32(pempty + rel_p)); }

    const int n0 = (w % n_nt) * N, pt = (w / n_nt) % n_pt, b = w / (n_nt * n_pt);
    const int x0 = (pt % tiles_x) * 16, y0 = (pt / tiles_x) * (8 * BY) + cw * (BY / 2) * 8;
#pragma unroll
    for (int i = 0; i < BY; ++i)
      halo_block_epilogue<N>(P, acc[i], smem_u32(s_bias + n0), n0, b, y0 + 8 * (i >> 1) + 2 * q, x0 + 8 * (i & 1) + g, g, t, lo);
  }
}

// Fused transposed-conv form (form 4): all four sub-pixel phases of one Conv2DTranspose (k3 or k4, stride 2) in a single
// persistent, warp-specialized launch.  The phase launches of form 0 each run a short K (1-4 weight slices per 64-channel
// chunk) over 128-pixel tiles and end in their own half-empty wave; here a work item is (phase, 16x16 input tile, N tile
// of at most 128 channels, frame), and both consumer warpgroups read every weight slice, so one L2 read of a slice feeds
// 256 pixels.  The phases keep their own filter columns and taps (the TcGroup lists of the four phase launches):
//   warpgroup 0 (registers cut to 56): lane 0 of warp 0 loads, per (item, chunk, filter column), one [64 ch, 16 px, 17 rows]
//     SW128 box by TMA -- exactly form 0's box with 8 more rows; the taps are whole-row start offsets inside it and TMA's
//     zero fill is the padding -- into a ring of box slots; lane 0 of warp 1 streams the [N x 64] weight slices in
//     (item, chunk, filter column, tap) order into a ring of weight slots, without waiting on the grid dependency.
//   warpgroups 1, 2 (registers raised to 224): warpgroup cw multiplies tile rows [8 cw, 8 cw + 8) as two m64 blocks of
//     4 x 16 pixels, one wgmma group per weight slice; slots are released as in k_conv_wg.  Then a register epilogue
//     (frag_rows_f16 / frag_rows_store): a thread's two fragment rows are input pixels (y, x) and (y, x + 8), stored to
//     output pixels (2 y + a, 2 x + b) and (2 y + a, 2 x + 16 + b) of phase (a, b).
// Items are dealt in rounds of gridDim.x, alternately forward and backward; the list is cut into blocks of gridDim.x
// (N tile, input tile, frame) units x 4 phases, phase-major with the heaviest phase first, so that the rounds even out
// the phases' unequal costs and the four phases of one input tile read its boxes while they are still in L2.
// Within each phase an output element gets form 0's products in form 0's order ((chunk, filter column, tap, k-step) on the
// same operand values) and tc_epilogue_cols_fast's arithmetic, so the outputs are bit-identical to forms 0 and 1.
constexpr int kTconvBoxRows = 17;                              // 16 input rows + the one-row halo of a dy0 = -1 phase
constexpr int kTconvBox = kTconvBoxRows * 16 * 128;            // one [64 ch, 16 px, 17 rows] box: 34 KB, 1024-aligned
struct TcPhases {                                              // the four phase launches' tap lists, (a, b) = (p / 2, p % 2)
  int n_groups[4], dy0[4], oy_add[4], ox_add[4];
  TcGroup groups[4][2];
};

// the item of round r of this CTA
__device__ __forceinline__ int tconv_item(int r) {
  const int G = gridDim.x;
  return r * G + ((r & 1) ? G - 1 - (int)blockIdx.x : (int)blockIdx.x);
}

// item w -> (phase, unit); units are (N tile fastest, input tile, frame)
__device__ __forceinline__ int2 tconv_decode(int w, int n_units) {
  const int G = gridDim.x, blk = w / (4 * G), r = w - blk * 4 * G, s = min(G, n_units - blk * G);
  return make_int2(r / s, blk * G + r % s);
}

template <int N>
__global__ void __launch_bounds__(kWideThreads, 1) k_tconv_wg_hw(const __grid_constant__ CUtensorMap mapA,
                                                                 const __grid_constant__ CUtensorMap mapB,
                                                                 const __grid_constant__ TcParams P,
                                                                 const __grid_constant__ TcPhases Q) {
  constexpr int WSLOT = N * 128;                               // one [N x 64-channel] weight slice
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* wring = base;                                       // n_b_slots weight slices (1024-aligned: SW128 atoms)
  uint8_t* aring = wring + (size_t)P.n_b_slots * WSLOT;        // n_a_slots activation boxes
  uint64_t* afull = reinterpret_cast<uint64_t*>(aring + (size_t)P.n_a_slots * kTconvBox);
  uint64_t* aempty = afull + P.n_a_slots;
  uint64_t* wfull = aempty + P.n_a_slots;
  uint64_t* wempty = wfull + P.n_b_slots;
  float* s_bias = reinterpret_cast<float*>(wempty + P.n_b_slots);   // [Cout]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_x = (P.W + 15) / 16, n_pt = tiles_x * ((P.H + 15) / 16);
  const int n_nt = P.Cout / N, n_units = n_nt * n_pt * P.batch, n_work = 4 * n_units;
  for (int i = threadIdx.x; i < P.Cout; i += blockDim.x) s_bias[i] = P.bias ? P.bias[i] : 0.f;
  if (threadIdx.x == 0) {
    // full: one TMA transaction; empty: one arrival per consumer warp
    for (int i = 0; i < P.n_a_slots; ++i) { mbar_init(smem_u32(afull + i), 1); mbar_init(smem_u32(aempty + i), 8); }
    for (int i = 0; i < P.n_b_slots; ++i) { mbar_init(smem_u32(wfull + i), 1); mbar_init(smem_u32(wempty + i), 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&mapB) : "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------ producer warpgroup ------------------------------
    setmaxnreg_dec<56>();
    if (warp == 0 && lane == 0) {
      griddep_wait();                                          // activations come from the previous kernel of the stream
      int s = 0;
      uint32_t ph = 0;
      for (int r = 0, w = tconv_item(0); w < n_work; w = tconv_item(++r)) {
        if (tconv_item(r + 1) >= n_work) griddep_launch();     // last item of this CTA
        const int2 it = tconv_decode(w, n_units);
        const int pt = (it.y / n_nt) % n_pt, b = it.y / (n_nt * n_pt);
        const int x0 = (pt % tiles_x) * 16, y0 = (pt / tiles_x) * 16 + Q.dy0[it.x];
        for (int ch = 0; ch < P.n_chunks; ++ch)
          for (int g = 0; g < Q.n_groups[it.x]; ++g) {
            mbar_wait(smem_u32(aempty + s), ph ^ 1);
            mbar_expect_tx(smem_u32(afull + s), (uint32_t)kTconvBox);
            tma_load_4d(smem_u32(aring + (size_t)s * kTconvBox), &mapA, smem_u32(afull + s), ch * 64, x0 + Q.groups[it.x][g].dx, y0, b);
            if (++s == P.n_a_slots) { s = 0; ph ^= 1; }
          }
      }
    } else if (warp == 1 && lane == 0) {
      // weights are static: no grid-dependency wait
      int s = 0;
      uint32_t ph = 0;
      for (int r = 0, w = tconv_item(0); w < n_work; w = tconv_item(++r)) {
        const int2 it = tconv_decode(w, n_units);
        const int n0 = (it.y % n_nt) * N;
        for (int ch = 0; ch < P.n_chunks; ++ch)
          for (int g = 0; g < Q.n_groups[it.x]; ++g)
            for (int t = 0; t < Q.groups[it.x][g].n_taps; ++t) {
              mbar_wait(smem_u32(wempty + s), ph ^ 1);
              mbar_expect_tx(smem_u32(wfull + s), (uint32_t)WSLOT);
              tma_load_3d(smem_u32(wring + (size_t)s * WSLOT), &mapB, smem_u32(wfull + s), ch * 64, n0, Q.groups[it.x][g].taps[t].w_tap);
              if (++s == P.n_b_slots) { s = 0; ph ^= 1; }
            }
      }
    }
    return;
  }

  // ------------------------------ consumers: warpgroup cw multiplies tile rows [8 cw, 8 cw + 8) ------------------------------
  setmaxnreg_inc<224>();
  const int cw = (warp >> 2) - 1, q = warp & 3, g = lane >> 2, t = lane & 3;
  const float lo = P.relu ? 0.f : -INFINITY;
  const uint64_t desc = make_desc(0, 128, 1);
  const uint32_t a_row0 = smem_u32(aring) + (uint32_t)(cw * 8 * 16 * 128), w_base = smem_u32(wring);
  constexpr uint32_t kBlockStep = (4 * 16 * 128) >> 4;         // descriptor start-address step of one m64 block (4 rows)
  float acc[2][N / 2];
  int sa = 0, sb = 0;
  uint32_t pha = 0, phb = 0;
  for (int r = 0, w = tconv_item(0); w < n_work; w = tconv_item(++r)) {
    const int2 it = tconv_decode(w, n_units);
    const int ph = it.x;
    int rel_a = -1, rel_b = -1;
    uint32_t scale_d = 0;
    for (int ch = 0; ch < P.n_chunks; ++ch) {
      for (int gi = 0; gi < Q.n_groups[ph]; ++gi) {
        mbar_wait(smem_u32(afull + sa), pha);
        const uint32_t a_base = a_row0 + (uint32_t)(sa * kTconvBox);
        const int n_taps = Q.groups[ph][gi].n_taps;
        for (int tt = 0; tt < n_taps; ++tt) {
          mbar_wait(smem_u32(wfull + sb), phb);
          const uint64_t da = desc + (uint64_t)((a_base + (uint32_t)(Q.groups[ph][gi].taps[tt].row_off * 16 * 128)) >> 4);
          const uint64_t db = desc + (uint64_t)((w_base + (uint32_t)(sb * WSLOT)) >> 4);
          wgmma_fence();
          wgmma_reg_fence(acc[0]);
          wgmma_reg_fence(acc[1]);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
#pragma unroll
            for (int i = 0; i < 2; ++i) wgmma_f16<N>(acc[i], da + i * kBlockStep + 2 * k, db + 2 * k, scale_d);
            scale_d = 1;
          }
          wgmma_commit();
          wgmma_reg_fence(acc[0]);
          wgmma_reg_fence(acc[1]);
          wgmma_wait<1>();               // the previous slice's products are done: its slots may be refilled
          __syncwarp();
          if (lane == 0) {
            if (rel_b >= 0) mbar_arrive(smem_u32(wempty + rel_b));
            if (rel_a >= 0) mbar_arrive(smem_u32(aempty + rel_a));
          }
          rel_b = sb;
          rel_a = tt == n_taps - 1 ? sa : -1;
          if (++sb == P.n_b_slots) { sb = 0; phb ^= 1; }
        }
        if (++sa == P.n_a_slots) { sa = 0; pha ^= 1; }
      }
    }
    wgmma_wait<0>();
    wgmma_reg_fence(acc[0]);
    wgmma_reg_fence(acc[1]);
    __syncwarp();
    if (lane == 0) { mbar_arrive(smem_u32(wempty + rel_b)); mbar_arrive(smem_u32(aempty + rel_a)); }

    const int n0 = (it.y % n_nt) * N, pt = (it.y / n_nt) % n_pt, b = it.y / (n_nt * n_pt);
    const int x = (pt % tiles_x) * 16 + g;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int y = (pt / tiles_x) * 16 + 8 * cw + 4 * i + q;
      uint32_t hv[N / 4];
      frag_rows_f16<N>(acc[i], smem_u32(s_bias + n0), t, lo, hv);
      __half* po = reinterpret_cast<__half*>(P.out) +
                   (((size_t)b * P.out_H + y * P.oy_mul + Q.oy_add[ph]) * P.out_W + x * P.ox_mul + Q.ox_add[ph]) * P.out_Ctot + P.out_coff + n0;
      frag_rows_store<N>(hv, po, (size_t)8 * P.ox_mul * P.out_Ctot, y < P.H && x < P.W, y < P.H && x + 8 < P.W, t);
    }
  }
}

// ------------------------------- host side ---------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}


// ------------------------------------------------------------------------------------------------
// 1x1 linear head (heads.py:55-63: Conv2D(channels, 1, activation="linear"), fp32 output): C_in x C_out per pixel is a few
// hundred MACs against C_in * 2 + C_out * 4 bytes of traffic, i.e. an HBM-bound layer: the implicit-GEMM conv kernel would
// write 13 (24) strided 4-byte stores per pixel.  Here: warp-level mma.sync m16n8k16 (fp16 x fp16 -> fp32; the layer is not
// tensor bound, what matters is that the MACs cost no issue slots), 16 pixels x C_in channels per warp staged with
// 16-byte-per-lane loads (whole 128-byte lines per warp instruction) and read back with ldmatrix, weights [N_pad][C_in]
// fp16 in shared memory, and the 16 x C_out fp32 results of a warp staged through shared memory so that the global stores
// are contiguous 4-byte-per-lane runs.  64 warps per SM keep ~128 KB of loads in flight.
template <int NT, int KCH>   // n-tiles of 8 output channels (C_out <= 8 * NT); input channels staged per pass (16 / 32 / 64 / 128)
__global__ void __launch_bounds__(256) k_head_1x1(const __half* __restrict__ in, int in_Ctot, int in_coff, int Cin,
                                                  const __half* __restrict__ w /*[Cout_pad][Cin]*/, const float* __restrict__ bias,
                                                  float* __restrict__ out, int out_Ctot, int out_coff, int Cout, int relu,
                                                  size_t npix, int n_ring) {
  extern __shared__ __align__(16) uint8_t hsm[];
  const int wpitch = Cin + 8;                              // halves per weight row (+16 B: conflict-free fragment loads)
  constexpr int apitch = KCH + 8;                          // halves per staged pixel row
  __half* s_w = reinterpret_cast<__half*>(hsm);            // [8 * NT][wpitch]
  __half* s_a = s_w + (size_t)8 * NT * wpitch;             // [8 warps][n_ring][16][apitch]
  float* s_out = reinterpret_cast<float*>(s_a + (size_t)8 * n_ring * 16 * apitch);     // [8 warps][16][8 * NT + 1]
  float* s_bias = s_out + 8 * 16 * (8 * NT + 1);
  for (int t = threadIdx.x; t < 8 * NT * (Cin / 8); t += 256) {
    const int r = t / (Cin / 8), c8 = t % (Cin / 8);
    *reinterpret_cast<uint4*>(s_w + (size_t)r * wpitch + 8 * c8) = *reinterpret_cast<const uint4*>(w + (size_t)r * Cin + 8 * c8);
  }
  for (int t = threadIdx.x; t < 8 * NT; t += 256) s_bias[t] = (t < Cout && bias) ? bias[t] : 0.f;
  __syncthreads();
  griddep_wait();                      // weights / bias above are static; the feature map comes from the previous kernel
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, tq = lane & 3;
  float* so = s_out + warp * 16 * (8 * NT + 1);
  __half* ring = s_a + (size_t)warp * n_ring * 16 * apitch;
  constexpr int c8n = KCH / 8;                             // 16-byte pieces per staged row
  constexpr int c8sh = KCH == 128 ? 4 : (KCH == 64 ? 3 : (KCH == 32 ? 2 : 1));
  constexpr int LI = c8n / 2;                              // 16-byte copies per lane and item
  const size_t n_tiles = (npix + 15) / 16;
  const int n_pass = Cin / KCH;
  // This warp's work items, in order: (tile, pass) with tile = first + j * stride.  Each item is 16 pixels x KCH channels
  // copied global -> shared with cp.async (16 bytes per lane and copy: a warp-wide copy covers whole 128-byte lines), one
  // commit group per item, n_ring - 1 items in flight while one is consumed: the copies never pass through registers, so
  // the bytes in flight per SM are bounded by shared memory, not by the register file (the previous cut staged through
  // registers: 2 KB per warp in flight, 2.2 TB/s at ~3 us of loaded DRAM latency).
  const size_t first = (size_t)blockIdx.x * 8 + warp, stride = (size_t)gridDim.x * 8;
  const size_t my_tiles = first < n_tiles ? (n_tiles - 1 - first) / stride + 1 : 0;
  const size_t n_items = my_tiles * (size_t)n_pass;
  auto issue = [&](size_t item) {
    if (item < n_items) {
      const size_t tile = first + (item / n_pass) * stride;
      const int k0 = (int)(item % n_pass) * KCH;
      const int rows = (int)min((size_t)16, npix - tile * 16);
      const __half* src = in + tile * 16 * in_Ctot + in_coff + k0;
      const uint32_t dst0 = smem_u32(ring + (size_t)(item % n_ring) * 16 * apitch);
#pragma unroll
      for (int i = 0; i < LI; ++i) {
        const int t = lane + 32 * i, r = t >> c8sh, c8 = t & (c8n - 1);
        const int rs = r < rows ? r : rows - 1;              // rows past the last pixel re-read it (never stored)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst0 + (uint32_t)(r * apitch + 8 * c8) * 2u),
                     "l"(src + (size_t)rs * in_Ctot + 8 * c8) : "memory");
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");     // one group per slot of the schedule, empty past the end
  };
  for (int j = 0; j < n_ring - 1; ++j) issue((size_t)j);
  float acc[NT][4];
  // a head that owns its buffer (out_Ctot == Cout) stores a tile as ONE run of 16 * Cout floats: lane l writes elements
  // l, l + 32, ... of the run; their (row, channel) positions in the staging tile are the same for every tile
  constexpr int NST = (16 * 8 * NT + 31) / 32;
  int st_off[NST];
#pragma unroll
  for (int k = 0; k < NST; ++k) {
    const int e = lane + 32 * k;
    st_off[k] = (e / Cout) * (8 * NT + 1) + e % Cout;
  }
  const bool linear = out_Ctot == Cout;
  for (size_t item = 0; item < n_items; ++item) {
    issue(item + (size_t)(n_ring - 1));
    // groups complete in order: all but the newest n_ring - 1 are done -> item `item` has landed
    switch (n_ring) {
      case 2: asm volatile("cp.async.wait_group 1;" ::: "memory"); break;
      case 3: asm volatile("cp.async.wait_group 2;" ::: "memory"); break;
      case 4: asm volatile("cp.async.wait_group 3;" ::: "memory"); break;
      case 5: asm volatile("cp.async.wait_group 4;" ::: "memory"); break;
      case 6: asm volatile("cp.async.wait_group 5;" ::: "memory"); break;
      case 7: asm volatile("cp.async.wait_group 6;" ::: "memory"); break;
      default: asm volatile("cp.async.wait_group 7;" ::: "memory"); break;
    }
    __syncwarp();
    const int pass = (int)(item % n_pass), k0 = pass * KCH;
    const size_t tile = first + (item / n_pass) * stride;
    if (pass == 0) {
#pragma unroll
      for (int n = 0; n < NT; ++n) { acc[n][0] = acc[n][1] = acc[n][2] = acc[n][3] = 0.f; }
    }
    const uint32_t sa_ld = smem_u32(ring + (size_t)(item % n_ring) * 16 * apitch + (size_t)(lane & 15) * apitch + (lane >> 4) * 8);
#pragma unroll
    for (int k = 0; k < KCH; k += 16) {
      uint32_t ra0, ra1, ra2, ra3;
      asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
                   : "=r"(ra0), "=r"(ra1), "=r"(ra2), "=r"(ra3) : "r"(sa_ld + 2u * (uint32_t)k));
#pragma unroll
      for (int n = 0; n < NT; ++n) {
        const __half* wb = s_w + (size_t)(8 * n + g) * wpitch + k0 + k + 2 * tq;
        const uint32_t rb0 = *reinterpret_cast<const uint32_t*>(wb), rb1 = *reinterpret_cast<const uint32_t*>(wb + 8);
        asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
                     : "+f"(acc[n][0]), "+f"(acc[n][1]), "+f"(acc[n][2]), "+f"(acc[n][3])
                     : "r"(ra0), "r"(ra1), "r"(ra2), "r"(ra3), "r"(rb0), "r"(rb1));
      }
    }
    __syncwarp();                                          // the slot may be refilled by the next issue()
    if (pass != n_pass - 1) continue;
    const int rows = (int)min((size_t)16, npix - tile * 16);
#pragma unroll
    for (int n = 0; n < NT; ++n) {
      const int c = 8 * n + 2 * tq;
      float v0 = acc[n][0] + s_bias[c], v1 = acc[n][1] + s_bias[c + 1], v2 = acc[n][2] + s_bias[c], v3 = acc[n][3] + s_bias[c + 1];
      if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); v2 = fmaxf(v2, 0.f); v3 = fmaxf(v3, 0.f); }
      so[g * (8 * NT + 1) + c] = v0; so[g * (8 * NT + 1) + c + 1] = v1;
      so[(g + 8) * (8 * NT + 1) + c] = v2; so[(g + 8) * (8 * NT + 1) + c + 1] = v3;
    }
    __syncwarp();
    float* ob = out + tile * 16 * out_Ctot + out_coff;
    if (linear) {                                         // whole 128-byte lines per warp store
      const int n_el = rows * Cout;
#pragma unroll
      for (int k = 0; k < NST; ++k)
        if (lane + 32 * k < n_el) ob[lane + 32 * k] = so[st_off[k]];
    } else if (NT <= 2) {                                 // two pixel rows per warp store: lanes 0-15 / 16-31 hold the channels of a row
      const int rr = lane >> 4, cc = lane & 15;
      if (cc < Cout) {
#pragma unroll
        for (int r = 0; r < 16; r += 2)
          if (r + rr < rows) ob[(size_t)(r + rr) * out_Ctot + cc] = so[(r + rr) * (8 * NT + 1) + cc];
      }
    } else if (lane < Cout) {
#pragma unroll
      for (int r = 0; r < 16; ++r)
        if (r < rows) ob[(size_t)r * out_Ctot + lane] = so[r * (8 * NT + 1) + lane];
    }
    __syncwarp();
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// Kernel forms of a tensor-core conv, all bit-identical.  Forms 0-3 run one launch (a conv, or one sub-pixel phase of a
// transposed conv): 0 = k_conv_wg (streaming, one CTA per tile and N tile), 1 = the persistent k_conv_wg_p with resident
// weights, 2 = the persistent halo-patch k_conv_wg_h, 3 = the persistent halo-patch k_conv_wg_hw with streamed weights
// and N tiles of at most 128.  Form 4 = the persistent k_tconv_wg_hw runs all four phases of a transposed conv in one
// launch; it is kept in the first phase's TcLaunch and, when picked, stands for the whole op.  The autotuner first keeps
// the fastest eligible form 0-3 per launch, then for each transposed conv the faster of its phase launches and form 4.
// SB_FORCE_VARIANT=n with n = 0-3 forces form n on every launch where it is eligible and keeps the phase launches; n = 4
// keeps the autotuned launch forms and forces form 4 where it is eligible; any other n >= 0 keeps the autotuned launch
// forms and the phase launches.
constexpr int kForms = 5, kTconvForm = 4;
struct TcForm {
  int ok;
  int threads;                 // CTA size
  size_t smem;
  int max_ctas;                // persistent forms: CTAs the GPU holds at once
  int n_items;                 // persistent forms: work items per frame
  TcParams P;                  // the launch's parameters with this form's ring sizes and N
  // forms 2 and 3: a halo-patch box (encode_patches); form 3: a [64, N, 1] weight box; form 4: a [64, 16, 17, 1] activation box
  CUtensorMap mapA, mapB;
  TcPhases Q;                  // form 4: the four phases' filter columns and taps
};

struct TcLaunch {
  dim3 grid;                   // form 0: tiles x N tiles (z = batch, set at launch)
  TcForm forms[kForms];
  int form;
};

}  // namespace

struct SbConvTcPlan {
  std::vector<TcLaunch> launches;   // 1 for conv, 4 phases for tconv
  const void* head = nullptr;       // the k_head_1x1 instantiation that runs this 1x1 fp32 head instead of the launches
  __half* w16 = nullptr;            // [taps][Cout_pad][Cin]
  int Cout_pad = 0;
  bool pool_fused = false;          // the launches write the 2x2 max-pool of the POOL op after this conv
  bool out_dead = false;            // nobody reads the full-resolution output (only the fused pool): stores are skipped
  // the residual ADD after this conv runs in its epilogue (launches); plain_launches store the conv's own output
  // instead, for a forward pass that asks for that tensor (the ADD op then runs)
  bool res_fused = false;
  std::vector<TcLaunch> plain_launches;
};

static CUtensorMapSwizzle swz_for(int KC) {
  return KC == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (KC == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

static bool tc_eligible(const SbModel* m, const SbOp& op) {
  if (getenv("SB_DISABLE_TC")) return false;
  if (op.kind() != SB_OPK_CONV && op.kind() != SB_OPK_TCONV) return false;
  const int Cin = op.in_C();
  // any channel count that keeps 16-byte aligned NHWC rows: K is cut into chunks of 16 / 32 / 64 channels and a
  // chunk that reaches past C_in is zero-filled by TMA on both operands (activations and weights)
  if (!(Cin >= 16 && Cin % 8 == 0)) return false;
  if (op.kind() == SB_OPK_CONV && !((op.k() == 1 || op.k() == 3 || op.k() == 5 || op.k() == 7) && op.stride() == 1) &&
      !(op.k() == 1 && op.stride() == 2))
    return false;
  // explicit padding: only the 1x1 VALID convs of ResNet (padding 0, the same as SAME for kernel 1)
  if (op.kind() == SB_OPK_CONV && op.explicit_pad() && (op.k() != 1 || op.pad_top() != 0 || op.pad_left() != 0)) return false;
  if (op.kind() == SB_OPK_TCONV && op.k() != 3 && op.k() != 4) return false;
  const SbBuffer& ib = m->buffers[op.in_buf()];
  const SbBuffer& ob = m->buffers[op.out_buf()];
  if (ib.f32) return false;
  // feature maps smaller than the TMA box (16 px x 8 + k - 1 rows) are taken too: the box simply hangs over the tensor,
  // the overhang is zero-filled like every other out-of-image tap
  if (ib.C % 8 || op.in_coff() % 8) return false;
  if (!ob.f32 && (ob.C % 8 || op.out_coff() % 8)) return false;
  return true;
}

void sb_conv_tc_drop(SbModel* m, int op_index) {
  SbConvTcPlan*& p = m->tc_plans[op_index];
  if (p->w16) cudaFree(p->w16);
  delete p;
  p = nullptr;
}

void sb_conv_tc_release(SbModel* m) {
  for (size_t oi = 0; oi < m->tc_plans.size(); ++oi)
    if (m->tc_plans[oi]) sb_conv_tc_drop(m, (int)oi);
  m->tc_plans.clear();
}

// the wgmma tile widths N that have instantiations
constexpr int kWgN[8] = {16, 32, 48, 64, 96, 128, 192, 256};

// N of the wgmma instantiation that covers `n` output channels (extra rows of the weight box are zero-filled by TMA)
static int wg_n(int n) {
  for (int c : kWgN) if (n <= c) return c;
  return 256;
}

// Instantiations of each form for K steps of 16 per staged slice of KS x 16 channels, by N (kWgN).  Resident: N <= 128
// (a 192 / 256-wide bank does not fit beside the activation ring at C_in >= 64, and N = 256 leaves no registers for the
// persistent loop state).  Halo: N <= 64.  Wide and fused tconv: chunks of 64 channels only, N of 32..128.
template <int KS>
static const void* form_kernel_ks(int form, int ni) {
  static const void* const kernels[kForms][8] = {
      {(const void*)k_conv_wg<KS, 16>, (const void*)k_conv_wg<KS, 32>, (const void*)k_conv_wg<KS, 48>,
       (const void*)k_conv_wg<KS, 64>, (const void*)k_conv_wg<KS, 96>, (const void*)k_conv_wg<KS, 128>,
       (const void*)k_conv_wg<KS, 192>, (const void*)k_conv_wg<KS, 256>},
      {(const void*)k_conv_wg_p<KS, 16>, (const void*)k_conv_wg_p<KS, 32>, (const void*)k_conv_wg_p<KS, 48>,
       (const void*)k_conv_wg_p<KS, 64>, (const void*)k_conv_wg_p<KS, 96>, (const void*)k_conv_wg_p<KS, 128>, nullptr, nullptr},
      {(const void*)k_conv_wg_h<KS, 16>, (const void*)k_conv_wg_h<KS, 32>, (const void*)k_conv_wg_h<KS, 48>,
       (const void*)k_conv_wg_h<KS, 64>, nullptr, nullptr, nullptr, nullptr},
      {nullptr, (const void*)k_conv_wg_hw<32>, (const void*)k_conv_wg_hw<48>, (const void*)k_conv_wg_hw<64>,
       (const void*)k_conv_wg_hw<96>, (const void*)k_conv_wg_hw<128>, nullptr, nullptr},
      {nullptr, (const void*)k_tconv_wg_hw<32>, (const void*)k_tconv_wg_hw<48>, (const void*)k_tconv_wg_hw<64>,
       (const void*)k_tconv_wg_hw<96>, (const void*)k_tconv_wg_hw<128>, nullptr, nullptr}};
  return form >= 3 && KS != 4 ? nullptr : kernels[form][ni];
}

// The kernel of `form` for input-channel chunks of KC and a wg_n() tile width N, or nullptr where the form has none.
// Forms 0-3 take (mapA, mapB, TcParams), form 4 (mapA, mapB, TcParams, TcPhases).
static const void* form_kernel(int form, int KC, int N) {
  const int ni = (int)(std::find(std::begin(kWgN), std::end(kWgN), N) - std::begin(kWgN));
  if (ni == 8) return nullptr;
  return KC == 16 ? form_kernel_ks<1>(form, ni) : (KC == 32 ? form_kernel_ks<2>(form, ni) : form_kernel_ks<4>(form, ni));
}

// shared memory of a k_conv_wg launch: rings, accumulator staging rows, barriers, bias / BN vectors of 256 channels
static size_t conv_smem(const TcParams& P, int n_a, int n_b) {
  return (size_t)n_a * P.a_slot_bytes + (size_t)n_b * P.b_slot_bytes + (size_t)128 * (stage_cols(P.N) + 4) * sizeof(float) +
         1024 /*align slack*/ + (size_t)(2 * n_a + 2 * n_b) * 8 + 16 + 3 * 256 * sizeof(float);
}

// shared memory of a k_conv_wg_p launch: activation ring, weight bank, staging rows, 2 n_a + 1 barriers, bias / BN vectors
static size_t conv_smem_resident(const TcParams& P, int n_a, int bank) {
  return (size_t)n_a * P.a_slot_bytes + (size_t)bank * P.b_slot_bytes + (size_t)128 * (stage_cols(P.N) + 4) * sizeof(float) +
         1024 /*align slack*/ + (size_t)(2 * n_a + 1) * 8 + 16 + 3 * (size_t)P.N * sizeof(float);
}

// shared memory of a k_conv_wg_h launch: weight bank (9 slices), n_a patch slots, 2 n_a + 1 barriers
static size_t conv_smem_halo(const TcParams& P, int n_a) {
  return 1024 /*align slack*/ + (size_t)9 * P.b_slot_bytes + (size_t)n_a * patch_slot_bytes(8 * halo_by(P.N, P.KC) + 2, P.KC) +
         (size_t)(2 * n_a + 1) * 8 +
         (size_t)P.N * sizeof(float);
}

// Rings of a k_conv_wg_hw / k_tconv_wg_hw launch (forms 3 and 4, N tiles of F.P.N): n_a activation slots of a_slot bytes
// and the deepest ring of 8 down to 4 weight slices that fits in 225 KB beside them, 2 (n_a + n_b) barriers and the bias.
// Sets F.ok where one fits.
static void fit_weight_ring(TcForm& F, int n_a, size_t a_slot) {
  for (int nb = 8; nb >= 4 && !F.ok; --nb) {
    const size_t smem = 1024 /*align slack*/ + (size_t)nb * F.P.N * 128 + (size_t)n_a * a_slot + (size_t)(2 * n_a + 2 * nb) * 8 +
                        (size_t)F.P.Cout * sizeof(float);
    if (smem <= kMaxDynSmem) { F.ok = 1; F.P.n_a_slots = n_a; F.P.n_b_slots = nb; F.smem = smem; }
  }
}

// Co-resident CTAs of persistent form f where it fits (F.ok); clears F.ok where not even one CTA per SM does.
static void fit_ctas(sb_handle_s* h, TcForm& F, int f) {
  if (!F.ok) return;
  int nb = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, form_kernel(f, F.P.KC, F.P.N), F.threads, F.smem) != cudaSuccess || nb < 1) {
    cudaGetLastError();
    F.ok = 0;
    return;
  }
  F.max_ctas = nb * h->sm_count;
}

// The halo forms take plain 3x3 stride-1 SAME convs (filter column g = dx + 1, tap ky of it = weight tap 3 ky + g) in the
// fast-epilogue output shape without a residual.
static bool halo_shape(const TcParams& P) {
  if (P.epi_mode != 1 || P.res != nullptr || P.n_groups != 3 || P.dy0 != -1 || P.box_rows != TH + 2 || P.oy_mul != 1 ||
      P.oy_add != 0 || P.ox_mul != 1 || P.ox_add != 0)
    return false;
  for (int g = 0; g < 3; ++g) {
    if (P.groups[g].dx != g - 1 || P.groups[g].n_taps != 3) return false;
    for (int ky = 0; ky < 3; ++ky)
      if (P.groups[g].taps[ky].row_off != ky || P.groups[g].taps[ky].w_tap != 3 * ky + g) return false;
  }
  return true;
}

// form 2: one input-channel chunk and one N tile of at most 64 channels
static bool halo_eligible(const TcLaunch& L) {
  const TcParams& P = L.forms[0].P;
  return L.grid.y == 1 && P.n_chunks == 1 && P.N <= 64 && halo_shape(P);
}

// form 3: chunks of 64 input channels, and N tiles of min(N, 128) channels that cover C_out exactly
static int wide_n(const TcParams& P) { return std::min(P.N, 128); }
static bool wide_eligible(const TcParams& P) { return P.KC == 64 && P.Cout % wide_n(P) == 0 && halo_shape(P); }

// Forms 1-4 of launch L as copies of its streaming form 0 (always eligible), and the eligibility, ring sizes, shared
// memory and co-resident grid size of forms 1-3 (form 4 is set up per op: setup_tconv_form).  Resident form: one N tile,
// and the whole bank of the launch's weight slices plus at least 2 activation slots fit in 225 KB; two CTAs per SM where
// they fit in 113 KB.  Halo form: halo_eligible, and the bank plus at least 4 patch slots (two being read, two
// prefetched) fit in 225 KB; up to 8 slots, one CTA per SM.  Wide form: wide_eligible, 2 patch slots and 4-8 weight
// slots in 225 KB, one CTA per SM.
static void setup_forms(sb_handle_s* h, TcLaunch& L, int total_steps) {
  const TcParams& P = L.forms[0].P;
  L.form = 0;
  for (int f = 1; f < kForms; ++f) {
    L.forms[f] = L.forms[0];
    L.forms[f].ok = 0;
  }
  if (TcForm& F = L.forms[3]; form_kernel(3, P.KC, wide_n(P)) && wide_eligible(P)) {
    F.threads = kWideThreads;
    F.P.N = wide_n(P);
    fit_weight_ring(F, 2, (size_t)patch_slot_bytes(wide_rows(F.P.N), 64));
    const int by = wide_by(F.P.N);
    F.n_items = (P.Cout / F.P.N) * ((P.W + 15) / 16) * ((P.H + 8 * by - 1) / (8 * by));
    fit_ctas(h, F, 3);
  }
  if (TcForm& F = L.forms[2]; form_kernel(2, P.KC, P.N) && halo_eligible(L)) {
    F.threads = kConvThreads;
    for (int na = 8; na >= 4 && !F.ok; --na)
      if (conv_smem_halo(P, na) <= kMaxDynSmem) { F.ok = 1; F.P.n_a_slots = na; F.P.n_b_slots = 9; F.smem = conv_smem_halo(P, na); }
    const int by = halo_by(P.N, P.KC);
    F.n_items = ((P.W + 15) / 16) * ((P.H + 8 * by - 1) / (8 * by));
    fit_ctas(h, F, 2);
  }
  TcForm& F = L.forms[1];
  if (!form_kernel(1, P.KC, P.N) || L.grid.y != 1) return;
  const int bank = P.n_chunks * total_steps;
  for (size_t budget : {(size_t)113 * 1024, kMaxDynSmem}) {
    for (int na = 4; na >= 2 && !F.ok; --na)
      if (conv_smem_resident(P, na, bank) <= budget) { F.ok = 1; F.P.n_a_slots = na; F.P.n_b_slots = bank; F.smem = conv_smem_resident(P, na, bank); }
    if (F.ok) break;
  }
  F.n_items = P.n_tiles;
  fit_ctas(h, F, 1);
}

// The residual ADD right after conv `oi` can run in its epilogue: the conv's output has no other reader (the compiler
// only sets SB_OPF_RESIDUAL then), the ADD is flagged, and the shortcut / sum slices are 16-byte aligned fp16.
static bool res_fusable(const SbModel* m, size_t oi) {
  const SbOp& op = m->ops[oi];
  if (op.kind() != SB_OPK_CONV || !op.residual() || oi + 1 >= m->ops.size() || getenv("SB_DISABLE_RES_FUSION")) return false;
  const SbOp& add = m->ops[oi + 1];
  if (add.kind() != SB_OPK_ADD || !(add.flags() & SB_OPF_FUSED_ADD) || add.out_buf() != op.sum_buf() || add.out_coff() != op.sum_coff()) return false;
  const SbBuffer& rb = m->buffers[op.res_buf()];
  const SbBuffer& sb = m->buffers[op.sum_buf()];
  const SbBuffer& ob = m->buffers[op.out_buf()];
  return !rb.f32 && !sb.f32 && !ob.f32 && rb.C % 8 == 0 && op.res_coff() % 8 == 0 && sb.C % 8 == 0 && op.sum_coff() % 8 == 0 &&
         rb.H == ob.H && rb.W == ob.W && sb.H == ob.H && sb.W == ob.W && op.pool_buf() < 0 && !(op.flags() & (SB_OPF_BN | SB_OPF_RELU));
}

// [tap][Cout_pad][Cin] weights of a plan, box [KC, box_n, 1]
static CUresult encode_weights(EncodeTiledFn enc, const SbConvTcPlan* plan, int Cin, int n_wtaps, int KC, int box_n, CUtensorMap* map) {
  cuuint64_t dims[3] = {(cuuint64_t)Cin, (cuuint64_t)plan->Cout_pad, (cuuint64_t)n_wtaps};
  cuuint64_t strides[2] = {(cuuint64_t)Cin * 2, (cuuint64_t)plan->Cout_pad * Cin * 2};
  cuuint32_t box[3] = {(cuuint32_t)KC, (cuuint32_t)box_n, 1};
  cuuint32_t es[3] = {1, 1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, (void*)plan->w16, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
             swz_for(KC), CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

// Forms 2 and 3: the input slice as a 4-D map {C_in, W, H, frames}, byte strides {C_tot 2, W C_tot 2, H W C_tot 2},
// whose box {KC, 18, rows, 1} at (c0, x - 1, y - 1, b) is one halo patch: it lands as the swizzled pixel rows
// [rows][18][KC ch] of a patch slot.  Pixels outside the image (SAME padding) and channels beyond C_in (the chunk's zero
// fill) are out of bounds of the map and zero-filled by TMA.
static CUresult encode_patches(EncodeTiledFn enc, const TcParams& P, int frames, int rows, CUtensorMap* map) {
  cuuint64_t dims[4] = {(cuuint64_t)P.in_C, (cuuint64_t)P.W, (cuuint64_t)P.H, (cuuint64_t)frames};
  cuuint64_t strides[3] = {(cuuint64_t)P.in_Ctot * 2, (cuuint64_t)P.W * P.in_Ctot * 2, (cuuint64_t)P.H * P.W * P.in_Ctot * 2};
  cuuint32_t box[4] = {(cuuint32_t)P.KC, kHaloCols, (cuuint32_t)rows, 1};
  cuuint32_t es[4] = {1, 1, 1, 1};
  return enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(P.in), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
             swz_for(P.KC), CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

static int make_launch(sb_handle_s* h, SbModel* m, const SbOp& op, SbConvTcPlan* plan, int n_groups,
                       const TcGroup* groups, int dy0, int extra_rows, int n_wtaps, int oy_mul, int oy_add,
                       int ox_mul, int ox_add, const SbTcView* view = nullptr, bool fuse_res = false,
                       std::vector<TcLaunch>* dst = nullptr) {
  EncodeTiledFn enc = get_encode();
  if (!enc) return sb_fail(h, SB_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  const SbBuffer& ib = view ? view->in : m->buffers[op.in_buf()];
  const SbBuffer& ob0 = view ? view->out : m->buffers[op.out_buf()];
  const SbBuffer& ob = fuse_res ? m->buffers[op.sum_buf()] : ob0;       // the residual sum goes to the ADD's output slice
  const int Cin = view ? view->in.C : op.in_C(), Cout = view ? view->Cout : op.out_C();
  const int in_coff = view ? 0 : op.in_coff(), out_coff = view ? view->out_coff : (fuse_res ? op.sum_coff() : op.out_coff());
  const int KC = Cin > 32 ? 64 : (Cin > 16 ? 32 : 16);
  // 1x1 stride-2: the GEMM runs over the output grid on a subsampled view of the input (pitches x 2)
  const int sub = (!view && op.kind() == SB_OPK_CONV) ? op.stride() : 1;
  const int gH = sub > 1 ? ob.H : ib.H, gW = sub > 1 ? ob.W : ib.W;
  TcLaunch L;
  memset(&L, 0, sizeof(L));
  TcForm& F0 = L.forms[0];
  TcParams& P = F0.P;
  P.H = gH; P.W = gW;
  P.tiles_x = (gW + TW - 1) / TW;
  const int tiles_y = (gH + TH - 1) / TH;
  P.n_chunks = (Cin + KC - 1) / KC; P.KC = KC;
  P.n_groups = n_groups;
  for (int g = 0; g < n_groups; ++g) P.groups[g] = groups[g];
  P.dy0 = dy0; P.box_rows = TH + extra_rows;
  const int N = wg_n(std::min(plan->Cout_pad, 256));
  P.N = N; P.Cout = Cout;
  P.out = ob.dev; P.out_f32 = ob.f32; P.out_H = ob.H; P.out_W = ob.W; P.out_Ctot = ob.C; P.out_coff = out_coff;
  P.oy_mul = oy_mul; P.oy_add = oy_add; P.ox_mul = ox_mul; P.ox_add = ox_add;
  if (view) {
    P.bias = view->bias; P.bn_scale = view->bn_scale; P.bn_shift = view->bn_shift; P.relu = view->relu;
  } else {
    P.bias = op.b_off() >= 0 ? m->weights_dev + op.b_off() : nullptr;
    P.bn_scale = (op.flags() & SB_OPF_BN) ? m->weights_dev + op.bn_scale_off() : nullptr;
    P.bn_shift = (op.flags() & SB_OPF_BN) ? m->weights_dev + op.bn_shift_off() : nullptr;
    P.relu = (op.flags() & SB_OPF_RELU) ? 1 : 0;
  }
  P.res = nullptr;
  if (fuse_res) {                  // + shortcut, then the ADD's ReLU
    const SbBuffer& rb = m->buffers[op.res_buf()];
    P.res = (const __half*)rb.dev; P.res_Ctot = rb.C; P.res_coff = op.res_coff();
    P.relu = (m->ops[&op - m->ops.data() + 1].flags() & SB_OPF_RELU) ? 1 : 0;
  }
  P.pool_out = nullptr;
  if (!view && op.kind() == SB_OPK_CONV && op.pool_buf() >= 0 && !ob.f32 && Cout % 16 == 0 &&
      m->buffers[op.pool_buf()].C % 8 == 0 && op.pool_coff() % 8 == 0 && ib.H % 2 == 0 && ib.W % 2 == 0) {
    const SbBuffer& pb = m->buffers[op.pool_buf()];
    P.pool_out = pb.dev; P.pool_H = pb.H; P.pool_W = pb.W; P.pool_Ctot = pb.C; P.pool_coff = op.pool_coff();
  }
  P.split = (m->precision == 2 && !ob.f32) ? 1 : 0;
  P.epi_mode = 0;
  if (!P.split && !ob.f32 && P.bn_scale == nullptr && Cout % 16 == 0 && plan->Cout_pad == Cout &&
      ob.C % 16 == 0 && out_coff % 16 == 0 && (P.pool_out == nullptr || (P.pool_Ctot % 16 == 0 && P.pool_coff % 16 == 0)))
    P.epi_mode = 1;                // (a residual slice is 16-byte aligned: res_fusable)
  P.row_bytes = KC * 2;
  P.layout_type = KC == 64 ? 1 : (KC == 32 ? 2 : 3);     // wgmma descriptor layout: SW128 / SW64 / SW32
  P.a_tx_bytes = P.box_rows * TW * KC * 2;
  P.b_tx_bytes = N * KC * 2;
  P.a_slot_bytes = (P.a_tx_bytes + 1023) / 1024 * 1024;
  P.b_slot_bytes = (P.b_tx_bytes + 1023) / 1024 * 1024;
  int total_steps = 0;
  for (int g = 0; g < n_groups; ++g) total_steps += groups[g].n_taps;
  // rings: up to 3 activation boxes and 4 weight slices in flight, within what is left of the SM's shared memory after
  // the accumulator staging rows, the barriers and the bias / BN vectors
  const size_t stage_bytes = (size_t)128 * (stage_cols(N) + 4) * sizeof(float);
  const size_t ring_budget = 200 * 1024 - stage_bytes;
  P.n_a_slots = std::min(3, P.n_chunks * n_groups);
  P.n_b_slots = std::min(4, P.n_chunks * total_steps);
  while ((size_t)P.n_a_slots * P.a_slot_bytes + (size_t)P.n_b_slots * P.b_slot_bytes > ring_budget && P.n_b_slots > 2) P.n_b_slots--;
  while ((size_t)P.n_a_slots * P.a_slot_bytes + (size_t)P.n_b_slots * P.b_slot_bytes > ring_budget && P.n_a_slots > 2) P.n_a_slots--;
  F0.ok = 1;
  F0.threads = kConvThreads;
  F0.smem = conv_smem(P, P.n_a_slots, P.n_b_slots);
  if (F0.smem > kMaxDynSmem) return sb_fail(h, SB_ERR_INVALID, "conv tile needs %zu bytes of shared memory", F0.smem);
  L.grid = dim3(P.tiles_x * tiles_y, (plan->Cout_pad + N - 1) / N, 1 /* z = batch, set at launch */);
  // A: NHWC view (slice channels, W, H, batch); pixel and row pitches x sub
  {
    cuuint64_t dims[4] = {(cuuint64_t)Cin, (cuuint64_t)gW, (cuuint64_t)gH, (cuuint64_t)m->B};
    cuuint64_t strides[3] = {(cuuint64_t)ib.C * 2 * sub, (cuuint64_t)ib.W * ib.C * 2 * sub, (cuuint64_t)ib.H * ib.W * ib.C * 2};
    cuuint32_t box[4] = {(cuuint32_t)KC, (cuuint32_t)TW, (cuuint32_t)P.box_rows, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    void* gptr = (void*)((__half*)ib.dev + in_coff);
    P.in = gptr; P.in_Ctot = ib.C; P.in_C = Cin;
    CUresult r = enc(&F0.mapA, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, gptr, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     swz_for(KC), CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return sb_fail(h, SB_ERR_CUDA, "cuTensorMapEncodeTiled(A) failed: %d", (int)r);
  }
  if (CUresult r = encode_weights(enc, plan, Cin, n_wtaps, KC, N, &F0.mapB); r != CUDA_SUCCESS)
    return sb_fail(h, SB_ERR_CUDA, "cuTensorMapEncodeTiled(B) failed: %d", (int)r);
  P.n_tiles = (int)L.grid.x;
  setup_forms(h, L, total_steps);
  if (L.forms[2].ok)
    if (CUresult r = encode_patches(enc, P, m->B, 8 * halo_by(P.N, KC) + 2, &L.forms[2].mapA); r != CUDA_SUCCESS)
      return sb_fail(h, SB_ERR_CUDA, "cuTensorMapEncodeTiled(patches, halo form) failed: %d", (int)r);
  if (L.forms[3].ok) {
    if (CUresult r = encode_patches(enc, P, m->B, wide_rows(L.forms[3].P.N), &L.forms[3].mapA); r != CUDA_SUCCESS)
      return sb_fail(h, SB_ERR_CUDA, "cuTensorMapEncodeTiled(patches, wide form) failed: %d", (int)r);
    if (CUresult r = encode_weights(enc, plan, Cin, n_wtaps, KC, L.forms[3].P.N, &L.forms[3].mapB); r != CUDA_SUCCESS)
      return sb_fail(h, SB_ERR_CUDA, "cuTensorMapEncodeTiled(B, wide form) failed: %d", (int)r);
  }
  (dst ? *dst : plan->launches).push_back(L);
  return 0;
}

// Form 4 of the transposed conv `op`, kept in the first of its four phase launches (plan->launches): chunks of 64 input
// channels, N tiles of min(N, 128) channels that cover C_out exactly, the fp16 fast-epilogue shape (so not precision 2),
// and phases whose taps all lie in one 17-row box (dy0 of -1 or 0, start rows 0 or 1: the k3 and k4 phases); 4 box
// slots and 4-8 weight slots in 225 KB, one CTA per SM.  The form stays ineligible where the op does not qualify.
static int setup_tconv_form(sb_handle_s* h, SbModel* m, const SbOp& op, SbConvTcPlan* plan) {
  if (plan->launches.size() != 4) return 0;
  TcForm& T = plan->launches[0].forms[kTconvForm];      // setup_forms: a copy of the first phase's form 0, not ok
  const TcParams& P0 = plan->launches[0].forms[0].P;
  T.threads = kWideThreads;
  T.P.N = std::min(P0.N, 128);
  if (!form_kernel(kTconvForm, P0.KC, T.P.N) || P0.Cout % T.P.N) return 0;
  for (int p = 0; p < 4; ++p) {
    const TcParams& P = plan->launches[p].forms[0].P;
    if (P.epi_mode != 1 || P.n_groups > 2 || P.dy0 < -1 || P.dy0 > 0) return 0;
    T.Q.n_groups[p] = P.n_groups; T.Q.dy0[p] = P.dy0; T.Q.oy_add[p] = P.oy_add; T.Q.ox_add[p] = P.ox_add;
    for (int g = 0; g < P.n_groups; ++g) {
      for (int t = 0; t < P.groups[g].n_taps; ++t)
        if (P.groups[g].taps[t].row_off < 0 || P.groups[g].taps[t].row_off > 1) return 0;
      T.Q.groups[p][g] = P.groups[g];
    }
  }
  fit_weight_ring(T, 4, kTconvBox);
  T.n_items = 4 * (P0.Cout / T.P.N) * ((P0.W + 15) / 16) * ((P0.H + 15) / 16);   // (phase, N tile, input tile)
  fit_ctas(h, T, kTconvForm);
  if (!T.ok) return 0;
  EncodeTiledFn enc = get_encode();
  {
    // the phase launches' activation view (slice channels, W, H, batch) with a [64, 16, 17, 1] box
    cuuint64_t dims[4] = {(cuuint64_t)P0.in_C, (cuuint64_t)P0.W, (cuuint64_t)P0.H, (cuuint64_t)m->B};
    cuuint64_t strides[3] = {(cuuint64_t)P0.in_Ctot * 2, (cuuint64_t)P0.W * P0.in_Ctot * 2, (cuuint64_t)P0.H * P0.W * P0.in_Ctot * 2};
    cuuint32_t box[4] = {64, 16, (cuuint32_t)kTconvBoxRows, 1};
    cuuint32_t es[4] = {1, 1, 1, 1};
    CUresult r = enc(&T.mapA, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(P0.in), dims, strides, box, es,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return sb_fail(h, SB_ERR_CUDA, "cuTensorMapEncodeTiled(A, fused tconv) failed: %d", (int)r);
  }
  if (CUresult r = encode_weights(enc, plan, op.in_C(), op.k() * op.k(), 64, T.P.N, &T.mapB); r != CUDA_SUCCESS)
    return sb_fail(h, SB_ERR_CUDA, "cuTensorMapEncodeTiled(B, fused tconv) failed: %d", (int)r);
  return 0;
}

int sb_conv_tc_view_prepare(sb_handle_s* h, SbModel* m, int op_index, const SbTcView& v, const std::vector<float>& w) {
  if (v.in.W < TW || v.in.H < TH + v.R - 1) return 0;         // the streaming TMA box must fit inside the view
  SbConvTcPlan* plan = new SbConvTcPlan();
  int cp = (v.Cout + 15) / 16 * 16;
  if (cp > 256) cp = (cp + 255) / 256 * 256;
  plan->Cout_pad = cp;
  std::vector<__half> w16((size_t)v.R * v.S * cp * 16, __float2half(0.f));
  for (int t = 0; t < v.R * v.S; ++t)
    for (int co = 0; co < v.Cout; ++co)
      for (int c = 0; c < 16; ++c) w16[((size_t)t * cp + co) * 16 + c] = __float2half_rn(w[((size_t)t * v.Cout + co) * 16 + c]);
  cudaError_t e = cudaMalloc((void**)&plan->w16, w16.size() * sizeof(__half));
  if (e == cudaSuccess) e = cudaMemcpy(plan->w16, w16.data(), w16.size() * sizeof(__half), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    if (plan->w16) cudaFree(plan->w16);
    delete plan;
    return sb_fail(h, SB_ERR_CUDA, "view conv weights: %s", cudaGetErrorString(e));
  }
  TcGroup g[MAX_GROUPS];                                      // filter column s, its rows r
  for (int s = 0; s < v.S; ++s) {
    g[s].dx = v.dx0 + s; g[s].n_taps = v.R;
    for (int r = 0; r < v.R; ++r) g[s].taps[r] = TcTap{r, r * v.S + s};
  }
  if (const int rc = make_launch(h, m, m->ops[op_index], plan, v.S, g, v.dy0, v.R - 1, v.R * v.S, 1, 0, 1, 0, &v)) {
    cudaFree(plan->w16);
    delete plan;
    return rc;
  }
  m->tc_plans[op_index] = plan;
  return 0;
}

// Shared memory of one k_head_1x1 launch: the weight bank, the output staging and the bias, plus a per-warp ring of n_ring
// staged items (16 pixels x kch channels each), as deep as fits with two blocks per SM, else with one block per SM
// (kHeadSmem).  n_ring = 0: not even a ring of 2 fits beside the bank (wide inputs with 17-32 outputs), so the op stays
// on the implicit-GEMM conv kernel.
constexpr long long kHeadSmem = 200 * 1024;
struct HeadShape {
  int nt, kch, n_ring;
  size_t smem;
};
static HeadShape head_shape(const SbOp& op) {
  HeadShape s;
  s.nt = (op.out_C() + 7) / 8;
  s.kch = std::min(op.in_C(), 128);
  // signed: the bank alone can exceed the two-blocks-per-SM budget
  const long long fixed = 8LL * s.nt * (op.in_C() + 8) * 2 + 8LL * 16 * (8 * s.nt + 1) * 4 + 8LL * s.nt * 4;
  const long long stage = 8LL * 16 * (s.kch + 8) * 2;
  long long n_ring = std::min<long long>(8, (110 * 1024 - fixed) / stage);
  if (n_ring < 4) n_ring = std::min<long long>(8, (kHeadSmem - fixed) / stage);
  s.n_ring = n_ring >= 2 ? (int)n_ring : 0;
  s.smem = (size_t)(fixed + s.n_ring * stage);
  return s;
}

// 1x1 fp32 heads on k_head_1x1 (HBM-bound; see the kernel) instead of the implicit-GEMM conv kernel
static bool head_kernel_ok(const SbModel* m, const SbOp& op, const SbConvTcPlan* plan) {
  const SbBuffer& ib = m->buffers[op.in_buf()];
  const SbBuffer& ob = m->buffers[op.out_buf()];
  return op.kind() == SB_OPK_CONV && op.k() == 1 && op.stride() == 1 && ob.f32 && !ib.f32 && !(op.flags() & SB_OPF_BN) && op.in_C() % 16 == 0 &&
         (op.in_C() == 16 || op.in_C() == 32 || op.in_C() == 64 || op.in_C() % 128 == 0) && op.out_C() <= 32 && ib.C % 8 == 0 && op.in_coff() % 8 == 0 && plan->w16 != nullptr && plan->Cout_pad >= (op.out_C() + 7) / 8 * 8 &&
         (size_t)plan->Cout_pad * (op.in_C() + 8) * 2 <= 160 * 1024 && head_shape(op).n_ring >= 2;
}

// the k_head_1x1 instantiation for NT x 8 output channels (NT <= 4: head_kernel_ok) and staged chunks of KCH channels
static const void* head_kernel(int nt, int kch) {
#define SB_HEAD_CASE(NT)                                                                                                 \
  case NT:                                                                                                               \
    return kch == 16 ? (const void*)k_head_1x1<NT, 16> : kch == 32 ? (const void*)k_head_1x1<NT, 32>                     \
         : kch == 64 ? (const void*)k_head_1x1<NT, 64> : (const void*)k_head_1x1<NT, 128>;
  switch (nt) {
    SB_HEAD_CASE(1) SB_HEAD_CASE(2) SB_HEAD_CASE(3) SB_HEAD_CASE(4)
    default: return nullptr;
  }
#undef SB_HEAD_CASE
}

int sb_conv_tc_prepare(sb_handle_s* h, SbModel* m) {
  m->tc_plans.assign(m->ops.size(), nullptr);
  if (m->precision == 1) return 0;
  const bool split = m->precision == 2;          // physical extent of a conv's output slice: 3 x C_out fp16 planes
  static bool attr_set = false;
  if (!attr_set) {
    for (int f = 0; f < kForms; ++f)
      for (int kc : {16, 32, 64})
        for (int n : kWgN)
          if (const void* k = form_kernel(f, kc, n))
            SB_CUDA(h, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxDynSmem));
    attr_set = true;
  }
  for (size_t oi = 0; oi < m->ops.size(); ++oi) {
    const SbOp& op = m->ops[oi];
    if (!tc_eligible(m, op)) continue;
    const int Cin = op.in_C(), Cout = op.out_C(), k = op.k(), taps = k * k;
    SbConvTcPlan* plan = new SbConvTcPlan();
    int cp = (Cout + 15) / 16 * 16;
    if (cp > 256) cp = (cp + 255) / 256 * 256;
    plan->Cout_pad = cp;
    // weights: fp32 blob [tap][Cin][Cout] -> fp16 [tap][Cout_pad][Cin] (K-major B operand)
    std::vector<__half> w16((size_t)taps * cp * Cin, __float2half(0.f));
    const float* w = m->weights_host.data() + op.w_off();
    for (int t = 0; t < taps; ++t)
      for (int ci = 0; ci < Cin; ++ci)
        for (int co = 0; co < Cout; ++co)
          w16[((size_t)t * cp + co) * Cin + ci] = __float2half_rn(w[((size_t)t * Cin + ci) * Cout + co]);
    cudaError_t e = cudaMalloc((void**)&plan->w16, w16.size() * sizeof(__half));
    if (e != cudaSuccess) { delete plan; return sb_fail(h, SB_ERR_CUDA, "cudaMalloc w16: %s", cudaGetErrorString(e)); }
    e = cudaMemcpy(plan->w16, w16.data(), w16.size() * sizeof(__half), cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { cudaFree(plan->w16); delete plan; return sb_fail(h, SB_ERR_CUDA, "copy w16: %s", cudaGetErrorString(e)); }
    int rc = 0;
    if (op.kind() == SB_OPK_CONV && k >= 3) {   // 3x3 / 5x5 / 7x7, stride 1, SAME: one staged tile per filter column, rows are start offsets
      TcGroup g[MAX_GROUPS];
      for (int kx = 0; kx < k; ++kx) {
        g[kx].dx = kx - k / 2; g[kx].n_taps = k;
        for (int ky = 0; ky < k; ++ky) g[kx].taps[ky] = TcTap{ky, ky * k + kx};
      }
      rc = make_launch(h, m, op, plan, k, g, -(k / 2), k - 1, taps, 1, 0, 1, 0);
    } else if (op.kind() == SB_OPK_CONV) {   // 1x1 (stride 1, or stride 2 on the subsampled view)
      TcGroup g[1];
      g[0].dx = 0; g[0].n_taps = 1; g[0].taps[0] = TcTap{0, 0};
      if (res_fusable(m, oi)) {
        rc = make_launch(h, m, op, plan, 1, g, 0, 0, 1, 1, 0, 1, 0, nullptr, false, &plan->plain_launches);
        if (!rc) rc = make_launch(h, m, op, plan, 1, g, 0, 0, 1, 1, 0, 1, 0, nullptr, true);
        plan->res_fused = rc == 0;
      } else {
        rc = make_launch(h, m, op, plan, 1, g, 0, 0, 1, 1, 0, 1, 0);
      }
    } else if (k == 4) {
      // Conv2DTranspose k4 s2 SAME (forward-conv padding 1): out[2i+a] gets (ky, iy) = a==0 ? {(1,i),(3,i-1)} :
      // {(0,i+1),(2,i)}; same along x.  Each phase: 2 filter columns x 2 rows, box rows i-1..i+TH-1 (a=0) / i..i+TH (a=1).
      for (int a = 0; a < 2 && !rc; ++a)
        for (int bx = 0; bx < 2 && !rc; ++bx) {
          TcGroup g[2];
          const int kxs[2] = {bx == 0 ? 1 : 2, bx == 0 ? 3 : 0}, dxs[2] = {0, bx == 0 ? -1 : 1};
          for (int q = 0; q < 2; ++q) {
            g[q].dx = dxs[q]; g[q].n_taps = 2;
            if (a == 0) {             // dy0 = -1: box row 1 = input row i, box row 0 = i-1
              g[q].taps[0] = TcTap{1, 1 * 4 + kxs[q]};
              g[q].taps[1] = TcTap{0, 3 * 4 + kxs[q]};
            } else {                  // dy0 = 0: box row 0 = input row i, box row 1 = i+1
              g[q].taps[0] = TcTap{0, 2 * 4 + kxs[q]};
              g[q].taps[1] = TcTap{1, 0 * 4 + kxs[q]};
            }
          }
          rc = make_launch(h, m, op, plan, 2, g, a == 0 ? -1 : 0, 1, 16, 2, a, 2, bx);
        }
    } else {
      // Conv2DTranspose k3 s2: out[2i+a] gets (ky, iy) = a==0 ? {(0,i),(2,i-1)} : {(1,i)}; same along x.
      for (int a = 0; a < 2 && !rc; ++a)
        for (int bx = 0; bx < 2 && !rc; ++bx) {
          TcGroup g[2];
          int ng = 0;
          const int kxs[2] = {bx == 0 ? 0 : 1, 2}, dxs[2] = {0, -1};
          const int nkx = bx == 0 ? 2 : 1;
          const int extra = a == 0 ? 1 : 0;               // rows y0-1 .. y0+TH-1 when a == 0
          for (int q = 0; q < nkx; ++q) {
            g[ng].dx = dxs[q];
            if (a == 0) {
              g[ng].n_taps = 2;
              g[ng].taps[0] = TcTap{1, 0 * 3 + kxs[q]};     // ky=0 reads row i   (box row 1)
              g[ng].taps[1] = TcTap{0, 2 * 3 + kxs[q]};     // ky=2 reads row i-1 (box row 0)
            } else {
              g[ng].n_taps = 1;
              g[ng].taps[0] = TcTap{0, 1 * 3 + kxs[q]};
            }
            ++ng;
          }
          rc = make_launch(h, m, op, plan, ng, g, a == 0 ? -1 : 0, extra, 9, 2, a, 2, bx);
        }
    }
    if (!rc && op.kind() == SB_OPK_TCONV) rc = setup_tconv_form(h, m, op, plan);
    if (rc) { cudaFree(plan->w16); delete plan; return rc; }
    m->tc_plans[oi] = plan;
    if (head_kernel_ok(m, op, plan)) {
      const HeadShape hs = head_shape(op);
      plan->head = head_kernel(hs.nt, hs.kch);
      SB_CUDA(h, cudaFuncSetAttribute(plan->head, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kHeadSmem));
    }
    if (op.kind() == SB_OPK_CONV && op.pool_buf() >= 0 && oi + 1 < m->ops.size() &&
        m->ops[oi + 1].kind() == SB_OPK_POOL && (m->ops[oi + 1].flags() & SB_OPF_FUSED_POOL))
      if (plan->launches[0].forms[0].P.pool_out != nullptr) {
        plan->pool_fused = true;
        // dead-store elimination: with the pool fused, the conv's own output is written only for other readers
        // (skip connections into the decoder, heads).  The two finest encoder blocks of a UNet with output_stride 4
        // have none: 268 + 134 MB of stores per 8-frame C4 step.
        bool read = false;
        for (size_t oj = 0; oj < m->ops.size() && !read; ++oj) {
          if (oj == oi || oj == oi + 1) continue;
          const SbOp& o2 = m->ops[oj];
          if (o2.kind() == SB_OPK_PREPROCESS) continue;
          const int ext = split ? 3 * Cout : Cout;
          const bool overl_in = o2.in_buf() == op.out_buf() && o2.in_coff() < op.out_coff() + ext && op.out_coff() < o2.in_coff() + o2.in_C();
          const bool overl_in2 = o2.kind() == SB_OPK_ADD && o2.in2_buf() == op.out_buf() && o2.in2_coff() < op.out_coff() + ext &&
                                 op.out_coff() < o2.in2_coff() + o2.in_C();
          read = overl_in || overl_in2;
        }
        plan->out_dead = !read;
      }
  }
  return 0;
}

// Programmatic dependent launch (sb_tc_prims.cuh): every conv launch carries the attribute (its producer thread waits on
// the grid dependency before the first activation load); a launch that owns its SMs (one CTA per SM) is padded to the
// SM's whole shared memory and triggers its dependents right after its prologue, so that the next layer's CTAs set up
// (barriers, bias staging, descriptor prefetch) while this layer's last tiles drain.  SB_DISABLE_PDL=1 switches it off.
bool sb_pdl_on() {
  static int v = -1;
  if (v < 0) v = getenv("SB_DISABLE_PDL") ? 0 : 1;
  return v != 0;
}

// Launches form L.form of L for B frames (form 4: all four phases of the op).  Form 0 runs one CTA per tile, N tile and
// frame.  The persistent forms run as many CTAs as fit at once (capped at the work count), without shared-memory padding;
// each CTA triggers its dependents when it starts its last work item.
static void launch_form(const TcLaunch& L, int B, cudaStream_t stream, int skip_out) {
  const TcForm& F = L.forms[L.form];
  TcParams P = F.P;
  P.skip_out = skip_out;
  dim3 grid(std::min(F.n_items * B, F.max_ctas));
  size_t smem = F.smem;
  if (L.form == 0) {
    grid = dim3(L.grid.x, L.grid.y, B);
    P.pdl_trigger = (sb_pdl_on() && smem >= 114 * 1024) ? 1 : 0;   // already one CTA per SM
    if (P.pdl_trigger) smem = std::max(smem, kMaxDynSmem);       // nothing of the successor fits beside it
  } else {
    P.batch = B;
  }
  void* args[4] = {const_cast<CUtensorMap*>(&F.mapA), const_cast<CUtensorMap*>(&F.mapB), &P, const_cast<TcPhases*>(&F.Q)};
  sb_launch_pdl(form_kernel(L.form, P.KC, P.N), grid, dim3(F.threads), smem, stream, args);
}

// The launches of one op: the sub-pixel phases of a transposed conv run back to back on the launching stream, and under
// programmatic dependent launch each phase's CTAs start as the previous phase's SMs drain.  Form 4 runs all four phases
// in the first launch.
static int tc_launch(sb_handle_s* h, const std::vector<TcLaunch>& launches, int B, int skip_out) {
  for (const TcLaunch& L : launches) {
    launch_form(L, B, h->stream, skip_out);
    SB_CHECK_LAUNCH(h);
    if (L.form == kTconvForm) break;
  }
  return 0;
}

int sb_time_min(sb_handle_s* h, const char* what, float& best, const std::function<int()>& run) {
  cudaEvent_t e0, e1;
  SB_CUDA(h, cudaEventCreate(&e0));
  SB_CUDA(h, cudaEventCreate(&e1));
  best = 1e30f;
  int rc = 0;
  for (int rep = 0; rep < 4 && !rc; ++rep) {
    cudaEventRecord(e0, h->stream);
    if ((rc = run())) break;
    cudaEventRecord(e1, h->stream);
    if (cudaError_t e = cudaStreamSynchronize(h->stream); e != cudaSuccess)
      rc = sb_fail(h, SB_ERR_CUDA, "autotune launch (%s) failed: %s", what, cudaGetErrorString(e));
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    if (rep > 0) best = std::min(best, ms);
  }
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  return rc;
}

// Picks, for every tensor-core conv launch (each transposed-conv phase included), the fastest eligible kernel form 0-3,
// then for a transposed conv its four phase launches or the fused form 4, by timing them on the device at the
// configured batch (buffers are already allocated; their contents do not matter for timing).
int sb_conv_tc_autotune(sb_handle_s* h, SbModel* m) {
  char what[64];
  const bool dbg = getenv("SB_DEBUG") != nullptr;
  const char* fvar = getenv("SB_FORCE_VARIANT");
  const int force = fvar ? atoi(fvar) : -1;
  static const char* const form_name[kForms] = {"streaming", "resident", "halo", "wide", "tconv-fused"};
  for (size_t oi = 0; oi < m->tc_plans.size(); ++oi) {
    SbConvTcPlan* plan = m->tc_plans[oi];
    if (!plan || plan->head) continue;
    for (std::vector<TcLaunch>* list : {&plan->launches, &plan->plain_launches})
      for (size_t li = 0; li < list->size(); ++li) {
        TcLaunch& L = (*list)[li];
        float best[kTconvForm];
        int pick = 0;
        for (int f = 0; f < kTconvForm; ++f) {
          best[f] = 1e30f;
          if (!L.forms[f].ok) continue;
          L.form = f;
          snprintf(what, sizeof what, "op %zu, %s form", oi, form_name[f]);
          const int rc = sb_time_min(h, what, best[f], [&] {
            launch_form(L, m->B, h->stream, plan->out_dead && list == &plan->launches);
            return 0;
          });
          if (rc) return rc;
          if (best[f] < best[pick]) pick = f;
        }
        L.form = (force >= 0 && force < kTconvForm && L.forms[force].ok) ? force : pick;
        if (dbg) {
          fprintf(stderr, "[sb_conv_tc] op %zu launch %zu%s:", oi, li, list == &plan->launches ? "" : " (own output)");
          for (int f = 0; f < kTconvForm; ++f)
            if (L.forms[f].ok) fprintf(stderr, " %s %.1f us", form_name[f], best[f] * 1e3f);
          fprintf(stderr, " -> %s\n", form_name[L.form]);
        }
      }
  }
  // transposed convs: the four phase launches (whatever forms were just picked for them) against the fused form 4
  for (size_t oi = 0; oi < m->tc_plans.size(); ++oi) {
    SbConvTcPlan* plan = m->tc_plans[oi];
    if (!plan || plan->launches.empty() || !plan->launches[0].forms[kTconvForm].ok) continue;
    TcLaunch& L0 = plan->launches[0];
    const int phase_form = L0.form;
    float best[2];
    for (int f = 0; f < 2; ++f) {
      L0.form = f ? kTconvForm : phase_form;
      snprintf(what, sizeof what, "op %zu, %s", oi, f ? "fused tconv" : "tconv phases");
      if (const int rc = sb_time_min(h, what, best[f], [&] { return tc_launch(h, plan->launches, m->B, 0); })) return rc;
    }
    L0.form = (force >= 0 ? force == kTconvForm : best[1] < best[0]) ? kTconvForm : phase_form;
    if (dbg)
      fprintf(stderr, "[sb_conv_tc] op %zu launches (4 tconv phases) %.1f us, fused k_tconv_wg_hw %.1f us -> %s\n", oi, best[0] * 1e3f,
              best[1] * 1e3f, L0.form == kTconvForm ? "tconv-fused" : "phases");
  }
  return 0;
}

// k_head_1x1 over the op's pixels.  `log`: SB_DEBUG prints the launch shape (the production program's slot).
static SbLaunchFn head_entry(const SbModel* m, const SbOp& op, const SbConvTcPlan* plan, bool log) {
  const SbBuffer& ib = m->buffers[op.in_buf()];
  const SbBuffer& ob = m->buffers[op.out_buf()];
  const HeadShape hs = head_shape(op);
  if (log && getenv("SB_DEBUG"))
    fprintf(stderr, "[sb_conv_tc] head k_head_1x1: Cin %d Cout %d NT %d KCH %d n_ring %d smem %zu\n", op.in_C(), op.out_C(), hs.nt,
            hs.kch, hs.n_ring, hs.smem);
  const void* kern = plan->head;
  const __half* in = (const __half*)ib.dev;
  const __half* w = plan->w16;
  const float* bias = op.b_off() >= 0 ? m->weights_dev + op.b_off() : nullptr;
  float* out = (float*)ob.dev;
  int in_Ctot = ib.C, in_coff = op.in_coff(), Cin = op.in_C(), out_Ctot = ob.C, out_coff = op.out_coff(), Cout = op.out_C();
  int relu = (op.flags() & SB_OPF_RELU) ? 1 : 0, n_ring = hs.n_ring;
  const size_t frame_pix = (size_t)ob.H * ob.W;
  return [=](sb_handle_s* h, const void*, int, int B) mutable {
    size_t npix = (size_t)B * frame_pix;
    void* args[] = {&in, &in_Ctot, &in_coff, &Cin, &w, &bias, &out, &out_Ctot, &out_coff, &Cout, &relu, &npix, &n_ring};
    const int grid = (int)std::min<size_t>((npix + 127) / 128, (size_t)h->sm_count * 2);
    sb_launch_pdl(kern, dim3(grid), dim3(256), hs.smem, h->stream, args);
    SB_CHECK_LAUNCH(h);
    return 0;
  };
}

// Production: a dead output is not stored, and a fused residual ADD runs in the epilogue.  All stores: the output is
// stored, by the plain launches where the ADD was fused (the ADD op then runs in its own slot).  A fused pool is written
// by both.  The slot refers to the plan's launches: the programs go before the plans.
SbTcEntry sb_conv_tc_entry(const SbModel* m, int op_index, bool all_stores) {
  const SbConvTcPlan* plan = m->tc_plans[op_index];
  SbTcEntry e;
  if (plan->head) {
    e.run = head_entry(m, m->ops[op_index], plan, !all_stores);
    return e;
  }
  const bool res = plan->res_fused && !all_stores;
  const int skip = plan->out_dead && !all_stores;
  const std::vector<TcLaunch>* launches = plan->res_fused && all_stores ? &plan->plain_launches : &plan->launches;
  e.run = [launches, skip](sb_handle_s* h, const void*, int, int B) { return tc_launch(h, *launches, B, skip); };
  if (plan->pool_fused || res) e.absorbs = op_index + 1;
  e.elides_out = skip || res;
  return e;
}
