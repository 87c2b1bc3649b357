// Fused first encoder block of the UNet for sm_90a: raw frame -> conv0 (3x3, 1 -> 16, bias, ReLU) -> conv1 (3x3,
// 16 -> 16, bias, ReLU) -> MaxPool2D(2, 2) in one kernel.  Neither the 16-channel full-resolution tensor between the
// two convolutions nor conv1's own full-resolution output leaves the SM: per 8-frame C4 step that removes 268 MB of
// writes + 268 MB of reads of the intermediate and conv1's dead full-resolution stores.
//
// Replaces, for that block: InferenceLayer.preprocess (sleap/nn/inference.py:940-967, uint8 -> float * 1/255, zero
// pad to the stride) and the Keras layers stack0_enc0_conv0/act0, conv1/act1 and the pool of enc1
// (sleap/nn/architectures/encoder_decoder.py:94-144, unet.py:140-205), as dispatched to cuDNN by TensorFlow.
//
// One CTA = one 16x8-pixel tile of conv1's output (M = 128), two warpgroups:
//   1. the 20x12 frame patch around the tile -> shared memory (fp16-rounded pixels, zero outside the frame);
//   2. conv0 on the CUDA cores for the 18x10 pixels conv1 reads, written as fp16 into three 32-byte-swizzled
//      [160 rows x 16 ch] A tiles, one per filter column of conv1 (tile kx row 16 yy + xx = conv0 pixel
//      (y0 - 1 + yy, x0 + kx - 1 + xx)), so that filter row ky of that column is the start offset 16 ky rows;
//   3. conv1 as nine wgmma m64n16k16 per warpgroup (fp32 accumulators in registers), weights [tap][co][ci] in shared memory;
//   4. accumulators -> shared-memory staging -> bias, ReLU, fp16 rounding, 2x2 max -> pooled NHWC output.
// The same rounding points as the separate launches (fp16 frame pixels and weights, fp16 intermediate, fp16 conv1
// output before the pool).
#include <cuda.h>

#include <algorithm>

#include "sb_model.h"

namespace {

#include "sb_tc_prims.cuh"

constexpr int TW = 16, TH = 8;
constexpr int PW = TW + 4, PH = TH + 4;     // frame patch
constexpr int CW0 = TW + 2, CH0 = TH + 2;   // conv0 pixels conv1 reads
constexpr int A_ROWS = CH0 * TW;            // 160 rows of 32 B per A tile
constexpr int A_BYTES = A_ROWS * 32;        // 5120
constexpr int SP = 20;                      // staging row pitch (floats)

constexpr int OFF_A = 0;                                // 3 A tiles
constexpr int OFF_W1 = OFF_A + 3 * A_BYTES;             // 9 taps x [16 co][16 ci] fp16 = 9 x 512 B
constexpr int OFF_STAGE = OFF_W1 + 9 * 512;             // [128][SP] fp32
constexpr int OFF_PATCH = OFF_STAGE + 128 * SP * 4;     // [PH][PW] fp32
constexpr int OFF_PAR = OFF_PATCH + PH * PW * 4;        // w0h[144] bias0[16] bias1[16]
constexpr int SMEM_BYTES = OFF_PAR + (144 + 32) * 4 + 1024;

struct C01Params {
  const void* frames;
  int frames_u8;
  int Hin, Win, Hnet, Wnet, tiles_x;
  __half* pool_out;
  int pool_H, pool_W, pool_Ctot, pool_coff;
  const float* bias0;
  const float* bias1;
  const float* w0h;          // conv0 weights rounded to fp16, as float: [9][16]
  const __half* w1t;         // conv1 weights [9][16 co][16 ci] fp16
  int relu0, relu1;
};

// byte offset of 16-byte chunk c of row r in a 32-byte-swizzled K-major tile (chunk bit 4 ^= address bit 7)
__device__ __forceinline__ int sw32(int r, int c) { return r * 32 + ((c ^ ((r >> 2) & 1)) << 4); }

template <typename TI>
__global__ void __launch_bounds__(256) k_conv01(const __grid_constant__ C01Params P) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  float* s_stage = reinterpret_cast<float*>(base + OFF_STAGE);
  float* s_patch = reinterpret_cast<float*>(base + OFF_PATCH);
  float* s_w0 = reinterpret_cast<float*>(base + OFF_PAR);
  float* s_b0 = s_w0 + 144;
  float* s_b1 = s_b0 + 16;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int x0 = (blockIdx.x % P.tiles_x) * TW, y0 = (blockIdx.x / P.tiles_x) * TH, b = blockIdx.y;

  // weights / biases (static) and the frame patch
  for (int i = tid; i < 9 * 16 * 2; i += 256) {        // 9 taps x 16 rows x 2 chunks
    const int t = i >> 5, r = (i >> 1) & 15, c = i & 1;
    *reinterpret_cast<uint4*>(base + OFF_W1 + t * 512 + sw32(r, c)) = reinterpret_cast<const uint4*>(P.w1t + (t * 16 + r) * 16)[c];
  }
  if (tid < 144) s_w0[tid] = P.w0h[tid];
  if (tid < 16) { s_b0[tid] = P.bias0 ? P.bias0[tid] : 0.f; s_b1[tid] = P.bias1 ? P.bias1[tid] : 0.f; }
  const float sc = P.frames_u8 ? (1.0f / 255.0f) : 1.0f;     // ensure_float (normalization.py:34-49)
  const TI* img = reinterpret_cast<const TI*>(P.frames) + (size_t)b * P.Hin * P.Win;
  for (int i = tid; i < PH * PW; i += 256) {
    const int y = y0 - 2 + i / PW, x = x0 - 2 + i % PW;
    float v = 0.f;
    if (y >= 0 && y < P.Hin && x >= 0 && x < P.Win) v = __half2float(__float2half_rn(__fmul_rn((float)img[(size_t)y * P.Win + x], sc)));
    s_patch[i] = v;
  }
  __syncthreads();

  // conv0 for the CH0 x CW0 pixels conv1 reads, 8 channels per item; zero outside the network image (conv1's SAME pad)
  for (int it = tid; it < CH0 * CW0 * 2; it += 256) {
    const int half = it & 1, p = it >> 1, yy = p / CW0, cx = p % CW0;
    const int y = y0 - 1 + yy, x = x0 - 1 + cx;
    __align__(16) __half h[8];
    if (y >= 0 && y < P.Hnet && x >= 0 && x < P.Wnet) {
      float acc[8];
#pragma unroll
      for (int c = 0; c < 8; ++c) acc[c] = 0.f;
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
          const float v = s_patch[(yy + ky) * PW + cx + kx];
#pragma unroll
          for (int c = 0; c < 8; ++c) acc[c] = fmaf(v, s_w0[(ky * 3 + kx) * 16 + 8 * half + c], acc[c]);
        }
#pragma unroll
      for (int c = 0; c < 8; ++c) {
        float v = acc[c] + s_b0[8 * half + c];
        if (P.relu0) v = fmaxf(v, 0.f);
        h[c] = __float2half_rn(v);
      }
    } else {
#pragma unroll
      for (int c = 0; c < 8; ++c) h[c] = __float2half_rn(0.f);
    }
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {                    // tile kx holds this pixel at column cx - kx
      const int xx = cx - kx;
      if (xx >= 0 && xx < TW) *reinterpret_cast<uint4*>(base + OFF_A + kx * A_BYTES + sw32(yy * TW + xx, half)) = *reinterpret_cast<uint4*>(h);
    }
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma
  __syncthreads();

  // conv1: warpgroup wg multiplies tile rows [64 wg, 64 wg + 64)
  const int wg = warp >> 2;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  const uint64_t desc_hi = make_desc(0, 32, 3);
  wgmma_fence();
  wgmma_reg_fence(acc);
#pragma unroll
  for (int ky = 0; ky < 3; ++ky)
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const uint32_t a = smem_u32(base + OFF_A + kx * A_BYTES + (ky * TW + 64 * wg) * 32);
      const uint32_t w = smem_u32(base + OFF_W1 + (ky * 3 + kx) * 512);
      wgmma_f16<16>(acc, desc_hi + (a >> 4), desc_hi + (w >> 4), (ky | kx) ? 1u : 0u);
    }
  wgmma_commit();
  wgmma_wait<0>();
  wgmma_reg_fence(acc);

  // accumulators -> staging (fragment rows 16 (warp % 4) + lane / 4 (+ 8), columns 8 j + 2 (lane % 4) (+ 1))
  const int frow = wg * 64 + (warp & 3) * 16 + (lane >> 2), fcol = 2 * (lane & 3);
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    *reinterpret_cast<float2*>(s_stage + frow * SP + 8 * j + fcol) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2*>(s_stage + (frow + 8) * SP + 8 * j + fcol) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
  __syncthreads();

  // bias, ReLU, fp16 rounding (conv1's stored value), 2x2 max: thread = (pooled pixel, channel pair)
  const int pp = tid >> 3, cp = 2 * (tid & 7);
  const int py = pp / (TW / 2), px = pp % (TW / 2);
  const int gy = (y0 >> 1) + py, gx = (x0 >> 1) + px;
  if (gy < P.pool_H && gx < P.pool_W) {
    __half2 m = __float2half2_rn(-INFINITY);
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const float* s = s_stage + ((2 * py + a) * TW + 2 * px + c) * SP + cp;
        float v0 = s[0] + s_b1[cp], v1 = s[1] + s_b1[cp + 1];
        if (P.relu1) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
        m = __hmax2(m, __floats2half2_rn(v0, v1));
      }
    *reinterpret_cast<__half2*>(P.pool_out + (((size_t)b * P.pool_H + gy) * P.pool_W + gx) * P.pool_Ctot + P.pool_coff + cp) = m;
  }
}

}  // namespace

struct SbConv01Plan {
  C01Params P;
  __half* w1t = nullptr;     // [9][16][16]
  float* w0h = nullptr;      // [9][16]
  int conv0_op = -1, conv1_op = -1;
};

void sb_conv01_release(SbModel* m) {
  if (!m->conv01) return;
  if (m->conv01->w1t) cudaFree(m->conv01->w1t);
  if (m->conv01->w0h) cudaFree(m->conv01->w0h);
  delete m->conv01;
  m->conv01 = nullptr;
}

// The block qualifies when: 1-channel frames, no resize; conv0 = 3x3 s1 1 -> 16 (+ReLU) fused with PREPROCESS;
// conv1 = 3x3 s1 16 -> 16 whose 2x2 max-pool is fused and whose own output has no other reader (sb_conv_tc.cu marks it).
int sb_conv01_prepare(sb_handle_s* h, SbModel* m, int conv0_op, int conv1_op, bool conv1_out_dead) {
  sb_conv01_release(m);
  if (getenv("SB_DISABLE_CONV01") || m->precision != 0 || !conv1_out_dead) return 0;
  const SbOp& c0 = m->ops[conv0_op];
  const SbOp& c1 = m->ops[conv1_op];
  if (m->Cin != 1 || c0.in_C() != 1 || c0.out_C() != 16 || c0.k() != 3 || c0.stride() != 1 || (c0.flags() & SB_OPF_BN)) return 0;
  if (c1.in_C() != 16 || c1.out_C() != 16 || c1.k() != 3 || c1.stride() != 1 || (c1.flags() & SB_OPF_BN)) return 0;
  if (c1.in_buf() != c0.out_buf() || c1.in_coff() != c0.out_coff() || c1.pool_buf() < 0) return 0;
  const SbBuffer& ob0 = m->buffers[c0.out_buf()];
  const SbBuffer& pb = m->buffers[c1.pool_buf()];
  if (ob0.f32 || pb.f32 || pb.C % 2 || c1.pool_coff() % 2 || ob0.H % 2 || ob0.W % 2) return 0;
  for (size_t oi = 0; oi < m->ops.size(); ++oi)            // conv0's output must feed conv1 only
    if ((int)oi != conv1_op && m->ops[oi].kind() != SB_OPK_PREPROCESS && (int)oi != conv0_op &&
        (m->ops[oi].in_buf() == c0.out_buf() || (m->ops[oi].kind() == SB_OPK_ADD && m->ops[oi].in2_buf() == c0.out_buf())))
      return 0;
  SbConv01Plan* pl = new SbConv01Plan();
  pl->conv0_op = conv0_op; pl->conv1_op = conv1_op;
  const float* w0 = m->weights_host.data() + c0.w_off();     // [9][1][16]
  const float* w1 = m->weights_host.data() + c1.w_off();     // [9][16][16]
  std::vector<__half> w1t((size_t)9 * 16 * 16);
  std::vector<float> w0h(144);
  for (int t = 0; t < 9; ++t)
    for (int co = 0; co < 16; ++co) {
      w0h[t * 16 + co] = __half2float(__float2half_rn(w0[t * 16 + co]));
      for (int ci = 0; ci < 16; ++ci) w1t[((size_t)t * 16 + co) * 16 + ci] = __float2half_rn(w1[((size_t)t * 16 + ci) * 16 + co]);
    }
  auto fail = [&](const char* what) { delete pl; return sb_fail(h, SB_ERR_CUDA, "conv01: %s", what); };
  if (cudaMalloc((void**)&pl->w1t, w1t.size() * 2) != cudaSuccess) return fail("cudaMalloc");
  if (cudaMalloc((void**)&pl->w0h, w0h.size() * 4) != cudaSuccess) { cudaFree(pl->w1t); return fail("cudaMalloc"); }
  m->conv01 = pl;                                          // released with the model from here on
  if (cudaMemcpy(pl->w1t, w1t.data(), w1t.size() * 2, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(pl->w0h, w0h.data(), w0h.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess) {
    sb_conv01_release(m);
    return sb_fail(h, SB_ERR_CUDA, "conv01: weight copy");
  }
  C01Params& P = pl->P;
  memset(&P, 0, sizeof(P));
  P.Hin = m->Hin; P.Win = m->Win; P.Hnet = ob0.H; P.Wnet = ob0.W;
  P.tiles_x = (ob0.W + TW - 1) / TW;
  P.pool_out = (__half*)pb.dev; P.pool_H = pb.H; P.pool_W = pb.W; P.pool_Ctot = pb.C; P.pool_coff = c1.pool_coff();
  P.bias0 = c0.b_off() >= 0 ? m->weights_dev + c0.b_off() : nullptr;
  P.bias1 = c1.b_off() >= 0 ? m->weights_dev + c1.b_off() : nullptr;
  P.w0h = pl->w0h; P.w1t = pl->w1t;
  P.relu0 = (c0.flags() & SB_OPF_RELU) ? 1 : 0;
  P.relu1 = (c1.flags() & SB_OPF_RELU) ? 1 : 0;
  return 0;
}

bool sb_conv01_can(const SbModel* m, int conv0_op) { return m->conv01 && m->conv01->conv0_op == conv0_op && m->conv01_enabled; }
int sb_conv01_conv1_op(const SbModel* m) { return m->conv01 ? m->conv01->conv1_op : -1; }

int sb_conv01_launch(sb_handle_s* h, SbModel* m, const void* frames_dev, int frames_are_u8, int B) {
  SbConv01Plan* pl = m->conv01;
  C01Params P = pl->P;
  P.frames = frames_dev; P.frames_u8 = frames_are_u8;
  const dim3 grid(P.tiles_x * ((P.Hnet + TH - 1) / TH), B);
  if (frames_are_u8) k_conv01<unsigned char><<<grid, 256, SMEM_BYTES, h->stream>>>(P);
  else k_conv01<float><<<grid, 256, SMEM_BYTES, h->stream>>>(P);
  SB_CHECK_LAUNCH(h);
  return 0;
}
