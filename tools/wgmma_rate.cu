// Issue rate of the wgmma groups the conv kernel forms run, with every operand already in shared memory: no loads, no
// barriers, no epilogue.  One CTA per SM, two warpgroups, each issuing per "slice" KSTEPS = 4 k-steps x BLOCKS m64 blocks
// of m64nNk16 as one group and waiting with wgmma.wait_group 1, as k_conv_wg (form 0) and k_conv_wg_hw (form 3) do.
// A is either the 128B-swizzled box of form 0 or the non-swizzled halo patch of forms 2 / 3 (8-channel planes
// [18][18][8], LBO = one plane, SBO = one patch row); B is a 128B-swizzled [N x 64] weight slice.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o /tmp/wgmma_rate tools/wgmma_rate.cu -lcuda && /tmp/wgmma_rate
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdint>

namespace {
#include "../sleap_b200/csrc/sb_tc_prims.cuh"

constexpr int kPlane = 18 * 18 * 16;         // one 8-channel plane of a 16x16-item halo patch
constexpr int kSmem = 160 * 1024;            // more than half the SM: one CTA per SM

template <int N, int BLOCKS, bool PATCH>
__global__ void __launch_bounds__(256, 1) k_rate(int slices, float* sink) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* a = base;                         // PATCH: 8 planes (41.5 KB); else BLOCKS x 2 warpgroups x 8 KB swizzled rows
  uint8_t* b = base + 64 * 1024;             // [N x 64] swizzled weight slice
  // non-trivial operand values (the tensor pipe's power, hence its clock, depends on them)
  for (int i = threadIdx.x; i < 32 * 1024 + N * 64; i += blockDim.x)
    reinterpret_cast<__half*>(base)[i] = __float2half(0.01f * (float)((i * 7) % 13 - 6));
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  const int wg = threadIdx.x >> 7;
  const uint64_t db = make_desc(0, 128, 1) + (uint64_t)(smem_u32(b) >> 4);
  float acc[BLOCKS][N / 2];
#pragma unroll
  for (int i = 0; i < BLOCKS; ++i)
#pragma unroll
    for (int j = 0; j < N / 2; ++j) acc[i][j] = 0.f;
  for (int s = 0; s < slices; ++s) {
    wgmma_fence();
#pragma unroll
    for (int i = 0; i < BLOCKS; ++i) wgmma_reg_fence(acc[i]);
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int i = 0; i < BLOCKS; ++i) {
        uint64_t da;
        if (PATCH) {
          // block (row wg * BLOCKS / 2 + i / 2, column i % 2) of the patch; k-step k = planes 2k, 2k + 1
          const uint32_t off = (uint32_t)(((8 * (wg * (BLOCKS / 2) + (i >> 1))) * 18 + 8 * (i & 1)) * 16 + 2 * k * kPlane);
          da = make_desc_interleave(0, kPlane, 18 * 16) + (uint64_t)((smem_u32(a) + (BLOCKS == 1 ? 0u : off)) >> 4);
        } else {
          da = make_desc(0, 128, 1) + (uint64_t)((smem_u32(a) + (uint32_t)((wg * BLOCKS + i) * 8192)) >> 4) + 2 * k;
        }
        wgmma_f16<N>(acc[i], da, db + 2 * k, 1u);
      }
    wgmma_commit();
#pragma unroll
    for (int i = 0; i < BLOCKS; ++i) wgmma_reg_fence(acc[i]);
    wgmma_wait<1>();
  }
  wgmma_wait<0>();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < BLOCKS; ++i)
#pragma unroll
    for (int j = 0; j < N / 2; ++j) t += acc[i][j];
  if (t == 12345.f) sink[threadIdx.x] = t;
}

// The fused first block's conv1 (sb_conv01.cu): per slice, nine m64n16k16 (one 3x3 filter) from WGS of the two
// warpgroups, spread round-robin over NACC independent accumulators, one group, wgmma.wait_group 1.  B is a 32B-swizzled
// 16x16 tap.  SS: A is the non-swizzled conv0 planes [18][34][8] of an 8x8-pixel block, tap (ky, kx) at start offset
// (ky * 34 + kx) * 16.  RS: A is three register fragments (one per kx) loaded with ldmatrix.x4 from 64 consecutive pixels
// of one plane row, reloaded every slice into the set the group before the last one read (three sets), as an image-row
// item does per input row.
template <bool RS, int NACC, int WGS>
__global__ void __launch_bounds__(256, 1) k_rate16(int slices, float* sink) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int kPlane01 = 18 * 66 * 16;     // RS: planes [18][66][8]; SS uses the first 18 x 34 pixels of each
  uint8_t* a = base;                         // 2 planes
  uint8_t* b = base + 2 * kPlane01;          // 9 taps x 512 B
  for (int i = threadIdx.x; i < (2 * kPlane01 + 9 * 512) / 2; i += blockDim.x)
    reinterpret_cast<__half*>(base)[i] = __float2half(0.01f * (float)((i * 7) % 13 - 6));
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  const int wg = threadIdx.x >> 7, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  if (wg >= WGS) return;
  const uint64_t db = make_desc(0, 32, 3) + (uint64_t)(smem_u32(b) >> 4);
  const uint64_t da = make_desc_interleave(0, kPlane01, 34 * 16) + (uint64_t)(smem_u32(a) >> 4);
  // ldmatrix row address of this lane: pixel 16 warp + (lane & 15) of plane row 1, 8-channel plane lane >> 4
  const uint32_t arow = smem_u32(a) + (uint32_t)((lane >> 4) * kPlane01 + (66 + 16 * warp + (lane & 15)) * 16);
  uint32_t f[3][3][4];
#pragma unroll
  for (int kx = 0; kx < 3; ++kx) ldmatrix_x4(f[0][kx], arow + 16 * kx);
  float acc[NACC][8];
#pragma unroll
  for (int i = 0; i < NACC; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  auto slice = [&](int s, int buf) {               // group s reads set buf; set (buf + 1) % 3 was read by group s - 2
    wgmma_fence();
#pragma unroll
    for (int i = 0; i < NACC; ++i) wgmma_reg_fence(acc[i]);
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      if (RS) wgmma_f16_rs16(acc[t % NACC], f[buf][t % 3], db + 32 * t, 1u);
      else wgmma_f16<16>(acc[t % NACC], da + (uint64_t)((((t / 3) * 34 + t % 3) * 16) >> 4), db + 32 * t, 1u);
    }
    wgmma_commit();
    if (RS) {
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) ldmatrix_x4(f[(buf + 1) % 3][kx], arow + (uint32_t)((s & 7) * 66 * 16) + 16 * kx);
    }
#pragma unroll
    for (int i = 0; i < NACC; ++i) wgmma_reg_fence(acc[i]);
    wgmma_wait<1>();
  };
  for (int s = 0; s < slices; s += 3) {
    slice(s, 0);
    slice(s + 1, 1);
    slice(s + 2, 2);
  }
  wgmma_wait<0>();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < NACC; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) t += acc[i][j];
  if (t == 12345.f) sink[threadIdx.x] = t;
}

template <typename K>
void time_kernel(K kern, const char* name, int sms, double flop_per_slice_cta) {
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
  float* sink;
  cudaMalloc(&sink, 1024 * sizeof(float));
  const int slices = 4098;             // a multiple of the RS loop's unroll by 3
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  for (int w = 0; w < 3; ++w) kern<<<sms, 256, kSmem>>>(slices, sink);
  cudaEventRecord(e0);
  const int reps = 10;
  for (int r = 0; r < reps; ++r) kern<<<sms, 256, kSmem>>>(slices, sink);
  cudaEventRecord(e1);
  cudaError_t e = cudaEventSynchronize(e1);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  const double flop = flop_per_slice_cta * (double)slices * sms * reps;
  printf("%-52s %7.1f TFLOP/s  %6.3f us per slice and CTA  %s\n", name, flop / (ms * 1e-3) / 1e12,
         ms * 1e3 / reps / slices, e == cudaSuccess ? "" : cudaGetErrorString(e));
  cudaFree(sink);
}

template <int N, int BLOCKS, bool PATCH>
void run(const char* name, int sms) {
  time_kernel(k_rate<N, BLOCKS, PATCH>, name, sms, 2.0 * 64 * N * 16 * 4 * BLOCKS * 2);
}

template <bool RS, int NACC, int WGS>
void run16(const char* name, int sms) {
  time_kernel(k_rate16<RS, NACC, WGS>, name, sms, 2.0 * 64 * 16 * 16 * 9 * WGS);
}
}  // namespace

int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  run<128, 1, false>("N 128, 1 block / wg, swizzled A (form 0)", sms);
  run<128, 2, false>("N 128, 2 blocks / wg, swizzled A", sms);
  run<128, 2, true>("N 128, 2 blocks / wg, patch A (form 3)", sms);
  run<256, 1, false>("N 256, 1 block / wg, swizzled A (form 0)", sms);
  run<256, 1, true>("N 256, 1 block / wg, patch A", sms);
  run<64, 4, false>("N 64, 4 blocks / wg, swizzled A", sms);
  run<64, 4, true>("N 64, 4 blocks / wg, patch A (form 3)", sms);
  run16<false, 1, 1>("m64n16k16 x 9, 1 acc, 1 wg, SS planes A", sms);
  run16<false, 3, 1>("m64n16k16 x 9, 3 acc, 1 wg, SS planes A", sms);
  run16<false, 1, 2>("m64n16k16 x 9, 1 acc, 2 wg, SS planes A", sms);
  run16<false, 3, 2>("m64n16k16 x 9, 3 acc, 2 wg, SS planes A", sms);
  run16<true, 1, 1>("m64n16k16 x 9, 1 acc, 1 wg, RS ldmatrix A", sms);
  run16<true, 3, 1>("m64n16k16 x 9, 3 acc, 1 wg, RS ldmatrix A", sms);
  run16<true, 1, 2>("m64n16k16 x 9, 1 acc, 2 wg, RS ldmatrix A", sms);
  run16<true, 3, 2>("m64n16k16 x 9, 3 acc, 2 wg, RS ldmatrix A", sms);
  return 0;
}
