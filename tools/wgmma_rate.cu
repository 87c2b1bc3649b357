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

template <int N, int BLOCKS, bool PATCH>
void run(const char* name, int sms) {
  auto kern = k_rate<N, BLOCKS, PATCH>;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
  float* sink;
  cudaMalloc(&sink, 1024 * sizeof(float));
  const int slices = 4096;
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
  const double flop = 2.0 * 64 * N * 16 * 4 * BLOCKS * 2 * (double)slices * sms * reps;
  printf("%-44s %7.1f TFLOP/s  %6.3f us per slice and CTA  %s\n", name, flop / (ms * 1e-3) / 1e12,
         ms * 1e3 / reps / slices, e == cudaSuccess ? "" : cudaGetErrorString(e));
  cudaFree(sink);
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
  return 0;
}
