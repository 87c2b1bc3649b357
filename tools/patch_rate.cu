// Rate of the halo-patch loaders of conv forms 2 and 3 (sb_conv_tc.cu), with no MMA: one CTA per SM on all SMs loops
// over the items of 8 NHWC frames and stages each item's (8 BY + 2) x 18-pixel patch into a ring of patch slots; one
// consumer warp waits for each slot and releases it.  Three loaders:
//   cp.async  the 16-byte cp.async loader the halo forms used before the TMA loader (128 threads for form 2's shapes,
//             96 for form 3's), one cp.async.mbarrier.arrive.noinc per loader thread, into KC / 8 non-swizzled
//             8-channel planes [rows][18][8]
//   tma       one elected thread, one cp.async.bulk.tensor.5d box {8, 18, rows, KC / 8, 1} per patch through the map
//             {8 ch, W, H, C / 8, B}, byte strides {C 2, W C 2, 16, H W C 2}, into the same planes (SAME padding and
//             the planes beyond C are TMA zero fill)
//   tma-sw    one elected thread, one cp.async.bulk.tensor.4d box {KC, 18, rows, 1} per patch through the map
//             {C, W, H, B}, byte strides {C 2, W C 2, H W C 2}, swizzled at the row width (SW128 / SW64 / SW32 for
//             KC 64 / 32 / 16), into pixel rows [rows][18][KC]: the loader of forms 2 and 3
// Each shape prints µs per patch and SM, the patch bytes over the whole GPU in GB/s, and whether the XOR of every staged
// word, at its position in the planes layout, agrees between the loaders.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o /tmp/patch_rate tools/patch_rate.cu -lcuda && /tmp/patch_rate
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstdio>

namespace {
#include "../sleap_b200/csrc/sb_tc_prims.cuh"

__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3,
                                            int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}

constexpr int kCols = 18;
constexpr int kThreads = 160;                 // 4 loader warps + 1 consumer warp

// the cp.async loader: loader thread lid of n_loaders issues its share of the 16-byte pieces (patch pixel p, plane pl),
// piece to thread (NP p + pl) mod n_loaders, zero-size source outside the image and beyond C
template <int NP>
__device__ __forceinline__ void stage_cp_async(const __half* in, int H, int W, int C, uint32_t dst, int plane, int rows, int c0,
                                               int b, int ys, int xs, int lid, int n_loaders) {
  const int pl = lid % NP, c = c0 + pl * 8;
  const bool c_ok = c < C;
  const __half* in_c = in + (size_t)b * H * W * C + c;
  const uint32_t d = dst + (uint32_t)(pl * plane);
  for (int p = lid / NP; p < rows * kCols; p += n_loaders / NP) {
    const int y = ys + p / kCols, x = xs + p % kCols;
    const bool ok = c_ok && y >= 0 && y < H && x >= 0 && x < W;
    const __half* src = ok ? in_c + ((size_t)y * W + x) * C : in;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d + (uint32_t)(p * 16)), "l"(src), "r"(ok ? 16 : 0) : "memory");
  }
}

// byte strides of a patch slot: the patch, rounded up to the swizzle pattern of its pixel rows (8 rows of NP * 16 bytes)
__host__ __device__ constexpr int slot_bytes(int np, int rows) { return (np * rows * kCols * 16 + 128 * np - 1) / (128 * np) * (128 * np); }

template <int NP>
__global__ void __launch_bounds__(kThreads, 1) k_patch(const __grid_constant__ CUtensorMap map, const __half* in, int B, int H,
                                                       int W, int C, int BY, int n_slots, int n_loaders, int mode, unsigned* check) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const int rows = 8 * BY + 2, plane = rows * kCols * 16, box = NP * plane, slot = slot_bytes(NP, rows);
  const bool tma = mode > 0;
  uint8_t* ring = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(ring + (size_t)n_slots * slot);
  uint64_t* empty = full + n_slots;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_x = (W + 15) / 16, n_tiles = tiles_x * ((H + 8 * BY - 1) / (8 * BY)), n_work = n_tiles * B;
  const int n_chunks = (C + 8 * NP - 1) / (8 * NP);
  if (threadIdx.x == 0) {
    for (int i = 0; i < n_slots; ++i) { mbar_init(smem_u32(full + i), tma ? 1 : n_loaders); mbar_init(smem_u32(empty + i), 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp < 4) {
    const bool issuer = tma ? threadIdx.x == 0 : (int)threadIdx.x < n_loaders;
    if (!issuer) return;
    for (int i = 0, w = blockIdx.x; w < n_work; w += gridDim.x) {
      const int tile = w % n_tiles, b = w / n_tiles;
      const int ys = (tile / tiles_x) * (8 * BY) - 1, xs = (tile % tiles_x) * 16 - 1;
      for (int ch = 0; ch < n_chunks; ++ch, ++i) {
        const int s = i % n_slots;
        const uint32_t dst = smem_u32(ring + (size_t)s * slot);
        mbar_wait(smem_u32(empty + s), ((i / n_slots) & 1) ^ 1);
        if (tma) {
          mbar_expect_tx(smem_u32(full + s), (uint32_t)box);
          if (mode == 1) tma_load_5d(dst, &map, smem_u32(full + s), 0, xs, ys, ch * NP, b);
          else tma_load_4d(dst, &map, smem_u32(full + s), ch * 8 * NP, xs, ys, b);
        } else {
          stage_cp_async<NP>(in, H, W, C, dst, plane, rows, ch * 8 * NP, b, ys, xs, threadIdx.x, n_loaders);
          asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(full + s)) : "memory");
        }
      }
    }
    if (!tma) asm volatile("cp.async.wait_all;" ::: "memory");
    return;
  }
  unsigned x = 0;
  for (int i = 0, w = blockIdx.x; w < n_work; w += gridDim.x)
    for (int ch = 0; ch < n_chunks; ++ch, ++i) {
      const int s = i % n_slots;
      mbar_wait(smem_u32(full + s), (i / n_slots) & 1);
      if (check) {
        const unsigned* p = reinterpret_cast<const unsigned*>(ring + (size_t)s * slot);
        for (int k = lane; k < box / 4; k += 32) {
          int kp = k;                                          // the word's index in the planes layout
          if (mode == 2) {
            const int l = 4 * k ^ (((4 * k) >> 7) & (NP - 1)) << 4, rb = 16 * NP;   // unswizzled byte offset
            kp = ((l % rb) / 16 * plane + l / rb * 16 + l % 16) / 4;
          }
          x ^= p[k] * (unsigned)(2 * kp + 1);
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(smem_u32(empty + s));
    }
  if (check) atomicXor(check, x);
}

__global__ void k_fill(__half* p, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    p[i] = __float2half((float)((i * 2654435761u) >> 20 & 1023) / 1024.f);
}

struct Shape { const char* name; int KC, BY, S, C, loaders, slots; };

template <int NP>
void run(const Shape& sh, int sms) {
  const int B = 8, H = sh.S, W = sh.S, C = sh.C;
  const size_t n = (size_t)B * H * W * C;
  __half* in;
  unsigned* check;
  cudaMalloc(&in, n * 2);
  cudaMalloc(&check, 3 * sizeof(unsigned));
  cudaMemset(check, 0, 3 * sizeof(unsigned));
  k_fill<<<1024, 256>>>(in, n);
  const int rows = 8 * sh.BY + 2, patch_bytes = NP * rows * kCols * 16, slot = slot_bytes(NP, rows);
  CUtensorMap map, map_sw;
  cuuint64_t dims[5] = {8, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)(C / 8), (cuuint64_t)B};
  cuuint64_t strides[4] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, 16, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[5] = {8, kCols, (cuuint32_t)rows, (cuuint32_t)NP, 1};
  cuuint32_t es[5] = {1, 1, 1, 1, 1};
  const CUresult enc = cuTensorMapEncodeTiled(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, in, dims, strides, box, es,
                                              CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                              CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  cuuint64_t dims_sw[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides_sw[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box_sw[4] = {(cuuint32_t)sh.KC, kCols, (cuuint32_t)rows, 1};
  const CUresult enc_sw = cuTensorMapEncodeTiled(
      &map_sw, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, in, dims_sw, strides_sw, box_sw, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
      NP == 8 ? CU_TENSOR_MAP_SWIZZLE_128B : (NP == 4 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B),
      CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (enc != CUDA_SUCCESS || enc_sw != CUDA_SUCCESS) {
    printf("%-40s cuTensorMapEncodeTiled failed: %d / %d\n", sh.name, (int)enc, (int)enc_sw);
    return;
  }
  const size_t smem = 1024 + (size_t)sh.slots * slot + 2 * sh.slots * 8;
  cudaFuncSetAttribute(k_patch<NP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  const long patches = (long)B * ((W + 15) / 16) * ((H + 8 * sh.BY - 1) / (8 * sh.BY)) * ((C + sh.KC - 1) / sh.KC);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  double us[3];
  for (int mode = 0; mode < 3; ++mode) {
    const CUtensorMap& m = mode == 2 ? map_sw : map;
    k_patch<NP><<<sms, kThreads, smem>>>(m, in, B, H, W, C, sh.BY, sh.slots, sh.loaders, mode, check + mode);
    for (int r = 0; r < 3; ++r) k_patch<NP><<<sms, kThreads, smem>>>(m, in, B, H, W, C, sh.BY, sh.slots, sh.loaders, mode, nullptr);
    const int reps = 20;
    cudaEventRecord(e0);
    for (int r = 0; r < reps; ++r) k_patch<NP><<<sms, kThreads, smem>>>(m, in, B, H, W, C, sh.BY, sh.slots, sh.loaders, mode, nullptr);
    cudaEventRecord(e1);
    const cudaError_t e = cudaEventSynchronize(e1);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, e0, e1);
    us[mode] = ms * 1e3 / reps;
    printf("%-40s %-11s %8.1f us per launch  %6.3f us per patch and SM  %7.0f GB/s  %s\n", sh.name,
           mode == 2 ? "tma-sw" : mode ? "tma" : (sh.loaders == 128 ? "cp.async128" : "cp.async96"), us[mode],
           us[mode] * sms / patches, (double)patch_bytes * patches / (us[mode] * 1e-6) / 1e9, e == cudaSuccess ? "" : cudaGetErrorString(e));
  }
  unsigned h[3];
  cudaMemcpy(h, check, sizeof(h), cudaMemcpyDeviceToHost);
  printf("%-40s tma / cp.async %.3f, tma-sw / tma %.3f, staged bytes %s\n", sh.name, us[1] / us[0], us[2] / us[1],
         h[0] == h[1] && h[0] == h[2] ? "agree" : "DIFFER");
  cudaFree(in);
  cudaFree(check);
}
}  // namespace

int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  printf("%s, %d SMs\n", prop.name, sms);
  // form 2: 128 loader threads, 4 slots; form 3: 96 loader threads, 2 slots
  run<2>({"KC 16, 16x16 item, 512^2 x 16 (op 4)", 16, 2, 512, 16, 128, 4}, sms);
  run<4>({"KC 32, 16x16 item, 512^2 x 32 (op 5)", 32, 2, 512, 32, 128, 4}, sms);
  run<4>({"KC 32, 16x8 item, 256^2 x 32 (op 7)", 32, 1, 256, 32, 128, 4}, sms);
  run<8>({"KC 64, 16x8 item, 256^2 x 64 (ops 8, 26)", 64, 1, 256, 64, 128, 4}, sms);
  run<8>({"KC 64, 16x32 item, 256^2 x 128 (op 25)", 64, 4, 256, 128, 96, 2}, sms);
  run<8>({"KC 64, 16x16 item, 128^2 x 128 (form 3, N 128)", 64, 2, 128, 128, 96, 2}, sms);
  return 0;
}
