// Issue rate of the wgmma groups the conv kernel forms run, with every operand already in shared memory: no loads, no
// barriers, no epilogue.  One CTA per SM, two warpgroups, each issuing per "slice" KSTEPS = 4 k-steps x BLOCKS m64 blocks
// of m64nNk16 as one group and waiting with wgmma.wait_group 1, as k_conv_wg (form 0) and k_conv_wg_hw (form 3) do.
// A is one of
//   box   the 128B-swizzled box of form 0 (tap (0, 0) only: form 0 loads one box per tap);
//   il    a halo patch of 8-channel planes [rows][18][8] (non-swizzled, LBO = one plane, SBO = one patch row), the layout
//         forms 2 / 3 used before the swizzled patch;
//   sw    a halo patch of 128-byte pixel rows [rows][18][64 ch], 128B-swizzled as TMA writes it (SBO = one patch row),
//         the layout of forms 2 / 3;
// and for the patches slice s issues tap s mod 9 (kx outer, ky inner) at every block of the warpgroup, as form 3 does.
// B is a 128B-swizzled [N x 64] weight slice.
//
// Before the rates, a probe checks the swizzled patch descriptor bit for bit: for SW128 / SW64 / SW32 (KC 64 / 32 / 16
// channels per pixel row) and a 34 x 18-pixel patch, every tap of every 8x8 block of a 16x32 item and every k-step runs
// one m64n64k16 from the swizzled patch and one from the 8-channel planes holding the same seeded values; all 32
// accumulators of all 128 threads must agree.  Two encodings of the descriptor's matrix base offset (bits 49-51) are
// tried: 0, and (start >> 7) & (pattern bytes / 128 - 1).
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o /tmp/wgmma_rate tools/wgmma_rate.cu -lcuda && /tmp/wgmma_rate
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <cstdio>
#include <cstdint>
#include <type_traits>

namespace {
#include "../sleap_b200/csrc/sb_tc_prims.cuh"

// Non-swizzled K-major descriptor (layout type 0) with explicit offsets.  The operand is built from 8-row x 16-byte core
// matrices whose rows are 16 bytes apart; lbo = distance between the two core matrices of one K = 16 step, sbo = distance
// between successive 8-row groups along M / N.  The start address only needs 16-byte alignment.
__device__ __forceinline__ uint64_t make_desc_interleave(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo >> 4) & 0x3FFF) << 32;
  return d;
}

constexpr int kSmem = 160 * 1024;            // more than half the SM: one CTA per SM
enum { kBox = 0, kIl = 1, kSw = 2 };

// swizzled K-major descriptor of a patch: 8-row groups one patch row (sbo bytes) apart, base offset field as encoded
__device__ __forceinline__ uint64_t patch_desc(uint32_t start, int layout_type, uint32_t sbo, int enc) {
  uint64_t d = ((uint64_t)((start >> 4) & 0x3FFF)) | ((uint64_t)1 << 16) | ((uint64_t)((sbo >> 4) & 0x3FFF) << 32) |
               ((uint64_t)layout_type << 62);
  if (enc) d |= (uint64_t)((start >> 7) & ((layout_type == 1 ? 8 : layout_type == 2 ? 4 : 2) - 1)) << 49;
  return d;
}

template <int N, int BLOCKS, int A>
__global__ void __launch_bounds__(256, 1) k_rate(int slices, int enc, float* sink) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int ROWS = 8 * BLOCKS + 2;       // patch rows of the item: BLOCKS / 2 block rows per warpgroup
  constexpr int PLANE = ROWS * 18 * 16;      // il: one 8-channel plane
  uint8_t* a = base;                         // box: BLOCKS x 2 warpgroups x 8 KB swizzled rows; il / sw: one patch (<= 77 KB)
  uint8_t* b = base + 80 * 1024;             // [N x 64] swizzled weight slice
  // non-trivial operand values (the tensor pipe's power, hence its clock, depends on them)
  for (int i = threadIdx.x; i < 40 * 1024 + N * 64; i += blockDim.x)
    reinterpret_cast<__half*>(base)[i] = __float2half(0.01f * (float)((i * 7) % 13 - 6));
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  const int wg = threadIdx.x >> 7;
  const uint64_t db = make_desc(0, 128, 1) + (uint64_t)(smem_u32(b) >> 4);
  const uint32_t a0 = smem_u32(a);
  float acc[BLOCKS][N / 2];
#pragma unroll
  for (int i = 0; i < BLOCKS; ++i)
#pragma unroll
    for (int j = 0; j < N / 2; ++j) acc[i][j] = 0.f;
  auto slice = [&](int kx, int ky) {
    wgmma_fence();
#pragma unroll
    for (int i = 0; i < BLOCKS; ++i) wgmma_reg_fence(acc[i]);
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int i = 0; i < BLOCKS; ++i) {
        // block (row wg * BLOCKS / 2 + i / 2, column i % 2) of the patch
        const int px = (8 * (wg * (BLOCKS / 2) + (i >> 1)) + ky) * 18 + 8 * (i & 1) + kx;
        uint64_t da;
        if (A == kIl) da = make_desc_interleave(0, PLANE, 18 * 16) + (uint64_t)((a0 + (uint32_t)(px * 16 + 2 * k * PLANE)) >> 4);
        else if (A == kSw) da = patch_desc(a0 + (uint32_t)(px * 128 + 32 * k), 1, 18 * 128, enc);
        else da = make_desc(0, 128, 1) + (uint64_t)((a0 + (uint32_t)((wg * BLOCKS + i) * 8192)) >> 4) + 2 * k;
        wgmma_f16<N>(acc[i], da, db + 2 * k, 1u);
      }
    wgmma_commit();
#pragma unroll
    for (int i = 0; i < BLOCKS; ++i) wgmma_reg_fence(acc[i]);
    wgmma_wait<1>();
  };
  for (int s = 0; s < slices; s += 9)
#pragma unroll
    for (int kx = 0; kx < 3; ++kx)
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) slice(A == kBox ? 0 : kx, A == kBox ? 0 : ky);
  wgmma_wait<0>();
  float t = 0.f;
#pragma unroll
  for (int i = 0; i < BLOCKS; ++i)
#pragma unroll
    for (int j = 0; j < N / 2; ++j) t += acc[i][j];
  if (t == 12345.f) sink[threadIdx.x] = t;
}

// The probe: one warpgroup; a [34][18][KC] patch with seeded values as 8-channel planes (il) and as swizzled KC-channel
// pixel rows (sw, pattern-aligned), a seeded [64 x KC] B in the same swizzle.  bad[case] counts the threads whose
// accumulators differ; case = ((tap * 8 + block) * KSTEPS + k), tap = kx * 3 + ky.
template <int KC>
__global__ void __launch_bounds__(128, 1) k_probe(int enc, unsigned seed, int* bad) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* base = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  constexpr int ROWS = 34, PX = ROWS * 18, RB = KC * 2, KSTEPS = KC / 16, PLANE = PX * 16;
  constexpr int LT = KC == 64 ? 1 : KC == 32 ? 2 : 3, MASK = KC == 64 ? 7 : KC == 32 ? 3 : 1;
  constexpr int PBYTES = (PX * RB + 1023) / 1024 * 1024;
  uint8_t* il = base;
  uint8_t* sw = base + PBYTES;
  uint8_t* bs = sw + PBYTES;
  auto swz = [](uint32_t off) { return off ^ (((off >> 7) & MASK) << 4); };
  auto val = [&](uint32_t i) {
    uint32_t h = (i + 1) * 2654435761u ^ seed;
    h ^= h >> 15; h *= 2246822519u; h ^= h >> 13;
    return __float2half((float)((int)(h & 2047) - 1024) / 1024.f);
  };
  for (int i = threadIdx.x; i < PX * KC; i += blockDim.x) {
    const int p = i / KC, c = i % KC;
    const __half v = val(i);
    *reinterpret_cast<__half*>(il + (c / 8) * PLANE + p * 16 + (c % 8) * 2) = v;
    *reinterpret_cast<__half*>(sw + swz((uint32_t)(p * RB + c * 2))) = v;
  }
  for (int i = threadIdx.x; i < 64 * KC; i += blockDim.x)
    *reinterpret_cast<__half*>(bs + swz((uint32_t)((i / KC) * RB + (i % KC) * 2))) = val(0x40000000u + i);
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  const uint64_t db = make_desc(smem_u32(bs), RB, LT);
  for (int tap = 0; tap < 9; ++tap)
    for (int bk = 0; bk < 8; ++bk)
      for (int k = 0; k < KSTEPS; ++k) {
        const int kx = tap / 3, ky = tap % 3;
        const int px = (8 * (bk >> 1) + ky) * 18 + 8 * (bk & 1) + kx;
        const uint64_t d_il = make_desc_interleave(0, PLANE, 18 * 16) + (uint64_t)((smem_u32(il) + (uint32_t)(px * 16 + 2 * k * PLANE)) >> 4);
        const uint64_t d_sw = patch_desc(smem_u32(sw) + (uint32_t)(px * RB + 32 * k), LT, 18 * RB, enc);
        float x[32], y[32];
        wgmma_fence();
        wgmma_f16<64>(x, d_il, db + 2 * k, 0u);
        wgmma_f16<64>(y, d_sw, db + 2 * k, 0u);
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_reg_fence(x);
        wgmma_reg_fence(y);
        bool diff = false;
#pragma unroll
        for (int j = 0; j < 32; ++j) diff |= __float_as_uint(x[j]) != __float_as_uint(y[j]);
        if (diff) atomicAdd(bad + (tap * 8 + bk) * KSTEPS + k, 1);
      }
}

template <int KC>
bool probe(int enc) {
  constexpr int KSTEPS = KC / 16, CASES = 9 * 8 * KSTEPS;
  const int smem = 1024 + 2 * ((34 * 18 * KC * 2 + 1023) / 1024 * 1024) + 64 * KC * 2;
  cudaFuncSetAttribute(k_probe<KC>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  int* bad;
  cudaMalloc(&bad, CASES * sizeof(int));
  cudaMemset(bad, 0, CASES * sizeof(int));
  for (unsigned seed = 1; seed <= 2; ++seed) k_probe<KC><<<1, 128, smem>>>(enc, seed * 0x9E3779B9u, bad);
  const cudaError_t e = cudaDeviceSynchronize();
  int h[CASES];
  cudaMemcpy(h, bad, sizeof(h), cudaMemcpyDeviceToHost);
  cudaFree(bad);
  int cases_bad = 0, tap_bad[9] = {};
  for (int c = 0; c < CASES; ++c)
    if (h[c]) { ++cases_bad; ++tap_bad[c / (8 * KSTEPS)]; }
  printf("probe SW%-3d (KC %2d) base offset %-22s %3d of %3d (tap, block, k-step) cases differ; per tap (kx ky):",
         2 * KC, KC, enc ? "(start >> 7) & (rows-1):" : "0:", cases_bad, CASES);
  for (int t = 0; t < 9; ++t) printf(" %d%d:%d", t / 3, t % 3, tap_bad[t]);
  printf("  %s\n", e == cudaSuccess ? (cases_bad ? "DIFFER" : "match") : cudaGetErrorString(e));
  return e == cudaSuccess && cases_bad == 0;
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
void time_kernel(K kern, const char* name, int sms, double flop_per_slice_cta, int enc = -1) {
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
  float* sink;
  cudaMalloc(&sink, 1024 * sizeof(float));
  const int slices = 4104;             // a multiple of the nine-tap loop and of the RS loop's unroll by 3
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  auto launch = [&]() {
    if constexpr (std::is_invocable_v<K, int, int, float*>) kern<<<sms, 256, kSmem>>>(slices, enc, sink);
    else kern<<<sms, 256, kSmem>>>(slices, sink);
  };
  for (int w = 0; w < 3; ++w) launch();
  cudaEventRecord(e0);
  const int reps = 40;
  for (int r = 0; r < reps; ++r) launch();
  cudaEventRecord(e1);
  cudaError_t e = cudaEventSynchronize(e1);
  float ms = 0.f;
  cudaEventElapsedTime(&ms, e0, e1);
  const double flop = flop_per_slice_cta * (double)slices * sms * reps;
  printf("%-52s %7.1f TFLOP/s  %6.3f us per slice and CTA  %s\n", name, flop / (ms * 1e-3) / 1e12,
         ms * 1e3 / reps / slices, e == cudaSuccess ? "" : cudaGetErrorString(e));
  cudaFree(sink);
}

template <int N, int BLOCKS, int A>
void run(const char* name, int sms, int enc = 0) {
  time_kernel(k_rate<N, BLOCKS, A>, name, sms, 2.0 * 64 * N * 16 * 4 * BLOCKS * 2, enc);
}

template <bool RS, int NACC, int WGS>
void run16(const char* name, int sms) {
  time_kernel(k_rate16<RS, NACC, WGS>, name, sms, 2.0 * 64 * 16 * 16 * 9 * WGS);
}
}  // namespace

int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  printf("%s, %d SMs\n", prop.name, sms);
  bool ok[2];
  for (int enc = 0; enc < 2; ++enc) ok[enc] = probe<64>(enc) & probe<32>(enc) & probe<16>(enc);
  const int enc = ok[0] ? 0 : 1;       // the rates below use the first encoding that matched (0 if none did)
  printf("base offset encoding %d used for the sw rates%s\n", enc, ok[0] || ok[1] ? "" : " (NEITHER MATCHED)");
  run<128, 1, kBox>("N 128, 1 block / wg, box A, tap (0, 0) (form 0)", sms);
  run<128, 2, kBox>("N 128, 2 blocks / wg, box A, tap (0, 0)", sms);
  run<128, 2, kIl>("N 128, 2 blocks / wg, il patch A, nine taps", sms);
  run<128, 2, kSw>("N 128, 2 blocks / wg, sw patch A, nine taps (form 3)", sms, enc);
  run<256, 1, kBox>("N 256, 1 block / wg, box A, tap (0, 0) (form 0)", sms);
  run<64, 4, kBox>("N 64, 4 blocks / wg, box A, tap (0, 0)", sms);
  run<64, 4, kIl>("N 64, 4 blocks / wg, il patch A, nine taps", sms);
  run<64, 4, kSw>("N 64, 4 blocks / wg, sw patch A, nine taps (form 3)", sms, enc);
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
