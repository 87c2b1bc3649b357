// Fused first encoder block of the UNet for sm_90a: raw frame -> conv0 (3x3, 1 -> 16, bias, ReLU) -> conv1 (3x3,
// 16 -> 16, bias, ReLU) -> MaxPool2D(2, 2) in one kernel.  Neither the 16-channel full-resolution tensor between the
// two convolutions nor conv1's own full-resolution output leaves the SM: per 8-frame C4 step that removes 268 MB of
// writes + 268 MB of reads of the intermediate and conv1's dead full-resolution stores.
//
// Replaces, for that block: InferenceLayer.preprocess (sleap/nn/inference.py:940-967, uint8 -> float * 1/255, zero
// pad to the stride) and the Keras layers stack0_enc0_conv0/act0, conv1/act1 and the pool of enc1
// (sleap/nn/architectures/encoder_decoder.py:94-144, unet.py:140-205), as dispatched to cuDNN by TensorFlow.
//
// Persistent and warp-specialized: one CTA per SM (as many as fit) walks a static list of (64x16-pixel tile of conv1's
// output, frame) items.  The conv1 bank, the conv0 weights and both biases are loaded once, before the grid-dependency
// wait.  Two roles hand conv0's output over through a ring of NSLOT plane slots with full / empty mbarriers:
//   * conv0 warpgroups (0, 1), on the CUDA cores: the 20x68 frame patch around the next item is fetched into registers
//     one item ahead and stored to shared memory as fp16-rounded pixels (zero outside the frame), double-buffered; conv0
//     for the 18x66 pixels conv1 reads is written once as fp16 into the slot's two non-swizzled 8-channel planes
//     [18][66][8] (16 bytes per pixel).  A named barrier among these 256 threads orders the patch buffers.
//   * the MMA warpgroup (2): conv1 as register-A wgmma over image rows.  An m64 block is the item's 64 pixels of one
//     output row.  Per plane row r, each warp loads three A fragments with ldmatrix.x4 (one per kx: +16 bytes on the row
//     addresses); each fragment feeds the ky = 0, 1, 2 taps of output rows r, r - 1, r - 2, whose accumulators rotate
//     through four sets.  Every A element is read from shared memory once, not once per tap.  Bias, ReLU, fp16 rounding
//     and the 2x2 max in registers: an even row's half2 values wait in registers for the odd row; the horizontal partner
//     is lane ^ 4.  Each warp store writes four whole pooled pixels (128 bytes).
// The same rounding points as the separate launches (fp16 frame pixels and weights, fp16 intermediate, fp16 conv1
// output before the pool), the same conv0 fma order, and every output pixel gets its nine wgmma products in (ky, kx)
// order on the same operand values as before: results are bit-identical to the 32x16 shared-A form this replaces.
#include <cuda.h>

#include <algorithm>

#include "sb_model.h"

namespace {

#include "sb_tc_prims.cuh"

constexpr int TW = 64, TH = 16;             // conv1 outputs per work item; TW = one wgmma M block
constexpr int CW0 = TW + 2, CH0 = TH + 2;   // conv0 pixels conv1 reads
constexpr int PW = TW + 4, PH = TH + 4;     // frame patch
constexpr int N_PATCH = PW * PH;
constexpr int N_C0 = CW0 * CH0;
constexpr int N_CONV0 = 256;                // conv0 threads (warpgroups 0, 1); the MMA warpgroup follows
constexpr int N_THREADS = N_CONV0 + 128;
constexpr int PATCH_PER_THREAD = (N_PATCH + N_CONV0 - 1) / N_CONV0;
constexpr int C0_PER_THREAD = (N_C0 + N_CONV0 / 2 - 1) / (N_CONV0 / 2);   // two threads per pixel, one per 8-channel half
constexpr int PLANE = N_C0 * 16;            // one 8-channel plane [CH0][CW0][8] fp16
constexpr int NSLOT = 3;                    // conv0 -> conv1 ring

constexpr int OFF_W1 = 0;                               // 9 taps x [16 co][16 ci] fp16, 32-byte swizzle
constexpr int OFF_A = OFF_W1 + 9 * 512;                 // NSLOT slots x 2 planes
constexpr int OFF_PATCH = OFF_A + NSLOT * 2 * PLANE;    // 2 buffers x [PH][PW] fp32
constexpr int OFF_BAR = OFF_PATCH + 2 * N_PATCH * 4;    // NSLOT full + NSLOT empty mbarriers
constexpr int SMEM_BYTES = OFF_BAR + 2 * NSLOT * 8 + 1024;
// plane stores of a quarter warp (4 pixels x 2 planes) and ldmatrix phases (8 consecutive pixels) are conflict-free
static_assert(PLANE % 128 == 64, "the two planes of a pixel must sit in different bank halves");

struct C01Params {
  const void* frames;
  int frames_u8;
  int Hin, Win, Hnet, Wnet, tiles_x, n_tiles, batch;
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

__device__ __forceinline__ void conv0_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(N_CONV0) : "memory"); }

template <typename TI>
__global__ void __launch_bounds__(N_THREADS, 1) k_conv01(const __grid_constant__ C01Params P) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // 1024-byte aligned by offsetting the array itself, so that the compiler keeps every access in the shared window
  uint8_t* base = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  const int tid = threadIdx.x;
  const int n_items = P.n_tiles * P.batch, G = gridDim.x;
  const uint32_t full0 = smem_u32(base + OFF_BAR), empty0 = full0 + 8 * NSLOT;

  // static operands, loaded while the predecessor drains
  for (int i = tid; i < 9 * 16 * 2; i += N_THREADS) {   // conv1 bank: 9 taps x 16 rows x 2 chunks
    const int t = i >> 5, r = (i >> 1) & 15, c = i & 1;
    *reinterpret_cast<uint4*>(base + OFF_W1 + t * 512 + sw32(r, c)) = reinterpret_cast<const uint4*>(P.w1t + (t * 16 + r) * 16)[c];
  }
  if (tid == 0)
    for (int s = 0; s < NSLOT; ++s) {
      mbar_init(full0 + 8 * s, N_CONV0);
      mbar_init(empty0 + 8 * s, 128);
    }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the conv1 bank -> visible to wgmma
  __syncthreads();

  if (tid < N_CONV0) {
    // ---- conv0 warpgroups: frame patch and conv0 of every item of this CTA into the plane ring ----
    const int hc = tid & 1;                             // this thread's 8-channel half (fixed: two threads per pixel)
    float w0[9][8], b0[8];
#pragma unroll
    for (int t = 0; t < 9; ++t)
#pragma unroll
      for (int c = 0; c < 8; ++c) w0[t][c] = P.w0h[t * 16 + 8 * hc + c];
#pragma unroll
    for (int c = 0; c < 8; ++c) b0[c] = P.bias0 ? P.bias0[8 * hc + c] : 0.f;
    float* s_patch = reinterpret_cast<float*>(base + OFF_PATCH);
    griddep_wait();                                     // frames belong to the stream's order

    const float sc = P.frames_u8 ? (1.0f / 255.0f) : 1.0f;     // ensure_float (normalization.py:34-49)
    TI pf[PATCH_PER_THREAD];
    auto fetch = [&](int w) {                           // frame patch of item w -> registers (zero outside the frame)
      const int tile = w % P.n_tiles, b = w / P.n_tiles;
      const int x0 = (tile % P.tiles_x) * TW, y0 = (tile / P.tiles_x) * TH;
      const TI* img = reinterpret_cast<const TI*>(P.frames) + (size_t)b * P.Hin * P.Win;
#pragma unroll
      for (int k = 0; k < PATCH_PER_THREAD; ++k) {
        const int e = tid + N_CONV0 * k;
        const int y = y0 - 2 + e / PW, x = x0 - 2 + e % PW;
        pf[k] = (w < n_items && e < N_PATCH && y >= 0 && y < P.Hin && x >= 0 && x < P.Win) ? img[(size_t)y * P.Win + x] : TI(0);
      }
    };
    auto stash = [&](float* dst) {
#pragma unroll
      for (int k = 0; k < PATCH_PER_THREAD; ++k)
        if (tid + N_CONV0 * k < N_PATCH) dst[tid + N_CONV0 * k] = __half2float(__float2half_rn(__fmul_rn((float)pf[k], sc)));
    };
    // conv0 for the CH0 x CW0 pixels conv1 reads, 8 channels per thread; zero outside the network image (conv1's SAME pad)
    auto conv0 = [&](const float* patch, uint8_t* A, int x0, int y0) {
#pragma unroll 1
      for (int k = 0; k < C0_PER_THREAD; ++k) {
        const int p = (tid >> 1) + (N_CONV0 / 2) * k;
        if (p >= N_C0) break;
        const int yy = p / CW0, cx = p % CW0;
        const int y = y0 - 1 + yy, x = x0 - 1 + cx;
        uint32_t q[4] = {0u, 0u, 0u, 0u};               // fp16 +0 outside
        if (y >= 0 && y < P.Hnet && x >= 0 && x < P.Wnet) {
          float acc[8];
#pragma unroll
          for (int c = 0; c < 8; ++c) acc[c] = 0.f;
#pragma unroll
          for (int ky = 0; ky < 3; ++ky)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {
              const float v = patch[(yy + ky) * PW + cx + kx];
#pragma unroll
              for (int c = 0; c < 8; ++c) acc[c] = fmaf(v, w0[ky * 3 + kx][c], acc[c]);
            }
#pragma unroll
          for (int c = 0; c < 8; ++c) {
            acc[c] += b0[c];
            if (P.relu0) acc[c] = fmaxf(acc[c], 0.f);
          }
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const __half2 t = __floats2half2_rn(acc[2 * c], acc[2 * c + 1]);
            q[c] = *reinterpret_cast<const uint32_t*>(&t);
          }
        }
        *reinterpret_cast<uint4*>(A + hc * PLANE + p * 16) = make_uint4(q[0], q[1], q[2], q[3]);
      }
    };

    int w = blockIdx.x;
    fetch(w);
    stash(s_patch);
    fetch(w + G);
    conv0_bar_sync();
    for (int k = 0; w < n_items; ++k, w += G) {
      if (w + G >= n_items) griddep_launch();           // last item of this CTA
      const int slot = k % NSLOT, use = k / NSLOT;
      if (use > 0) mbar_wait(empty0 + 8 * slot, (use - 1) & 1);   // the MMA warpgroup has read the slot's last item
      const int tile = w % P.n_tiles;
      conv0(s_patch + (k & 1) * N_PATCH, base + OFF_A + slot * 2 * PLANE, (tile % P.tiles_x) * TW, (tile / P.tiles_x) * TH);
      mbar_arrive(full0 + 8 * slot);
      // patch[k & 1] was last read by conv0 above; patch[(k + 1) & 1]'s last reader, conv0 of item k - 1, finished
      // before the previous barrier
      stash(s_patch + ((k + 1) & 1) * N_PATCH);
      fetch(w + 2 * G);
      conv0_bar_sync();
    }
    return;
  }

  // ---- MMA warpgroup: conv1 + bias + ReLU + pool of every item of this CTA ----
  const int ctid = tid - N_CONV0, warp = ctid >> 5, lane = ctid & 31;
  const int g = lane >> 2, odd = g & 1, fc = 2 * (lane & 3);
  float b1[2][2];
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int e = 0; e < 2; ++e) b1[j][e] = P.bias1 ? P.bias1[8 * j + fc + e] : 0.f;
  const uint64_t desc_b = make_desc(0, 32, 3) + (uint64_t)(smem_u32(base + OFF_W1) >> 4);
  // ldmatrix row address of this lane in plane row 0, kx = 0: pixel 16 warp + lane % 16, 8-channel plane lane / 16
  const uint32_t a_lane = smem_u32(base + OFF_A) + (uint32_t)((lane >> 4) * PLANE + (16 * warp + (lane & 15)) * 16);
  griddep_wait();                                       // the pooled buffer belongs to the stream's order

  float acc[4][8];                                      // output row y accumulates in set y % 4
  uint32_t fr[3][3][4];                                 // A fragments of plane row r in set r % 3, one per kx
  __half2 even[2][2];                                   // an even output row's values (channel group j, pixel half a)

  // bias, ReLU, fp16 rounding (conv1's stored value) of output row y, then for an odd row the 2x2 max with the row above.
  // Thread pixels: 16 warp + g + 8 a, a = 0, 1; the even column of a pair pools channels 0-7, the odd one 8-15, after
  // trading the other half with lane ^ 4.
  auto epilogue = [&](int y, const float (&d)[8], __half* pool_row, int gx0) {
    auto val = [&](int j, int a) {                      // conv1 output of channel pair (8 j + fc, + 1), pixel half a
      float v0 = d[4 * j + 2 * a] + b1[j][0], v1 = d[4 * j + 2 * a + 1] + b1[j][1];
      if (P.relu1) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
      return __floats2half2_rn(v0, v1);
    };
    if ((y & 1) == 0) {
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int a = 0; a < 2; ++a) even[j][a] = val(j, a);
      return;
    }
#pragma unroll
    for (int a = 0; a < 2; ++a) {
      const __half2 o0 = val(0, a), o1 = val(1, a);
      const __half2 mine0 = odd ? even[1][a] : even[0][a], mine1 = odd ? o1 : o0;
      const __half2 theirs0 = __shfl_xor_sync(0xffffffffu, odd ? even[0][a] : even[1][a], 4);
      const __half2 theirs1 = __shfl_xor_sync(0xffffffffu, odd ? o0 : o1, 4);
      __half2 m = __float2half2_rn(-INFINITY);          // order (row, column) = (0, 0), (0, 1), (1, 0), (1, 1)
      m = __hmax2(m, odd ? theirs0 : mine0);
      m = __hmax2(m, odd ? mine0 : theirs0);
      m = __hmax2(m, odd ? theirs1 : mine1);
      m = __hmax2(m, odd ? mine1 : theirs1);
      const int gx = gx0 + 4 * a;
      if (pool_row && gx < P.pool_W) *reinterpret_cast<__half2*>(pool_row + (size_t)gx * P.pool_Ctot) = m;
    }
  };

  int w = blockIdx.x;
  for (int k = 0; w < n_items; ++k, w += G) {
    if (w + G >= n_items) griddep_launch();             // last item of this CTA
    const int slot = k % NSLOT;
    mbar_wait(full0 + 8 * slot, (k / NSLOT) & 1);
    const uint32_t a0 = a_lane + (uint32_t)(slot * 2 * PLANE);
    const int tile = w % P.n_tiles, b = w / P.n_tiles;
    const int x0 = (tile % P.tiles_x) * TW, y0 = (tile / P.tiles_x) * TH;
    const int gx0 = (x0 >> 1) + 8 * warp + (g >> 1);
    __half* pool_img = P.pool_out + (size_t)b * P.pool_H * P.pool_W * P.pool_Ctot + P.pool_coff + 8 * odd + fc;
    auto row_of = [&](int y) -> __half* {               // pooled row of output row y (nullptr below the map)
      const int gy = (y0 + y) >> 1;
      return gy < P.pool_H ? pool_img + (size_t)gy * P.pool_W * P.pool_Ctot : nullptr;
    };
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) ldmatrix_x4(fr[0][kx], a0 + 16 * kx);
#pragma unroll
    for (int r = 0; r < CH0; ++r) {
      // group r: plane row r's fragments into the ky = 0, 1, 2 taps of output rows r, r - 1, r - 2
      wgmma_fence();
#pragma unroll
      for (int s = 0; s < 4; ++s) wgmma_reg_fence(acc[s]);
#pragma unroll
      for (int ky = 0; ky < 3; ++ky) {
        const int y = r - ky;
        if (y < 0 || y >= TH) continue;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx)
          wgmma_f16_rs16(acc[y & 3], fr[r % 3][kx], desc_b + 32 * (ky * 3 + kx), (ky | kx) ? 1u : 0u);
      }
      wgmma_commit();
      if (r + 1 < CH0) {
        // set (r + 1) % 3 was last read by group r - 2, complete since the previous wait
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) ldmatrix_x4(fr[(r + 1) % 3][kx], a0 + (uint32_t)((r + 1) * CW0 * 16) + 16 * kx);
      } else {
        mbar_arrive(empty0 + 8 * slot);                 // every ldmatrix of this slot has returned
      }
#pragma unroll
      for (int s = 0; s < 4; ++s) wgmma_reg_fence(acc[s]);
      wgmma_wait<1>();                                  // groups <= r - 1 done: output row r - 3 is complete
      if (r >= 3) {
        wgmma_reg_fence(acc[(r - 3) & 3]);
        epilogue(r - 3, acc[(r - 3) & 3], row_of(r - 3), gx0);
      }
    }
    wgmma_wait<0>();
    wgmma_reg_fence(acc[(TH - 1) & 3]);
    epilogue(TH - 1, acc[(TH - 1) & 3], row_of(TH - 1), gx0);
  }
}

}  // namespace

struct SbConv01Plan {
  C01Params P;
  __half* w1t = nullptr;     // [9][16][16]
  float* w0h = nullptr;      // [9][16]
  int max_ctas = 0;          // co-resident CTAs of k_conv01 on this GPU
};

void sb_conv01_release(SbModel* m) {
  SbConv01Plan*& pl = m->entry.conv01;
  if (!pl) return;
  if (pl->w1t) cudaFree(pl->w1t);
  if (pl->w0h) cudaFree(pl->w0h);
  delete pl;
  pl = nullptr;
}

// The parameters of k_conv01 over conv0_op -> conv1_op -> pool, a block the input stage found it takes (sb_entry.cu).
int sb_conv01_prepare(sb_handle_s* h, SbModel* m, int conv0_op, int conv1_op) {
  const SbOp& c0 = m->ops[conv0_op];
  const SbOp& c1 = m->ops[conv1_op];
  const SbBuffer& ob0 = m->buffers[c0.out_buf()];
  const SbBuffer& pb = m->buffers[c1.pool_buf()];
  SbConv01Plan* pl = new SbConv01Plan();
  for (auto kern : {k_conv01<unsigned char>, k_conv01<float>}) {
    int nb = 0;
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES) != cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kern, N_THREADS, SMEM_BYTES) != cudaSuccess || nb < 1) {
      delete pl;
      return sb_fail(h, SB_ERR_CUDA, "conv01: kernel attributes / occupancy: %s", cudaGetErrorString(cudaGetLastError()));
    }
    pl->max_ctas = pl->max_ctas ? std::min(pl->max_ctas, nb * h->sm_count) : nb * h->sm_count;
  }
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
  m->entry.conv01 = pl;                                    // released with the model from here on
  if (cudaMemcpy(pl->w1t, w1t.data(), w1t.size() * 2, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(pl->w0h, w0h.data(), w0h.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess) {
    sb_conv01_release(m);
    return sb_fail(h, SB_ERR_CUDA, "conv01: weight copy");
  }
  C01Params& P = pl->P;
  memset(&P, 0, sizeof(P));
  P.Hin = m->Hin; P.Win = m->Win; P.Hnet = ob0.H; P.Wnet = ob0.W;
  P.tiles_x = (ob0.W + TW - 1) / TW;
  P.n_tiles = P.tiles_x * ((ob0.H + TH - 1) / TH);
  P.pool_out = (__half*)pb.dev; P.pool_H = pb.H; P.pool_W = pb.W; P.pool_Ctot = pb.C; P.pool_coff = c1.pool_coff();
  P.bias0 = c0.b_off() >= 0 ? m->weights_dev + c0.b_off() : nullptr;
  P.bias1 = c1.b_off() >= 0 ? m->weights_dev + c1.b_off() : nullptr;
  P.w0h = pl->w0h; P.w1t = pl->w1t;
  P.relu0 = (c0.flags() & SB_OPF_RELU) ? 1 : 0;
  P.relu1 = (c1.flags() & SB_OPF_RELU) ? 1 : 0;
  return 0;
}

// Persistent launch: as many CTAs as are co-resident (capped at the item count), with programmatic stream serialization
// so that the weight loads overlap the predecessor's tail; each CTA triggers its dependents when it starts its last item.
int sb_conv01_launch(sb_handle_s* h, const SbConv01Plan* pl, const void* frames_dev, int frames_are_u8, int B) {
  C01Params P = pl->P;
  P.frames = frames_dev; P.frames_u8 = frames_are_u8; P.batch = B;
  void* args[] = {&P};
  sb_launch_pdl(frames_are_u8 ? (const void*)k_conv01<unsigned char> : (const void*)k_conv01<float>,
                dim3(std::min(P.n_tiles * B, pl->max_ctas)), dim3(N_THREADS), SMEM_BYTES, h->stream, args);
  SB_CHECK_LAUNCH(h);
  return 0;
}
