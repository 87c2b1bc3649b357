// The input stage: everything from the raw frame to the first activation the generic op loop reads.  One of five routes
// (SbEntryPlan) takes the PREPROCESS op and the first conv, and the fused first encoder block k_conv01 may take conv1
// too.  sb_entry_prepare resolves the route from the op list and builds its views, sb_entry_autotune times the
// candidates once at configure time, and sb_entry_build fills the slots the plan covers in both programs.
//
// Replaces InferenceLayer.preprocess (sleap/nn/inference.py:940-967, uint8 -> float * 1/255, zero pad to the stride)
// fused with the first conv of the backbone (encoder_decoder.py:117-131; hourglass.py:49-100; resnet.py's stem).
#include <algorithm>

#include "sb_model.h"

// ---- first layer fused with preprocessing on the CUDA cores ------------------------------------------------------
// For the common case "no channel conversion, no resize": raw uint8 (or float) frame -> * (1/255) -> zero pad to the
// net size -> 3x3 SAME conv + bias + ReLU -> fp16 NHWC.  One output pixel per thread, all COUT channels in registers;
// the frame is read once from HBM (neighbour re-reads hit L1), the output is written once, so the kernel runs at HBM
// speed instead of paying a separate preprocess pass.
template <typename TI, int CIN, int COUT, int PX>
__global__ void __launch_bounds__(256) k_conv_first(const TI* __restrict__ img, int Hin, int Win, int Hnet, int Wnet,
                                                    __half* __restrict__ out, int out_Ctot, int out_coff,
                                                    const float* __restrict__ w /*[9][CIN][COUT]*/,
                                                    const float* __restrict__ bias, int relu, int in_is_u8, int split = 0) {
  // each thread: PX horizontally adjacent output pixels x COUT channels (weights read once from
  // shared memory per PX pixels; the thread's PX*COUT fp16 outputs are contiguous in NHWC)
  __shared__ __align__(16) float s_w[9 * CIN * COUT];
  __shared__ float s_b[COUT];
  for (int t = threadIdx.y * 32 + threadIdx.x; t < 9 * CIN * COUT; t += 256) s_w[t] = w[t];
  for (int t = threadIdx.y * 32 + threadIdx.x; t < COUT; t += 256) s_b[t] = bias ? bias[t] : 0.f;
  __syncthreads();
  const int ox0 = (blockIdx.x * 32 + threadIdx.x) * PX, oy = blockIdx.y * 8 + threadIdx.y, b = blockIdx.z;
  if (ox0 >= Wnet || oy >= Hnet) return;
  const TI* im = img + (size_t)b * Hin * Win * CIN;
  const float sc = in_is_u8 ? (1.0f / 255.0f) : 1.0f;
  float acc[PX][COUT];
#pragma unroll
  for (int p = 0; p < PX; ++p)
#pragma unroll
    for (int c = 0; c < COUT; ++c) acc[p][c] = s_b[c];
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int iy = oy + ky - 1;
    if (iy < 0 || iy >= Hin) continue;                       // SAME padding / bottom zero pad
    float in[PX + 2][CIN];
#pragma unroll
    for (int j = 0; j < PX + 2; ++j) {
      const int ix = ox0 + j - 1;
      const bool ok = ix >= 0 && ix < Win;
#pragma unroll
      for (int ci = 0; ci < CIN; ++ci)
        in[j][ci] = ok ? __fmul_rn((float)im[((size_t)iy * Win + ix) * CIN + ci], sc) : 0.f;
    }
#pragma unroll
    for (int kx = 0; kx < 3; ++kx)
#pragma unroll
      for (int ci = 0; ci < CIN; ++ci) {
        const float4* w4 = reinterpret_cast<const float4*>(s_w + ((ky * 3 + kx) * CIN + ci) * COUT);
#pragma unroll
        for (int q = 0; q < COUT / 4; ++q) {
          const float4 ww = w4[q];
#pragma unroll
          for (int p = 0; p < PX; ++p) {
            const float v = in[p + kx][ci];
            acc[p][4 * q + 0] = fmaf(v, ww.x, acc[p][4 * q + 0]);
            acc[p][4 * q + 1] = fmaf(v, ww.y, acc[p][4 * q + 1]);
            acc[p][4 * q + 2] = fmaf(v, ww.z, acc[p][4 * q + 2]);
            acc[p][4 * q + 3] = fmaf(v, ww.w, acc[p][4 * q + 3]);
          }
        }
      }
  }
#pragma unroll
  for (int p = 0; p < PX; ++p) {
    if (ox0 + p >= Wnet) break;
    __half* po = out + (((size_t)b * Hnet + oy) * Wnet + ox0 + p) * out_Ctot + out_coff;
    if (split) {                                             // precision 2: [lo | hi | hi] planes, COUT channels apart
#pragma unroll
      for (int q = 0; q < COUT / 8; ++q) {
        __align__(16) __half hh[8], ll[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float a = acc[p][8 * q + j];
          if (relu) a = fmaxf(a, 0.f);
          hh[j] = __float2half_rn(a);
          ll[j] = __float2half_rn(a - __half2float(hh[j]));
        }
        reinterpret_cast<uint4*>(po)[q] = *reinterpret_cast<uint4*>(ll);
        reinterpret_cast<uint4*>(po + COUT)[q] = *reinterpret_cast<uint4*>(hh);
        reinterpret_cast<uint4*>(po + 2 * COUT)[q] = *reinterpret_cast<uint4*>(hh);
      }
      continue;
    }
#pragma unroll
    for (int q = 0; q < COUT / 8; ++q) {
      __align__(16) __half2 h[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float a = acc[p][8 * q + 2 * j], c2 = acc[p][8 * q + 2 * j + 1];
        if (relu) { a = fmaxf(a, 0.f); c2 = fmaxf(c2, 0.f); }
        h[j] = __floats2half2_rn(a, c2);
      }
      reinterpret_cast<uint4*>(po)[q] = *reinterpret_cast<uint4*>(h);
    }
  }
}

// ---- first layer (1 input channel, 3x3) as a Toeplitz GEMM over groups of 8 output pixels ----------
// out[y][8g+j][co] = sum_{ky,kx} in[y+ky-1][8g+j+kx-1] * w[ky][kx][co]   (SAME padding)
// With G[y][g][c] = in[y][8g-1+c] (c = 0..9; c = 10..15 zero) the layer is an ordinary 3x1 convolution
// over the [H][W/8] grid of groups with 16 "input channels" (the window) and 8*Cout "output channels"
// (pixel j of the group x filter co): W'[ky][j*Cout+co][c] = w[ky][c-j][co] for 0 <= c-j <= 2.  The
// output [H][W/8][8*Cout] is byte-identical to NHWC [H][W][Cout], so the stock wgmma conv kernel runs
// it unchanged: each epilogue thread writes 8 pixels (8*Cout*2 contiguous bytes) instead of gathering a
// 3x3 neighbourhood per pixel, which is what bounds the CUDA-core k_conv_first.  Tensor work grows 3.5x (16x8*Cout
// MACs per tap row instead of 9*Cout per pixel) on a pipe that is otherwise idle in this layer.
template <typename TI>
__global__ void __launch_bounds__(256) k_first_view(const TI* __restrict__ img, int Hin, int Win, int Hnet, int Wg,
                                                    __half* __restrict__ G, int in_is_u8, size_t total) {
  const float sc = in_is_u8 ? (1.0f / 255.0f) : 1.0f;       // ensure_float (normalization.py:34-49)
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (size_t)gridDim.x * 256) {
    const int g = (int)(i % Wg);
    const size_t r = i / Wg;
    const int y = (int)(r % Hnet), b = (int)(r / Hnet);
    __align__(16) __half v[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) v[c] = __float2half_rn(0.f);
    if (y < Hin) {                                           // rows below the frame: bottom zero pad (resizing.py:34-68)
      const TI* row = img + ((size_t)b * Hin + y) * Win;
#pragma unroll
      for (int c = 0; c < 10; ++c) {
        const int x = 8 * g - 1 + c;
        if (x >= 0 && x < Win) v[c] = __float2half_rn(__fmul_rn((float)row[x], sc));
      }
    }
    uint4* dst = reinterpret_cast<uint4*>(G + i * 16);
    dst[0] = *reinterpret_cast<const uint4*>(&v[0]);
    dst[1] = *reinterpret_cast<const uint4*>(&v[8]);
  }
}

// ---- 7x7 stride-2 stem (hourglass.py:49-100; 1 or 3 input channels) on the tensor cores -----------------------
// SAME padding of an even-sized input puts 2 rows / columns before and 3 after: output pixel o reads input rows
// 2o-2 .. 2o+4.  With the frame regrouped into 2x2 blocks ("space to depth": block (Y, X) holds pixels (2Y+py, 2X+px),
// 4*Cin values, padded to 16 channels) those are blocks o-1 .. o+2, i.e. a 4x4 stride-1 convolution over the block grid
// with W'[dy][dx][(py, px, c)][co] = w[2(dy+1)+py][2(dx+1)+px][c][co] (zero where the index reaches 7).  The view kernel
// does InferenceLayer.preprocess (uint8 -> float * 1/255, zero pad) on the way; the stock wgmma conv kernel runs
// the convolution (K = 16 taps x 16 channels = 256 instead of 147: the stem was on the CUDA cores before).
// The ResNet stem (ZeroPadding2D(3) + VALID, resnet.py) pads 3|3 instead: output pixel o reads rows 2o-3 .. 2o+3, i.e.
// blocks o-2 .. o+1 with the zero tap at the top / left (W'[dy][dx][(py, px, c)] = w[2dy+py-1][2dx+px-1]).  Its view
// carries the pretrained preprocessing too (pre_mode != 0): tile_channels (1 -> 3, or gray -> 3 for a grayscale-trained
// model fed colour frames), then x * 255, RGB -> BGR, minus the caffe means, on the padded [0, 1] image -- so rows /
// columns of the net input beyond the frame hold -mean, while the conv's own padding (outside the view) stays 0.
template <typename TI>
__global__ void __launch_bounds__(256) k_s2d_view(const TI* __restrict__ img, int Hin, int Win, int Cin, int Hs, int Ws,
                                                  __half* __restrict__ G, int in_is_u8, size_t total, int pre_mode = 0) {
  const float sc = in_is_u8 ? (1.0f / 255.0f) : 1.0f;
  for (size_t i = (size_t)blockIdx.x * 256 + threadIdx.x; i < total; i += (size_t)gridDim.x * 256) {
    const int X = (int)(i % Ws);
    const size_t r = i / Ws;
    const int Y = (int)(r % Hs), b = (int)(r / Hs);
    __align__(16) __half v[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) v[c] = __float2half_rn(0.f);
#pragma unroll
    for (int py = 0; py < 2; ++py)
#pragma unroll
      for (int px = 0; px < 2; ++px) {
        const int y = 2 * Y + py, x = 2 * X + px;
        const bool in = y < Hin && x < Win;
        const TI* p = img + (((size_t)b * Hin + y) * Win + x) * Cin;
        if (pre_mode == SB_PRE_PLAIN) {
          if (in)
            for (int c = 0; c < Cin; ++c) v[(py * 2 + px) * Cin + c] = __float2half_rn(__fmul_rn((float)p[c], sc));
          continue;
        }
        const float g = (in && Cin == 3 && pre_mode == SB_PRE_IMAGENET_CAFFE_GRAY) ? sb_gray_pre(p, in_is_u8) : 0.f;
#pragma unroll
        for (int c = 0; c < 3; ++c) {              // BGR channel c
          float f = 0.f;
          if (in) f = (Cin == 3 && pre_mode == SB_PRE_IMAGENET_CAFFE_GRAY) ? g : __fmul_rn((float)p[Cin == 1 ? 0 : 2 - c], sc);
          v[(py * 2 + px) * 3 + c] = __float2half_rn(__fsub_rn(__fmul_rn(f, 255.f), sb_imagenet_caffe_mean(c)));
        }
      }
    uint4* dst = reinterpret_cast<uint4*>(G + i * 16);
    dst[0] = *reinterpret_cast<const uint4*>(&v[0]);
    dst[1] = *reinterpret_cast<const uint4*>(&v[8]);
  }
}

namespace {

// ---- which route takes the first conv ------------------------------------------------------------------------------

// No op but `reader` reads buffer `buf` (PREPROCESS reads the frame, not a buffer).
bool only_reader(const SbModel* m, int buf, int reader) {
  for (size_t i = 0; i < m->ops.size(); ++i) {
    const SbOp& o = m->ops[i];
    if ((int)i == reader || o.kind() == SB_OPK_PREPROCESS) continue;
    if (o.in_buf() == buf || (o.kind() == SB_OPK_ADD && o.in2_buf() == buf)) return false;
  }
  return true;
}

// k_conv_first can fuse the first conv with the PREPROCESS op `p` before it: a 3x3 SAME conv straight from a 1- or
// 3-channel frame without resize or conversion, its fp16 output in an 8-aligned slice, and nobody else reads the
// preprocessed frame.
bool first_fusable(const SbModel* m, int p) {
  const SbOp& pre = m->ops[p];
  const SbOp& cv = m->ops[p + 1];
  if (cv.kind() != SB_OPK_CONV || cv.in_buf() != pre.out_buf() || cv.k() != 3 || cv.stride() != 1 || cv.explicit_pad()) return false;
  if (pre.input_scale() != 1.0f || pre.pre_mode() != SB_PRE_PLAIN) return false;
  const SbBuffer& ib = m->buffers[pre.out_buf()];
  const SbBuffer& ob = m->buffers[cv.out_buf()];
  if (m->Cin != ib.C || (ib.C != 1 && ib.C != 3) || cv.in_C() != ib.C) return false;
  if (ob.f32 || (cv.flags() & SB_OPF_BN) || ob.C % 8 || cv.out_coff() % 8) return false;
  const int co = cv.out_C();
  return (co == 8 || co == 16 || co == 24 || co == 32 || co == 64) && only_reader(m, pre.out_buf(), p + 1);
}

// The one-channel 3x3 first conv as the Toeplitz GEMM: from the frame (1-channel frames, first_fusable) or, after a
// resize / channel conversion, from the PREPROCESS op's one-channel fp16 output.  N = 8 Cout <= 256 in multiples of 16,
// the whole unpooled fp16 output tensor without BN, whole 8-pixel groups.
bool toeplitz_ok(const SbModel* m, int p, bool from_buffer) {
  const SbOp& cv = m->ops[p + 1];
  if (cv.kind() != SB_OPK_CONV || cv.in_buf() != m->ops[p].out_buf() || cv.in_C() != 1 || cv.k() != 3 || cv.stride() != 1) return false;
  const SbBuffer& ib = m->buffers[cv.in_buf()];
  const SbBuffer& ob = m->buffers[cv.out_buf()];
  if (from_buffer ? (ib.C != 1 || ib.f32 || cv.in_coff() != 0) : m->Cin != 1) return false;
  const int Cout = cv.out_C();
  if (!(Cout == 8 || Cout == 16 || Cout == 24 || Cout == 32)) return false;
  return !ob.f32 && ob.C == Cout && cv.out_coff() == 0 && cv.pool_buf() < 0 && !(cv.flags() & SB_OPF_BN) && ob.W % 8 == 0;
}

// The 7x7 stride-2 stem right after PREPROCESS `p` (hourglass: SAME; ResNet: explicit 3|3 after ImageNet preprocessing)
// with 1 / 3 input channels, no resize, even input extent, an fp16 output in an 8-aligned slice, and nobody else reading
// the preprocessed frame: k_s2d_view then does the preprocessing.
bool stem_fusable(const SbModel* m, int p) {
  const SbOp& pre = m->ops[p];
  const SbOp& cv = m->ops[p + 1];
  if (cv.kind() != SB_OPK_CONV || cv.in_buf() != pre.out_buf() || cv.k() != 7 || cv.stride() != 2) return false;
  if (cv.explicit_pad() && (cv.pad_top() != 3 || cv.pad_left() != 3)) return false;
  if (pre.input_scale() != 1.0f) return false;
  const SbBuffer& ib = m->buffers[pre.out_buf()];
  const SbBuffer& ob = m->buffers[cv.out_buf()];
  if (pre.pre_mode() == SB_PRE_PLAIN ? (m->Cin != ib.C || (ib.C != 1 && ib.C != 3))
                                     : (ib.C != 3 || (m->Cin != 1 && m->Cin != 3))) return false;
  if (cv.in_C() != ib.C || !only_reader(m, pre.out_buf(), p + 1)) return false;
  if (ib.H % 2 || ib.W % 2 || ob.H != ib.H / 2 || ob.W != ib.W / 2) return false;
  return !ob.f32 && ob.C % 8 == 0 && cv.out_coff() % 8 == 0;
}

// k_conv01 takes conv0 (the fused first conv c0) -> conv1 -> pool: 1-channel frames, conv0 = 3x3 s1 1 -> 16, conv1 =
// 3x3 s1 16 -> 16 reading all of conv0's output, no BN, conv1's 2x2 max-pool fused on the tensor-core path with its own
// output dead (so no residual either), even extents, fp16 tensors, and conv1 the only reader of conv0's output.
bool conv01_fusable(const SbModel* m, int c0i) {
  if (m->precision != 0 || c0i + 1 >= (int)m->ops.size()) return false;
  const SbOp& c0 = m->ops[c0i];
  const SbOp& c1 = m->ops[c0i + 1];
  if (m->Cin != 1 || c0.in_C() != 1 || c0.out_C() != 16 || c0.k() != 3 || c0.stride() != 1 || (c0.flags() & SB_OPF_BN)) return false;
  if (c1.kind() != SB_OPK_CONV || c1.in_C() != 16 || c1.out_C() != 16 || c1.k() != 3 || c1.stride() != 1 || (c1.flags() & SB_OPF_BN)) return false;
  if (c1.in_buf() != c0.out_buf() || c1.in_coff() != c0.out_coff() || c1.pool_buf() < 0) return false;
  const SbBuffer& ob0 = m->buffers[c0.out_buf()];
  const SbBuffer& pb = m->buffers[c1.pool_buf()];
  if (ob0.f32 || pb.f32 || pb.C % 2 || c1.pool_coff() % 2 || ob0.H % 2 || ob0.W % 2) return false;
  return m->tc_plans[c0i + 1] && sb_conv_tc_entry(m, c0i + 1, false).elides_out && only_reader(m, c0.out_buf(), c0i + 1);
}

// ---- views -----------------------------------------------------------------------------------------------------------

void free_view(SbEntryPlan& e) {
  if (e.view) cudaFree(e.view);
  if (e.view_bias) cudaFree(e.view_bias);
  e.view = nullptr;
  e.view_bias = nullptr;
}

// Allocates the zeroed view of `route`, and the GEMM plan of the first conv over it (weights w: [R*S][Cout][16]).  The
// route stays as it is where the tensor-core module takes no plan.
int view_prepare(sb_handle_s* h, SbModel* m, int route, SbTcView& V, const std::vector<float>& w) {
  SbEntryPlan& e = m->entry;
  const size_t bytes = (size_t)m->B * e.view_H * e.view_W * 16 * sizeof(__half) + 256;
  SB_CUDA(h, cudaMalloc((void**)&e.view, bytes));
  SB_CUDA(h, cudaMemset(e.view, 0, bytes));
  V.in = SbBuffer(); V.in.C = 16; V.in.H = e.view_H; V.in.W = e.view_W; V.in.dev = e.view;
  if (const int rc = sb_conv_tc_view_prepare(h, m, e.conv_op, V, w)) return rc;
  if (m->tc_plans[e.conv_op]) e.route = route;
  else free_view(e);
  return 0;
}

// The Toeplitz view of the first conv: [B][H][W/8][16] windows, the GEMM writes [H][W/8][8 Cout] = the NHWC output.
int toeplitz_prepare(sb_handle_s* h, SbModel* m, int route) {
  SbEntryPlan& e = m->entry;
  const SbOp& op = m->ops[e.conv_op];
  const SbBuffer& ob = m->buffers[op.out_buf()];
  const int Cout = op.out_C(), N = 8 * Cout;
  e.view_H = ob.H; e.view_W = ob.W / 8;
  std::vector<float> w((size_t)3 * N * 16, 0.f);
  const float* w0 = m->weights_host.data() + op.w_off();                           // [9][1][Cout]
  for (int ky = 0; ky < 3; ++ky)
    for (int j = 0; j < 8; ++j)
      for (int kx = 0; kx < 3; ++kx)
        for (int co = 0; co < Cout; ++co) w[((size_t)ky * N + j * Cout + co) * 16 + j + kx] = w0[(size_t)(ky * 3 + kx) * Cout + co];
  std::vector<float> brep(N, 0.f);
  if (op.b_off() >= 0)
    for (int n = 0; n < N; ++n) brep[n] = m->weights_host[op.b_off() + n % Cout];
  SB_CUDA(h, cudaMalloc((void**)&e.view_bias, N * sizeof(float)));
  SB_CUDA(h, cudaMemcpy(e.view_bias, brep.data(), N * sizeof(float), cudaMemcpyHostToDevice));
  SbTcView V;
  V.out = SbBuffer(); V.out.C = N; V.out.H = ob.H; V.out.W = e.view_W; V.out.dev = ob.dev;
  V.Cout = N;
  V.R = 3; V.S = 1; V.dy0 = -1; V.dx0 = 0;
  V.bias = e.view_bias;
  V.relu = (op.flags() & SB_OPF_RELU) ? 1 : 0;
  return view_prepare(h, m, route, V, w);
}

// The space-to-depth view of the stem: [B][H/2][W/2][16] 2x2 blocks, a 4x4 stride-1 conv over them.
int stem_prepare(sb_handle_s* h, SbModel* m) {
  SbEntryPlan& e = m->entry;
  const SbOp& op = m->ops[e.conv_op];
  const SbBuffer& ob = m->buffers[op.out_buf()];
  const int Cin = op.in_C(), Cout = op.out_C();
  const int sh = op.explicit_pad() ? 1 : 0;                  // 3|3 padding: the 4x4 block window starts one block earlier
  e.view_H = ob.H; e.view_W = ob.W;
  e.pre_mode = m->ops[e.conv_op - 1].pre_mode();
  std::vector<float> w((size_t)16 * Cout * 16, 0.f);
  const float* w7 = m->weights_host.data() + op.w_off();     // [7*7][Cin][Cout]
  for (int dy = 0; dy < 4; ++dy)
    for (int dx = 0; dx < 4; ++dx)
      for (int py = 0; py < 2; ++py)
        for (int px = 0; px < 2; ++px) {
          const int ky = 2 * dy + py - sh, kx = 2 * dx + px - sh;
          if (ky < 0 || kx < 0 || ky > 6 || kx > 6) continue;
          for (int c = 0; c < Cin; ++c)
            for (int co = 0; co < Cout; ++co)
              w[((size_t)(dy * 4 + dx) * Cout + co) * 16 + (py * 2 + px) * Cin + c] = w7[((size_t)(ky * 7 + kx) * Cin + c) * Cout + co];
        }
  SbTcView V;
  V.out = ob;
  V.Cout = Cout; V.out_coff = op.out_coff();
  V.R = 4; V.S = 4; V.dy0 = V.dx0 = -1 - sh;
  V.bias = op.b_off() >= 0 ? m->weights_dev + op.b_off() : nullptr;
  V.relu = (op.flags() & SB_OPF_RELU) ? 1 : 0;
  V.bn_scale = (op.flags() & SB_OPF_BN) ? m->weights_dev + op.bn_scale_off() : nullptr;
  V.bn_shift = (op.flags() & SB_OPF_BN) ? m->weights_dev + op.bn_shift_off() : nullptr;
  return view_prepare(h, m, SB_ENTRY_STEM_VIEW, V, w);
}

// ---- launches --------------------------------------------------------------------------------------------------------

template <typename TI, int CIN>
void launch_first(int co, int B, cudaStream_t s, const TI* img, int Hin, int Win, int Hnet, int Wnet, __half* out,
                  int Ctot, int coff, const float* w, const float* b, int relu, int is_u8, int split) {
  dim3 blk(32, 8);
  auto grid = [&](int px) { return dim3((Wnet + 32 * px - 1) / (32 * px), (Hnet + 7) / 8, B); };
  switch (co) {
    case 8: k_conv_first<TI, CIN, 8, 4><<<grid(4), blk, 0, s>>>(img, Hin, Win, Hnet, Wnet, out, Ctot, coff, w, b, relu, is_u8, split); break;
    case 16: k_conv_first<TI, CIN, 16, 4><<<grid(4), blk, 0, s>>>(img, Hin, Win, Hnet, Wnet, out, Ctot, coff, w, b, relu, is_u8, split); break;
    case 24: k_conv_first<TI, CIN, 24, 2><<<grid(2), blk, 0, s>>>(img, Hin, Win, Hnet, Wnet, out, Ctot, coff, w, b, relu, is_u8, split); break;
    case 32: k_conv_first<TI, CIN, 32, 2><<<grid(2), blk, 0, s>>>(img, Hin, Win, Hnet, Wnet, out, Ctot, coff, w, b, relu, is_u8, split); break;
    default: k_conv_first<TI, CIN, 64, 1><<<grid(1), blk, 0, s>>>(img, Hin, Win, Hnet, Wnet, out, Ctot, coff, w, b, relu, is_u8, split); break;
  }
}

// The direct route: k_conv_first (precision 2: its split store).
SbLaunchFn direct_entry(const SbModel* m) {
  const SbOp& op = m->ops[m->entry.conv_op];
  const SbBuffer ob = m->buffers[op.out_buf()];
  const float* Wt = m->weights_dev + op.w_off();
  const float* bias = op.b_off() >= 0 ? m->weights_dev + op.b_off() : nullptr;
  const int relu = (op.flags() & SB_OPF_RELU) ? 1 : 0;
  const int split = m->precision == 2 ? op.out_C() : 0;
  const int Cin = m->Cin, Hin = m->Hin, Win = m->Win, co = op.out_C(), coff = op.out_coff();
  // rows/cols beyond the resized frame (Hres, Wres) are the bottom/right zero padding
  return [=](sb_handle_s* h, const void* frames_dev, int frames_are_u8, int B) {
    cudaStream_t s = h->stream;
    if (frames_are_u8) {
      if (Cin == 1) launch_first<unsigned char, 1>(co, B, s, (const unsigned char*)frames_dev, Hin, Win, ob.H, ob.W, (__half*)ob.dev, ob.C, coff, Wt, bias, relu, 1, split);
      else launch_first<unsigned char, 3>(co, B, s, (const unsigned char*)frames_dev, Hin, Win, ob.H, ob.W, (__half*)ob.dev, ob.C, coff, Wt, bias, relu, 1, split);
    } else {
      if (Cin == 1) launch_first<float, 1>(co, B, s, (const float*)frames_dev, Hin, Win, ob.H, ob.W, (__half*)ob.dev, ob.C, coff, Wt, bias, relu, 0, split);
      else launch_first<float, 3>(co, B, s, (const float*)frames_dev, Hin, Win, ob.H, ob.W, (__half*)ob.dev, ob.C, coff, Wt, bias, relu, 0, split);
    }
    SB_CHECK_LAUNCH(h);
    return 0;
  };
}

// The view routes: the route's view kernel, then the GEMM over the view (its plan stores its whole output in both programs).
SbLaunchFn view_entry(SbModel* m) {
  const SbEntryPlan& e = m->entry;
  const int route = e.route, view_H = e.view_H, view_W = e.view_W, pre_mode = e.pre_mode;
  const int Cin = m->Cin, Hin = m->Hin, Win = m->Win;
  __half* view = e.view;
  const SbBuffer ib = m->buffers[m->ops[e.conv_op].in_buf()];
  const SbLaunchFn gemm = sb_conv_tc_entry(m, e.conv_op, false).run;
  return [=](sb_handle_s* h, const void* frames_dev, int frames_are_u8, int B) {
    const size_t total = (size_t)B * view_H * view_W;
    const int grid = (int)std::min<size_t>((total + 255) / 256, (size_t)h->sm_count * 16);
    cudaStream_t s = h->stream;
    if (route == SB_ENTRY_BUFFER_VIEW) {
      k_first_view<__half><<<grid, 256, 0, s>>>((const __half*)ib.dev, ib.H, ib.W, view_H, view_W, view, 0, total);
    } else if (route == SB_ENTRY_STEM_VIEW) {
      if (frames_are_u8)
        k_s2d_view<unsigned char><<<grid, 256, 0, s>>>((const unsigned char*)frames_dev, Hin, Win, Cin, view_H, view_W, view, 1,
                                                       total, pre_mode);
      else
        k_s2d_view<float><<<grid, 256, 0, s>>>((const float*)frames_dev, Hin, Win, Cin, view_H, view_W, view, 0, total, pre_mode);
    } else if (frames_are_u8) {
      k_first_view<unsigned char><<<grid, 256, 0, s>>>((const unsigned char*)frames_dev, Hin, Win, view_H, view_W, view, 1, total);
    } else {
      k_first_view<float><<<grid, 256, 0, s>>>((const float*)frames_dev, Hin, Win, view_H, view_W, view, 0, total);
    }
    SB_CHECK_LAUNCH(h);
    return gemm(h, frames_dev, frames_are_u8, B);
  };
}

// The first conv as picked, without the fused block.
SbLaunchFn first_conv_entry(SbModel* m) {
  return m->entry.route == SB_ENTRY_DIRECT ? direct_entry(m) : view_entry(m);
}

// The fused first block.
SbLaunchFn conv01_entry(const SbConv01Plan* pl) {
  return [pl](sb_handle_s* h, const void* frames_dev, int frames_are_u8, int B) {
    return sb_conv01_launch(h, pl, frames_dev, frames_are_u8, B);
  };
}

}  // namespace

// Precision 1 keeps the generic route.  Precision 2 fuses the first conv into k_conv_first (split store) where it can,
// else its preprocessed frame stays fp32 for k_conv_direct.  Precision 0 takes a view where the shape allows one.
int sb_entry_prepare(sb_handle_s* h, SbModel* m) {
  SbEntryPlan& e = m->entry;
  int p = 0;                                             // the PREPROCESS op (sb_load_model allows one)
  while (p < (int)m->ops.size() && m->ops[p].kind() != SB_OPK_PREPROCESS) ++p;
  if (m->precision == 1 || p + 1 >= (int)m->ops.size()) return 0;
  const bool views = m->precision == 0 && !getenv("SB_DISABLE_TC");
  const bool first_view = views && !getenv("SB_DISABLE_FIRST_VIEW"), stem_view = views && !getenv("SB_DISABLE_STEM_VIEW");
  e.conv_op = p + 1;
  int rc = 0;
  if (first_fusable(m, p)) {
    e.route = SB_ENTRY_DIRECT;
    if (first_view && toeplitz_ok(m, p, false)) rc = toeplitz_prepare(h, m, SB_ENTRY_FRAME_VIEW);
    if (!rc && conv01_fusable(m, e.conv_op)) rc = sb_conv01_prepare(h, m, e.conv_op, e.conv_op + 1);
  } else if (stem_view && stem_fusable(m, p)) {
    rc = stem_prepare(h, m);
  } else if (first_view && toeplitz_ok(m, p, true)) {
    rc = toeplitz_prepare(h, m, SB_ENTRY_BUFFER_VIEW);
  }
  if (e.route == SB_ENTRY_GENERIC) e.conv_op = -1;
  else if (e.route != SB_ENTRY_BUFFER_VIEW) e.pre_op = p;
  return rc;
}

// The frame view against k_conv_first, then the fused block against conv0 + conv1 as just picked (their launch forms
// as sb_conv_tc_autotune picked them), at the configured batch on the model's own buffers.
int sb_entry_autotune(sb_handle_s* h, SbModel* m) {
  SbEntryPlan& e = m->entry;
  const bool dbg = getenv("SB_DEBUG") != nullptr;
  char what[64];
  if (e.route == SB_ENTRY_FRAME_VIEW) {
    const SbLaunchFn cand[2] = {direct_entry(m), view_entry(m)};
    float best[2];
    for (int f = 0; f < 2; ++f) {
      snprintf(what, sizeof what, "first layer, form %d", f);
      const int rc = sb_time_min(h, what, best[f], [&] { return cand[f](h, m->frames_dev, 1, m->B); });
      if (rc) return rc;
    }
    bool view = best[1] < best[0];
    if (const char* fv = getenv("SB_FORCE_FIRST_VIEW")) view = atoi(fv) != 0;
    if (dbg) fprintf(stderr, "[sb_conv_tc] op %d first layer: k_conv_first %.1f us, Toeplitz view + wgmma %.1f us -> %s\n", e.conv_op,
                     best[0] * 1e3f, best[1] * 1e3f, view ? "view" : "direct");
    if (!view) {
      sb_conv_tc_drop(m, e.conv_op);
      free_view(e);
      e.route = SB_ENTRY_DIRECT;
    }
  }
  if (e.conv01) {
    const SbLaunchFn conv0 = first_conv_entry(m), conv1 = sb_conv_tc_entry(m, e.conv_op + 1, false).run, fused_block = conv01_entry(e.conv01);
    float best[2];
    for (int f = 0; f < 2; ++f) {
      snprintf(what, sizeof what, "first block, fused %d", f);
      const int rc = sb_time_min(h, what, best[f], [&] {
        if (f == 1) return fused_block(h, m->frames_dev, 1, m->B);
        const int rc0 = conv0(h, m->frames_dev, 1, m->B);
        return rc0 ? rc0 : conv1(h, m->frames_dev, 1, m->B);
      });
      if (rc) return rc;
    }
    bool fused = best[1] < best[0];
    if (const char* fv = getenv("SB_FORCE_CONV01")) fused = atoi(fv) != 0;
    if (dbg) fprintf(stderr, "[sb_conv_tc] first block (B = %d): conv0 + conv1 launches %.1f us, fused k_conv01 %.1f us -> %s\n", m->B,
                     best[0] * 1e3f, best[1] * 1e3f, fused ? "fused" : "separate");
    if (fused) e.conv1_op = e.conv_op + 1;
  }
  return 0;
}

// The PREPROCESS op's slot is empty where the first conv's launch preprocesses the frame.  The first conv runs its route,
// or in the production program the fused block, whose conv1 and pool slots are then empty.  The all-stores program runs
// the separate launches instead (conv1 as an ordinary tensor-core conv), which store the block's two tensors.
void sb_entry_build(SbModel* m, bool all_stores, std::vector<char>& taken) {
  const SbEntryPlan& e = m->entry;
  if (e.pre_op >= 0) taken[e.pre_op] = 1;
  if (e.conv_op < 0) return;
  const bool fused = e.conv1_op >= 0 && !all_stores;
  m->prog[all_stores][e.conv_op] = fused ? conv01_entry(e.conv01) : first_conv_entry(m);
  taken[e.conv_op] = 1;
  if (fused) taken[e.conv1_op] = taken[e.conv1_op + 1] = 1;
  if (e.conv01) m->buf_elided[m->ops[e.conv_op].out_buf()] = m->buf_elided[m->ops[e.conv_op + 1].out_buf()] = 1;
}

// The views and the fused block's plan; the view's GEMM plan goes with the tensor-core plans (sb_conv_tc_release).
void sb_entry_release(SbModel* m) {
  free_view(m->entry);
  sb_conv01_release(m);
  m->entry = SbEntryPlan();
}
