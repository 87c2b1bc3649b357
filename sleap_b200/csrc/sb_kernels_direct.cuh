// CUDA-core ("direct") layer kernels: the fp32 strict-parity path, the first layers with C_in of
// 1 or 3, and every non-GEMM op (pool / upsample / add / preprocess).  Activations are NHWC with a
// channel-slice view (buffer row pitch Ctot, slice offset) so that skip connections are
// concatenated by construction (producers write straight into their slice of the concat buffer).
//
// Reference ops restated (file:line under /root/reference):
//   conv + bias + ReLU (+ BN affine after ReLU): architectures/encoder_decoder.py:117-131,
//        369-389; hourglass.py:36-45; heads.py:55-63 (1x1 linear)
//   Conv2DTranspose k3 s2 SAME:  encoder_decoder.py:304-310
//   MaxPool2D 2x2 s2 SAME:       encoder_decoder.py:109-114; unet.py:36-41; hourglass.py:94-98,133
//   UpSampling2D bilinear/nearest: encoder_decoder.py:335-339; hourglass.py:185-187
//   Add:                         hourglass.py:190
//   preprocess:                  inference.py:940-967; data/normalization.py:34-114;
//                                data/resizing.py:34-106
#pragma once
#include "sb_common.cuh"

namespace sbd {

template <typename T> __device__ __forceinline__ float ld(const T* p);
template <> __device__ __forceinline__ float ld<float>(const float* p) { return *p; }
template <> __device__ __forceinline__ float ld<__half>(const __half* p) { return __half2float(*p); }
__device__ __forceinline__ void st(float* p, float v) { *p = v; }
__device__ __forceinline__ void st(__half* p, float v) { *p = __float2half_rn(v); }
// Split-fp16 activations (precision 2): a tensor of C logical channels occupies 3C fp16 channels [lo | hi | hi] with
// hi = fp16(v), lo = fp16(v - hi); a consumer conv whose weight rows are [Wh | Wl | Wh] (Wh = fp16(W), Wl = fp16(W - Wh))
// then accumulates lo*Wh + hi*Wl + hi*Wh = v*W up to the dropped lo*Wl term (2^-22 relative) on the fp16 tensor cores.
// The two correction planes come FIRST in channel (= K) order: the tensor core's fp32 accumulator truncates, each MMA
// step losing ~ulp(accumulator), so the 2^-11-sized terms are added while the accumulator is still small.
// `split` = C (the distance between the three planes), 0 = plain store.
__device__ __forceinline__ void st_split(float* p, float v, int) { *p = v; }
__device__ __forceinline__ void st_split(__half* p, float v, int split) {
  const __half hi = __float2half_rn(v);
  if (split) { p[0] = __float2half_rn(v - __half2float(hi)); p[split] = hi; p[2 * split] = hi; }
  else *p = hi;
}
__device__ __forceinline__ float ld_split(const __half* p, int split) { return __half2float(p[0]) + __half2float(p[split]); }

struct View {       // channel-slice view of an NHWC buffer
  void* ptr;
  int H, W, Ctot, coff;
};

constexpr int DC_TILE = 16;   // output tile 16x16 pixels, one pixel per thread
constexpr int DC_CO = 16;     // output channels per thread
constexpr int DC_CK = 8;      // input-channel chunk staged in shared memory

// Generic k x k, stride s, TF-"SAME" convolution.  weights: [k*k][Cin][Cout] fp32.
// Epilogue: + bias, ReLU (flag), * bn_scale + bn_shift (flag).
template <typename TI, typename TO>
__global__ void __launch_bounds__(256) k_conv_direct(
    const TI* __restrict__ in, int Hin, int Win, int in_Ctot, int in_coff, int Cin,
    TO* __restrict__ out, int Hout, int Wout, int out_Ctot, int out_coff, int Cout,
    const float* __restrict__ w, const float* __restrict__ bias, const float* __restrict__ bn_scale,
    const float* __restrict__ bn_shift, int k, int stride, int pad_top, int pad_left, int relu, int split = 0) {
  extern __shared__ float smem[];
  const int in_tile = (DC_TILE - 1) * stride + k;
  float* s_in = smem;                                   // [in_tile][in_tile][DC_CK]
  float* s_w = smem + in_tile * in_tile * DC_CK;        // [k*k][DC_CK][DC_CO]
  const int tiles_x = (Wout + DC_TILE - 1) / DC_TILE;
  const int tx0 = (blockIdx.x % tiles_x) * DC_TILE, ty0 = (blockIdx.x / tiles_x) * DC_TILE;
  const int co0 = blockIdx.y * DC_CO;
  const int b = blockIdx.z;
  const int lx = threadIdx.x % DC_TILE, ly = threadIdx.x / DC_TILE;
  const int ox = tx0 + lx, oy = ty0 + ly;
  const int iy0 = ty0 * stride - pad_top, ix0 = tx0 * stride - pad_left;
  const TI* in_b = in + (size_t)b * Hin * Win * in_Ctot + in_coff;
  float acc[DC_CO];
#pragma unroll
  for (int c = 0; c < DC_CO; ++c) acc[c] = 0.f;
  for (int c0 = 0; c0 < Cin; c0 += DC_CK) {
    __syncthreads();
    for (int t = threadIdx.x; t < in_tile * in_tile * DC_CK; t += 256) {
      const int c = t % DC_CK;
      const int xx = (t / DC_CK) % in_tile, yy = t / (DC_CK * in_tile);
      const int gy = iy0 + yy, gx = ix0 + xx;
      float v = 0.f;
      if (gy >= 0 && gy < Hin && gx >= 0 && gx < Win && c0 + c < Cin)
        v = ld<TI>(in_b + ((size_t)gy * Win + gx) * in_Ctot + c0 + c);
      s_in[t] = v;
    }
    for (int t = threadIdx.x; t < k * k * DC_CK * DC_CO; t += 256) {
      const int co = t % DC_CO;
      const int c = (t / DC_CO) % DC_CK;
      const int tap = t / (DC_CO * DC_CK);
      float v = 0.f;
      if (c0 + c < Cin && co0 + co < Cout) v = w[((size_t)tap * Cin + c0 + c) * Cout + co0 + co];
      s_w[t] = v;
    }
    __syncthreads();
    for (int ky = 0; ky < k; ++ky)
      for (int kx = 0; kx < k; ++kx) {
        const float* pin = s_in + ((ly * stride + ky) * in_tile + lx * stride + kx) * DC_CK;
        const float* pw = s_w + (ky * k + kx) * DC_CK * DC_CO;
#pragma unroll
        for (int c = 0; c < DC_CK; ++c) {
          const float v = pin[c];
          const float4* w4 = reinterpret_cast<const float4*>(pw + c * DC_CO);
#pragma unroll
          for (int q = 0; q < DC_CO / 4; ++q) {
            const float4 ww = w4[q];
            acc[4 * q + 0] = fmaf(v, ww.x, acc[4 * q + 0]);
            acc[4 * q + 1] = fmaf(v, ww.y, acc[4 * q + 1]);
            acc[4 * q + 2] = fmaf(v, ww.z, acc[4 * q + 2]);
            acc[4 * q + 3] = fmaf(v, ww.w, acc[4 * q + 3]);
          }
        }
      }
  }
  if (ox < Wout && oy < Hout) {
    TO* po = out + (((size_t)b * Hout + oy) * Wout + ox) * out_Ctot + out_coff + co0;
#pragma unroll
    for (int c = 0; c < DC_CO; ++c) {
      if (co0 + c < Cout) {
        float v = acc[c] + (bias ? bias[co0 + c] : 0.f);
        if (relu) v = fmaxf(v, 0.f);
        if (bn_scale) v = v * bn_scale[co0 + c] + bn_shift[co0 + c];
        st_split(po + c, v, split);
      }
    }
  }
}

// Conv2DTranspose(k, strides=2, padding="same"), k = 3 or 4: out (2H, 2W), out[o] += in[i] * W[o - 2i + p] with the
// forward-conv padding p = (k - 2) / 2 (0 for k3, 1 for k4).  Per axis:
//   k3: out[2i] = in[i]*W[0] + in[i-1]*W[2];            out[2i+1] = in[i]*W[1]
//   k4: out[2i] = in[i]*W[1] + in[i-1]*W[3];            out[2i+1] = in[i+1]*W[0] + in[i]*W[2]
// weights [k*k][Cin][Cout].
template <typename TI, typename TO>
__global__ void __launch_bounds__(256) k_tconv_direct(
    const TI* __restrict__ in, int Hin, int Win, int in_Ctot, int in_coff, int Cin,
    TO* __restrict__ out, int out_Ctot, int out_coff, int Cout, const float* __restrict__ w,
    const float* __restrict__ bias, int relu, int split = 0, int k = 3) {
  const int Hout = 2 * Hin, Wout = 2 * Win;
  const int b = blockIdx.z;
  const int co0 = blockIdx.y * DC_CO;
  const int pix = blockIdx.x * 256 + threadIdx.x;
  if (pix >= Hout * Wout) return;
  const int oy = pix / Wout, ox = pix - oy * Wout;
  const TI* in_b = in + (size_t)b * Hin * Win * in_Ctot + in_coff;
  float acc[DC_CO];
#pragma unroll
  for (int c = 0; c < DC_CO; ++c) acc[c] = 0.f;
  int kys[2], iys[2], nky = 0, kxs[2], ixs[2], nkx = 0;
  const int p = (k - 2) / 2;
  for (int kk = 0; kk < k; ++kk) {              // taps with o - kk + p even and the input index inside the map
    const int ty = oy - kk + p, tx = ox - kk + p;
    if (!(ty & 1) && ty >= 0 && (ty >> 1) < Hin) { kys[nky] = kk; iys[nky] = ty >> 1; ++nky; }
    if (!(tx & 1) && tx >= 0 && (tx >> 1) < Win) { kxs[nkx] = kk; ixs[nkx] = tx >> 1; ++nkx; }
  }
  for (int a = 0; a < nky; ++a)
    for (int bb = 0; bb < nkx; ++bb) {
      const TI* pin = in_b + ((size_t)iys[a] * Win + ixs[bb]) * in_Ctot;
      const float* pw = w + (size_t)(kys[a] * k + kxs[bb]) * Cin * Cout + co0;
      for (int c = 0; c < Cin; ++c) {
        const float v = ld<TI>(pin + c);
#pragma unroll
        for (int q = 0; q < DC_CO; ++q)
          if (co0 + q < Cout) acc[q] = fmaf(v, pw[(size_t)c * Cout + q], acc[q]);
      }
    }
  TO* po = out + (((size_t)b * Hout + oy) * Wout + ox) * out_Ctot + out_coff + co0;
#pragma unroll
  for (int c = 0; c < DC_CO; ++c)
    if (co0 + c < Cout) {
      float v = acc[c] + (bias ? bias[co0 + c] : 0.f);
      if (relu) v = fmaxf(v, 0.f);
      st_split(po + c, v, split);
    }
}

template <typename T>
__global__ void k_maxpool2(const T* __restrict__ in, int Hin, int Win, int in_Ctot, int in_coff, int C,
                           T* __restrict__ out, int Hout, int Wout, int out_Ctot, int out_coff, size_t total) {
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(t % C);
    const int ox = (int)((t / C) % Wout);
    const int oy = (int)((t / ((size_t)C * Wout)) % Hout);
    const int b = (int)(t / ((size_t)C * Wout * Hout));
    const T* pin = in + (size_t)b * Hin * Win * in_Ctot + in_coff + c;
    float m = -INFINITY;
    for (int dy = 0; dy < 2; ++dy)
      for (int dx = 0; dx < 2; ++dx) {
        const int iy = 2 * oy + dy, ix = 2 * ox + dx;
        if (iy < Hin && ix < Win) m = fmaxf(m, ld<T>(pin + ((size_t)iy * Win + ix) * in_Ctot));
      }
    st(out + (((size_t)b * Hout + oy) * Wout + ox) * out_Ctot + out_coff + c, m);
  }
}

// ZeroPadding2D(1) + MaxPooling2D(3, strides=2, padding="valid") (ResNet stem): out[o] = max(in[2o-1 .. 2o+1]) with
// positions outside the map reading 0 (the zero padding), not -inf.
template <typename T>
__global__ void k_maxpool3s2(const T* __restrict__ in, int Hin, int Win, int in_Ctot, int in_coff, int C,
                             T* __restrict__ out, int Hout, int Wout, int out_Ctot, int out_coff, size_t total) {
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(t % C);
    const int ox = (int)((t / C) % Wout);
    const int oy = (int)((t / ((size_t)C * Wout)) % Hout);
    const int b = (int)(t / ((size_t)C * Wout * Hout));
    const T* pin = in + (size_t)b * Hin * Win * in_Ctot + in_coff + c;
    float m = -INFINITY;
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const int iy = 2 * oy + dy, ix = 2 * ox + dx;
        m = fmaxf(m, (iy >= 0 && iy < Hin && ix >= 0 && ix < Win) ? ld<T>(pin + ((size_t)iy * Win + ix) * in_Ctot) : 0.f);
      }
    st(out + (((size_t)b * Hout + oy) * Wout + ox) * out_Ctot + out_coff + c, m);
  }
}

// x2 upsampling: bilinear with half-pixel centres (weights 1/4, 3/4, edge clamp) or nearest.
template <typename T>
__global__ void k_upsample2(const T* __restrict__ in, int Hin, int Win, int in_Ctot, int in_coff, int C,
                            T* __restrict__ out, int out_Ctot, int out_coff, int bilinear, size_t total) {
  const int Hout = 2 * Hin, Wout = 2 * Win;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(t % C);
    const int ox = (int)((t / C) % Wout);
    const int oy = (int)((t / ((size_t)C * Wout)) % Hout);
    const int b = (int)(t / ((size_t)C * Wout * Hout));
    const T* pin = in + (size_t)b * Hin * Win * in_Ctot + in_coff + c;
    float v;
    if (!bilinear) {
      v = ld<T>(pin + ((size_t)(oy >> 1) * Win + (ox >> 1)) * in_Ctot);
    } else {
      const float sy = ((float)oy + 0.5f) * 0.5f - 0.5f, sx = ((float)ox + 0.5f) * 0.5f - 0.5f;
      const float fy = floorf(sy), fx = floorf(sx);
      const int y0 = max((int)fy, 0), y1 = min((int)ceilf(sy), Hin - 1);
      const int x0 = max((int)fx, 0), x1 = min((int)ceilf(sx), Win - 1);
      const float ly = sy - fy, lx = sx - fx;
      const float tl = ld<T>(pin + ((size_t)y0 * Win + x0) * in_Ctot), tr = ld<T>(pin + ((size_t)y0 * Win + x1) * in_Ctot);
      const float bl = ld<T>(pin + ((size_t)y1 * Win + x0) * in_Ctot), br = ld<T>(pin + ((size_t)y1 * Win + x1) * in_Ctot);
      const float tp = tl + (tr - tl) * lx, bt = bl + (br - bl) * lx;
      v = tp + (bt - tp) * ly;
    }
    st(out + (((size_t)b * Hout + oy) * Wout + ox) * out_Ctot + out_coff + c, v);
  }
}

template <typename T>
__global__ void k_add(const T* __restrict__ a, int a_Ctot, int a_coff, const T* __restrict__ bsrc, int b_Ctot,
                      int b_coff, T* __restrict__ out, int out_Ctot, int out_coff, int C, size_t npix, int relu = 0) {
  const size_t total = npix * C;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(t % C);
    const size_t p = t / C;
    const float v = ld<T>(a + p * a_Ctot + a_coff + c) + ld<T>(bsrc + p * b_Ctot + b_coff + c);
    st(out + p * out_Ctot + out_coff + c, relu ? fmaxf(v, 0.f) : v);
  }
}

template <typename T>
__global__ void k_copy(const T* __restrict__ a, int a_Ctot, int a_coff, T* __restrict__ out, int out_Ctot,
                       int out_coff, int C, size_t npix) {
  const size_t total = npix * C;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(t % C);
    const size_t p = t / C;
    out[p * out_Ctot + out_coff + c] = a[p * a_Ctot + a_coff + c];
  }
}

// Preprocess (InferenceLayer.preprocess): gray<->rgb, u8 -> float * (1/255), bilinear resize by
// input_scale (half-pixel centres, no antialias), zero pad bottom/right to the net input size.
//   mode_ch: 0 keep, 1 rgb->gray (u8: truncating round trip like tf.image.rgb_to_grayscale; with Cnet = 3 the gray value
//            fills all three channels), 2 gray->rgb
//   imagenet: then imagenet_preproc_v1 (resnet.py) on the padded [0, 1] image: x * 255, RGB -> BGR, minus the caffe
//             means -- the bottom / right padding becomes -mean, as in the reference, where it runs inside the model
template <typename TI, typename TO>
__global__ void k_preprocess(const TI* __restrict__ in, int Hin, int Win, int Cin, TO* __restrict__ out,
                             int Hnet, int Wnet, int Cnet, int Hres, int Wres, int resize, int mode_ch,
                             int in_is_u8, size_t total, int imagenet = 0) {
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(t % Cnet);
    const int ox = (int)((t / Cnet) % Wnet);
    const int oy = (int)((t / ((size_t)Cnet * Wnet)) % Hnet);
    const int b = (int)(t / ((size_t)Cnet * Wnet * Hnet));
    float v = 0.f;
    if (oy < Hres && ox < Wres) {
      const TI* img = in + (size_t)b * Hin * Win * Cin;
      auto fetch = [&](int y, int x) -> float {
        const TI* p = img + ((size_t)y * Win + x) * Cin;
        float f;
        if (mode_ch == 1) {
          f = sb_gray_pre(p, in_is_u8);
        } else {
          const int cc = (mode_ch == 2) ? 0 : (imagenet ? 2 - c : c);     // imagenet: BGR channel c reads RGB 2 - c
          f = (float)p[cc];
          if (in_is_u8) f = __fmul_rn(f, 1.0f / 255.0f);
        }
        return f;
      };
      v = resize ? sb_resize_sample(fetch, oy, ox, Hin, Win, Hres, Wres) : fetch(oy, ox);
    }
    if (imagenet) v = __fsub_rn(__fmul_rn(v, 255.f), sb_imagenet_caffe_mean(c));
    st(out + t, v);
  }
}

// ---- precision 2 (split-fp16 activations, see st_split): the elementwise ops act on v = hi + lo ----
// C is the LOGICAL channel count; the tensors hold 3C channels [lo | hi | hi] from their channel offset.
__global__ void k_maxpool2_split(const __half* __restrict__ in, int Hin, int Win, int in_Ctot, int in_coff, int C,
                                 __half* __restrict__ out, int Hout, int Wout, int out_Ctot, int out_coff, size_t total) {
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(t % C);
    const int ox = (int)((t / C) % Wout);
    const int oy = (int)((t / ((size_t)C * Wout)) % Hout);
    const int b = (int)(t / ((size_t)C * Wout * Hout));
    const __half* pin = in + (size_t)b * Hin * Win * in_Ctot + in_coff + c;
    float m = -INFINITY;
    for (int dy = 0; dy < 2; ++dy)
      for (int dx = 0; dx < 2; ++dx) {
        const int iy = 2 * oy + dy, ix = 2 * ox + dx;
        if (iy < Hin && ix < Win) m = fmaxf(m, ld_split(pin + ((size_t)iy * Win + ix) * in_Ctot, C));
      }
    st_split(out + (((size_t)b * Hout + oy) * Wout + ox) * out_Ctot + out_coff + c, m, C);
  }
}

__global__ void k_upsample2_split(const __half* __restrict__ in, int Hin, int Win, int in_Ctot, int in_coff, int C,
                                  __half* __restrict__ out, int out_Ctot, int out_coff, int bilinear, size_t total) {
  const int Hout = 2 * Hin, Wout = 2 * Win;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(t % C);
    const int ox = (int)((t / C) % Wout);
    const int oy = (int)((t / ((size_t)C * Wout)) % Hout);
    const int b = (int)(t / ((size_t)C * Wout * Hout));
    const __half* pin = in + (size_t)b * Hin * Win * in_Ctot + in_coff + c;
    float v;
    if (!bilinear) {
      v = ld_split(pin + ((size_t)(oy >> 1) * Win + (ox >> 1)) * in_Ctot, C);
    } else {
      const float sy = ((float)oy + 0.5f) * 0.5f - 0.5f, sx = ((float)ox + 0.5f) * 0.5f - 0.5f;
      const float fy = floorf(sy), fx = floorf(sx);
      const int y0 = max((int)fy, 0), y1 = min((int)ceilf(sy), Hin - 1);
      const int x0 = max((int)fx, 0), x1 = min((int)ceilf(sx), Win - 1);
      const float ly = sy - fy, lx = sx - fx;
      const float tl = ld_split(pin + ((size_t)y0 * Win + x0) * in_Ctot, C), tr = ld_split(pin + ((size_t)y0 * Win + x1) * in_Ctot, C);
      const float bl = ld_split(pin + ((size_t)y1 * Win + x0) * in_Ctot, C), br = ld_split(pin + ((size_t)y1 * Win + x1) * in_Ctot, C);
      const float tp = tl + (tr - tl) * lx, bt = bl + (br - bl) * lx;
      v = tp + (bt - tp) * ly;
    }
    st_split(out + (((size_t)b * Hout + oy) * Wout + ox) * out_Ctot + out_coff + c, v, C);
  }
}

__global__ void k_add_split(const __half* __restrict__ a, int a_Ctot, int a_coff, const __half* __restrict__ bsrc, int b_Ctot,
                            int b_coff, __half* __restrict__ out, int out_Ctot, int out_coff, int C, size_t npix, int relu = 0) {
  const size_t total = npix * C;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(t % C);
    const size_t p = t / C;
    const float v = ld_split(a + p * a_Ctot + a_coff + c, C) + ld_split(bsrc + p * b_Ctot + b_coff + c, C);
    st_split(out + p * out_Ctot + out_coff + c, relu ? fmaxf(v, 0.f) : v, C);
  }
}

__global__ void k_maxpool3s2_split(const __half* __restrict__ in, int Hin, int Win, int in_Ctot, int in_coff, int C,
                                   __half* __restrict__ out, int Hout, int Wout, int out_Ctot, int out_coff, size_t total) {
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (size_t)gridDim.x * blockDim.x) {
    const int c = (int)(t % C);
    const int ox = (int)((t / C) % Wout);
    const int oy = (int)((t / ((size_t)C * Wout)) % Hout);
    const int b = (int)(t / ((size_t)C * Wout * Hout));
    const __half* pin = in + (size_t)b * Hin * Win * in_Ctot + in_coff + c;
    float m = -INFINITY;
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const int iy = 2 * oy + dy, ix = 2 * ox + dx;
        m = fmaxf(m, (iy >= 0 && iy < Hin && ix >= 0 && ix < Win) ? ld_split(pin + ((size_t)iy * Win + ix) * in_Ctot, C) : 0.f);
      }
    st_split(out + (((size_t)b * Hout + oy) * Wout + ox) * out_Ctot + out_coff + c, m, C);
  }
}

}  // namespace sbd
