// Pyramidal Lucas-Kanade flow shift of the optical-flow trackers (sleap/nn/tracking.py:262-360, which calls
// cv2.calcOpticalFlowPyrLK).  Per frame: upload, gray + resize (k_flow_level0), pyrDown (k_flow_pyrdown) and the
// Scharr derivatives plus the reflect-101 image border of every level (k_flow_finish).  Per tracked frame: one
// k_flow_lk launch, one warp per (reference frame, point) pair.
//
// OpenCV's rules, each confirmed black-box against cv2 4.13:
//   gray     (B*3735 + G*19235 + R*9798 + 2^14) >> 15
//   resize   fx = fy = 0.5 with INTER_LINEAR runs OpenCV's 2x2 area path: (sum + 2) >> 2, and rint(sum / count) in
//            the partial last row / column; output size rint(w * 0.5) (half to even)
//   pyrDown  [1 4 6 4 1]^2 with reflect-101, (sum + 128) >> 8, size ((w+1)/2, (h+1)/2)
//   Scharr   dx = [3 10 3]^T x [-1 0 1], dy = [-1 0 1]^T x [3 10 3], reflect-101, int16
//   levels   after level l, stop when ((w+1)/2 <= win || (h+1)/2 <= win)
// Every level is stored with a border of `win` pixels (image: reflect-101, derivatives: 0), as OpenCV pads its
// pyramid, so the window reads of the LK kernel need no bounds checks.  The ring's pyramids are one allocation for the
// images and one for the derivatives, slot s at s times a fixed slot stride, so the ring has no size cap of its own.
//
// The LK iteration follows OpenCV's tracker: 14-bit fixed-point bilinear weights, image samples kept with 5
// fractional bits and derivative samples with none, sums scaled by 2^-20, the min-eigenvalue / determinant test,
// 30 iterations or a step below 0.01 px, the oscillation guard, and err = sum|J - I| / (32 win^2).  The window
// sums are accumulated exactly in integers (OpenCV sums the same integer products in float, in SIMD-lane order),
// so the sums equal OpenCV's to float rounding and found points agree to the stopping step.  Built with
// -fmad=false: the float steps (weights, eigenvalue, update) then round like OpenCV's x86 build, which contracts
// nothing into FMAs.
#include <algorithm>
#include <cfloat>
#include <cmath>

#include "sb_common.cuh"

namespace {

constexpr int kFlowMaxLevels = 16;
constexpr int kFlowMaxWin = 41;
constexpr int kFlowWarps = 4;                  // points per LK block
// k_flow_lk sums each lane's share of the window in 32-bit ints.  The largest term is b1's |J - I| * |Ix|: image
// samples carry 5 fraction bits (|J - I| <= 255 * 32) and a Scharr derivative of uint8 pixels is at most 16 * 255.
constexpr long long kFlowLanePixels = (kFlowMaxWin * kFlowMaxWin + 31) / 32;
static_assert(kFlowLanePixels * (255 * 32) * (16 * 255) < (1ll << 31),
              "k_flow_lk's per-lane int sums could overflow at kFlowMaxWin");

struct FlowLevel {
  int w, h;                                     // interior size
  long long img_off, der_off;                   // element offsets of the padded (h + 2 win) x (w + 2 win) level
};
struct FlowGeom {
  int win, n_levels;
  FlowLevel lv[kFlowMaxLevels];
};
struct FlowIn { float x, y; int slot, pad; };
struct FlowOut { float x, y, err; int status; };

__host__ __device__ inline int reflect101(int p, int n) {
  if (n == 1) return 0;
  while ((unsigned)p >= (unsigned)n) p = p < 0 ? -p : 2 * n - 2 - p;
  return p;
}

__device__ inline int gray_at(const uint8_t* f, int W, int C, int y, int x) {
  const uint8_t* p = f + ((size_t)y * W + x) * C;
  return C == 1 ? p[0] : (p[0] * 3735 + p[1] * 19235 + p[2] * 9798 + (1 << 14)) >> 15;
}

// level-0 interior from the uploaded frame: gray, then (half != 0) the 2x2 area reduction
__global__ void k_flow_level0(const uint8_t* __restrict__ frame, int H, int W, int C, int half, FlowGeom g,
                              uint8_t* __restrict__ img) {
  const FlowLevel L = g.lv[0];
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= L.w || y >= L.h) return;
  int v;
  if (!half) {
    v = gray_at(frame, W, C, y, x);
  } else if (2 * y + 2 <= H && 2 * x + 2 <= W) {
    v = (gray_at(frame, W, C, 2 * y, 2 * x) + gray_at(frame, W, C, 2 * y, 2 * x + 1) +
         gray_at(frame, W, C, 2 * y + 1, 2 * x) + gray_at(frame, W, C, 2 * y + 1, 2 * x + 1) + 2) >> 2;
  } else {
    int sum = 0, cnt = 0;
    for (int sy = 2 * y; sy < min(2 * y + 2, H); ++sy)
      for (int sx = 2 * x; sx < min(2 * x + 2, W); ++sx) { sum += gray_at(frame, W, C, sy, sx); ++cnt; }
    v = __float2int_rn(__fdiv_rn((float)sum, (float)cnt));
  }
  img[L.img_off + (long long)(y + g.win) * (L.w + 2 * g.win) + x + g.win] = (uint8_t)v;
}

// level l interior = pyrDown(level l - 1 interior)
__global__ void k_flow_pyrdown(FlowGeom g, int l, uint8_t* __restrict__ img) {
  const FlowLevel S = g.lv[l - 1], D = g.lv[l];
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= D.w || y >= D.h) return;
  const int k[5] = {1, 4, 6, 4, 1}, sp = S.w + 2 * g.win;
  const uint8_t* src = img + S.img_off + (long long)g.win * sp + g.win;
  int xs[5];
#pragma unroll
  for (int i = 0; i < 5; ++i) xs[i] = reflect101(2 * x - 2 + i, S.w);
  int sum = 0;
#pragma unroll
  for (int r = 0; r < 5; ++r) {
    const uint8_t* row = src + (long long)reflect101(2 * y - 2 + r, S.h) * sp;
    int s = 0;
#pragma unroll
    for (int i = 0; i < 5; ++i) s += k[i] * row[xs[i]];
    sum += k[r] * s;
  }
  img[D.img_off + (long long)(y + g.win) * (D.w + 2 * g.win) + x + g.win] = (uint8_t)((sum + 128) >> 8);
}

// over the padded level: interior pixels get their Scharr derivatives, border pixels the reflect-101 image value
// (the derivative border stays at the zeros it was allocated with)
__global__ void k_flow_finish(FlowGeom g, int l, uint8_t* __restrict__ img, short2* __restrict__ der) {
  const FlowLevel L = g.lv[l];
  const int win = g.win, pw = L.w + 2 * win;
  const int px = blockIdx.x * blockDim.x + threadIdx.x, py = blockIdx.y * blockDim.y + threadIdx.y;
  if (px >= pw || py >= L.h + 2 * win) return;
  uint8_t* base = img + L.img_off;
  const uint8_t* in = base + (long long)win * pw + win;
  const int x = px - win, y = py - win;
  if (x >= 0 && x < L.w && y >= 0 && y < L.h) {
    const uint8_t *r0 = in + (long long)reflect101(y - 1, L.h) * pw, *r1 = in + (long long)y * pw,
                  *r2 = in + (long long)reflect101(y + 1, L.h) * pw;
    const int xm = reflect101(x - 1, L.w), xp = reflect101(x + 1, L.w);
    const int vm = (r0[xm] + r2[xm]) * 3 + r1[xm] * 10, vp = (r0[xp] + r2[xp]) * 3 + r1[xp] * 10;
    const int dm = r2[xm] - r0[xm], d0 = r2[x] - r0[x], dp = r2[xp] - r0[xp];
    der[L.der_off + (long long)py * pw + px] = make_short2((short)(vp - vm), (short)((dp + dm) * 3 + d0 * 10));
  } else {
    base[(long long)py * pw + px] = in[(long long)reflect101(y, L.h) * pw + reflect101(x, L.w)];
  }
}

__device__ __forceinline__ long long warp_sum(long long v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void bilinear_weights(float a, float b, int& w00, int& w01, int& w10, int& w11) {
  w00 = __float2int_rn((1.f - a) * (1.f - b) * 16384.f);
  w01 = __float2int_rn(a * (1.f - b) * 16384.f);
  w10 = __float2int_rn((1.f - a) * b * 16384.f);
  w11 = 16384 - w00 - w01 - w10;
}

#define FLOW_DESCALE(x, n) (((x) + (1 << ((n) - 1))) >> (n))

// One warp per point; lanes stride over the win x win window.  Every lane reduces to the same sums (integer
// butterfly), so all control flow below is warp-uniform.
__global__ void __launch_bounds__(kFlowWarps * 32) k_flow_lk(FlowGeom g, const uint8_t* __restrict__ img,
                                                              const short2* __restrict__ der, long long img_stride,
                                                              long long der_stride, int cur_slot,
                                                              const FlowIn* __restrict__ in, FlowOut* __restrict__ out,
                                                              int n) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int pt = blockIdx.x * kFlowWarps + warp;
  if (pt >= n) return;
  const int win = g.win, area = win * win, area2 = (area + 1) & ~1;
  short* Iw = (short*)smem_raw + (size_t)warp * area2;                                  // I patch, 5 fraction bits
  short2* dIw = (short2*)((short*)smem_raw + (size_t)kFlowWarps * area2) + (size_t)warp * area;   // (Ix, Iy) patch
  const FlowIn p = in[pt];
  const uint8_t* Ibase = img + p.slot * img_stride;
  const short2* Dbase = der + p.slot * der_stride;
  const uint8_t* Jbase = img + cur_slot * img_stride;
  const float halfw = (win - 1) * 0.5f;
  const float FLT_SCALE = 1.f / (1 << 20);
  int status = 1;
  float err = 0.f, nx = 0.f, ny = 0.f;
  if (!isfinite(p.x) || !isfinite(p.y)) status = 0;
  for (int level = g.n_levels - 1; level >= 0 && status; --level) {
    const FlowLevel L = g.lv[level];
    const int pitch = L.w + 2 * win;
    const float sc = (float)(1.0 / (1 << level));
    float px = p.x * sc, py = p.y * sc;
    if (level == g.n_levels - 1) { nx = px; ny = py; } else { nx = nx * 2.f; ny = ny * 2.f; }
    px -= halfw; py -= halfw;
    const int ipx = (int)floorf(px), ipy = (int)floorf(py);
    if (ipx < -win || ipx >= L.w || ipy < -win || ipy >= L.h) {
      if (level == 0) { status = 0; err = 0.f; }
      continue;
    }
    int w00, w01, w10, w11;
    bilinear_weights(px - ipx, py - ipy, w00, w01, w10, w11);
    const uint8_t* I = Ibase + L.img_off + (long long)(ipy + win) * pitch + ipx + win;
    const short2* D = Dbase + L.der_off + (long long)(ipy + win) * pitch + ipx + win;
    int s11 = 0, s12 = 0, s22 = 0;
    for (int i = lane; i < area; i += 32) {
      const int y = i / win, x = i - y * win;
      const uint8_t* q = I + y * pitch + x;
      const short2* d = D + y * pitch + x;
      const short2 d00 = d[0], d01 = d[1], d10 = d[pitch], d11 = d[pitch + 1];
      const int iv = FLOW_DESCALE(q[0] * w00 + q[1] * w01 + q[pitch] * w10 + q[pitch + 1] * w11, 9);
      const int ix = FLOW_DESCALE(d00.x * w00 + d01.x * w01 + d10.x * w10 + d11.x * w11, 14);
      const int iy = FLOW_DESCALE(d00.y * w00 + d01.y * w01 + d10.y * w10 + d11.y * w11, 14);
      Iw[i] = (short)iv;
      dIw[i] = make_short2((short)ix, (short)iy);
      s11 += ix * ix; s12 += ix * iy; s22 += iy * iy;
    }
    const float A11 = (float)warp_sum(s11) * FLT_SCALE, A12 = (float)warp_sum(s12) * FLT_SCALE,
                A22 = (float)warp_sum(s22) * FLT_SCALE;
    float det = A11 * A22 - A12 * A12;
    const float min_eig = (A22 + A11 - sqrtf((A11 - A22) * (A11 - A22) + 4.f * A12 * A12)) / (float)(2 * area);
    if (min_eig < 1e-4f || det < FLT_EPSILON) {
      if (level == 0) status = 0;
      continue;
    }
    det = 1.f / det;
    float qx = nx - halfw, qy = ny - halfw, pdx = 0.f, pdy = 0.f;
    for (int j = 0; j < 30; ++j) {
      const int jx = (int)floorf(qx), jy = (int)floorf(qy);
      if (jx < -win || jx >= L.w || jy < -win || jy >= L.h) {
        if (level == 0) status = 0;
        break;
      }
      bilinear_weights(qx - jx, qy - jy, w00, w01, w10, w11);
      const uint8_t* J = Jbase + L.img_off + (long long)(jy + win) * pitch + jx + win;
      int b1 = 0, b2 = 0;
      for (int i = lane; i < area; i += 32) {
        const int y = i / win, x = i - y * win;
        const uint8_t* q = J + y * pitch + x;
        const int diff = FLOW_DESCALE(q[0] * w00 + q[1] * w01 + q[pitch] * w10 + q[pitch + 1] * w11, 9) - Iw[i];
        const short2 d = dIw[i];
        b1 += diff * d.x; b2 += diff * d.y;
      }
      const float B1 = (float)warp_sum(b1) * FLT_SCALE, B2 = (float)warp_sum(b2) * FLT_SCALE;
      const float dx = (A12 * B2 - A22 * B1) * det, dy = (A12 * B1 - A11 * B2) * det;
      qx += dx; qy += dy;
      nx = qx + halfw; ny = qy + halfw;
      if ((double)dx * dx + (double)dy * dy <= 0.01 * 0.01) break;
      if (j > 0 && (double)fabsf(dx + pdx) < 0.01 && (double)fabsf(dy + pdy) < 0.01) {
        nx -= dx * 0.5f; ny -= dy * 0.5f;
        break;
      }
      pdx = dx; pdy = dy;
    }
    if (status && level == 0) {
      const float ex = nx - halfw, ey = ny - halfw;
      const int jx = (int)floorf(ex), jy = (int)floorf(ey);
      if (jx < -win || jx >= L.w || jy < -win || jy >= L.h) {
        status = 0;
        break;
      }
      bilinear_weights(ex - jx, ey - jy, w00, w01, w10, w11);
      const uint8_t* J = Jbase + L.img_off + (long long)(jy + win) * pitch + jx + win;
      int e = 0;
      for (int i = lane; i < area; i += 32) {
        const int y = i / win, x = i - y * win;
        const uint8_t* q = J + y * pitch + x;
        e += abs(FLOW_DESCALE(q[0] * w00 + q[1] * w01 + q[pitch] * w10 + q[pitch + 1] * w11, 9) - Iw[i]);
      }
      err = (float)warp_sum(e) * 1.f / (float)(32 * area);
    }
  }
  if (lane == 0) out[pt] = FlowOut{nx, ny, err, status};
}

}  // namespace

struct SbFlow {
  int win = 0, max_levels = 0, half = 0, ring = 0;
  int H = 0, W = 0;                               // frame size the ring holds
  FlowGeom geom{};
  long long img_elems = 0, der_elems = 0;         // per slot: the slot stride of img and der
  uint8_t* img = nullptr;                         // ring * img_elems
  short2* der = nullptr;                          // ring * der_elems
  std::vector<long long> slot_t, stamp;           // frame index (-1: empty) and last use of every slot
  long long clock = 0;
  uint8_t* frame_dev = nullptr;
  size_t frame_cap = 0;
  FlowIn *in_dev = nullptr, *in_host = nullptr;   // host staging is page-locked: one async copy each way
  FlowOut *out_dev = nullptr, *out_host = nullptr;
  int cap = 0;

  void free_ring() {
    cudaFree(img); cudaFree(der);
    img = nullptr; der = nullptr;
    slot_t.clear(); stamp.clear();
    H = W = 0;
  }
  uint8_t* slot_img(int slot) const { return img + slot * img_elems; }
  short2* slot_der(int slot) const { return der + slot * der_elems; }
  ~SbFlow() {
    free_ring();
    cudaFree(frame_dev); cudaFree(in_dev); cudaFree(out_dev);
    cudaFreeHost(in_host); cudaFreeHost(out_host);
  }
  int find(long long t) const {
    for (int i = 0; i < (int)slot_t.size(); ++i)
      if (slot_t[i] == t) return i;
    return -1;
  }
};

void sb_flows_free(sb_handle_s* h) {
  for (SbFlow* f : h->flows) delete f;
  h->flows.clear();
}

namespace {

SbFlow* get_flow(sb_handle_s* h, int id) {
  return (id >= 0 && id < (int)h->flows.size()) ? h->flows[id] : nullptr;
}

// pyramid geometry of an (H, W) frame, cv2.buildOpticalFlowPyramid's level rule
int flow_alloc_ring(sb_handle_s* h, SbFlow* f, int H, int W) {
  f->free_ring();
  FlowGeom& g = f->geom;
  g.win = f->win;
  int w = f->half ? (int)std::nearbyint(W * 0.5) : W, hh = f->half ? (int)std::nearbyint(H * 0.5) : H;
  if (w < 1 || hh < 1) return sb_fail(h, SB_ERR_INVALID, "sb_flow_add_frame: frame %dx%d is too small", H, W);
  long long io = 0, dof = 0;
  g.n_levels = 0;
  for (int l = 0; l <= f->max_levels && l < kFlowMaxLevels; ++l) {
    g.lv[l] = FlowLevel{w, hh, io, dof};
    const long long padded = (long long)(w + 2 * g.win) * (hh + 2 * g.win);
    io += (padded + 15) & ~15ll;
    dof += (padded + 3) & ~3ll;
    g.n_levels = l + 1;
    w = (w + 1) / 2; hh = (hh + 1) / 2;
    if (w <= g.win || hh <= g.win) break;
  }
  f->img_elems = io; f->der_elems = dof;
  const size_t n_img = (size_t)io * f->ring, n_der = (size_t)dof * f->ring;
  int rc;
  if ((rc = sb_dev_alloc(h, &f->img, n_img)) || (rc = sb_dev_alloc(h, &f->der, n_der))) return rc;
  SB_CUDA(h, cudaMemsetAsync(f->der, 0, n_der * sizeof(short2), h->stream));
  f->slot_t.assign(f->ring, -1); f->stamp.assign(f->ring, -1);
  f->H = H; f->W = W;
  return SB_OK;
}

}  // namespace

extern "C" {

int sb_flow_create(sb_handle_t h, int window, int max_levels, float img_scale, int ring, int* out_flow_id) {
  if (!h || !out_flow_id) return sb_fail(h, SB_ERR_INVALID, "sb_flow_create: null argument");
  if (window < 3 || window > kFlowMaxWin) return sb_fail(h, SB_ERR_UNSUPPORTED, "sb_flow_create: window %d outside 3..%d", window, kFlowMaxWin);
  if (max_levels < 0) return sb_fail(h, SB_ERR_INVALID, "sb_flow_create: max_levels %d < 0", max_levels);
  if (img_scale != 1.f && img_scale != 0.5f)
    return sb_fail(h, SB_ERR_UNSUPPORTED, "sb_flow_create: img_scale %g (the device flow resizes by 1 or 0.5)", img_scale);
  if (ring < 2) return sb_fail(h, SB_ERR_UNSUPPORTED, "sb_flow_create: ring %d < 2", ring);
  SbFlow* f = new SbFlow();
  f->win = window; f->max_levels = max_levels; f->half = img_scale == 0.5f; f->ring = ring;
  h->flows.push_back(f);
  *out_flow_id = (int)h->flows.size() - 1;
  return SB_OK;
}

int sb_flow_destroy(sb_handle_t h, int flow_id) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  SbFlow* f = get_flow(h, flow_id);
  if (!f) return sb_fail(h, SB_ERR_INVALID, "sb_flow_destroy: no flow %d", flow_id);
  cudaSetDevice(h->device);
  cudaStreamSynchronize(h->stream);
  delete f;
  h->flows[flow_id] = nullptr;
  return SB_OK;
}

int sb_flow_add_frame(sb_handle_t h, int flow_id, int64_t t, const uint8_t* frame_host, int H, int W, int C,
                      int replace) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  SbFlow* f = get_flow(h, flow_id);
  if (!f) return sb_fail(h, SB_ERR_INVALID, "sb_flow_add_frame: no flow %d", flow_id);
  if (!frame_host || H <= 0 || W <= 0 || (C != 1 && C != 3))
    return sb_fail(h, SB_ERR_INVALID, "sb_flow_add_frame: frame (%d, %d, %d) must be uint8 with 1 or 3 channels", H, W, C);
  if (t < 0) return sb_fail(h, SB_ERR_INVALID, "sb_flow_add_frame: frame index %lld < 0", (long long)t);
  SB_CUDA(h, cudaSetDevice(h->device));
  int rc;
  if (H != f->H || W != f->W)
    if ((rc = flow_alloc_ring(h, f, H, W))) { f->free_ring(); return rc; }
  int slot = f->find(t);
  if (slot >= 0 && !replace) { f->stamp[slot] = ++f->clock; return SB_OK; }
  if (slot < 0) {                                    // an empty slot, else the least recently used one
    slot = 0;
    for (int i = 1; i < f->ring; ++i)
      if (f->stamp[i] < f->stamp[slot]) slot = i;
  }
  const size_t bytes = (size_t)H * W * C;
  if (bytes > f->frame_cap) {
    cudaFree(f->frame_dev);
    f->frame_dev = nullptr; f->frame_cap = 0;
    if ((rc = sb_dev_alloc(h, &f->frame_dev, bytes))) return rc;
    f->frame_cap = bytes;
  }
  f->slot_t[slot] = -1;                              // not readable until its pyramid is complete
  SB_CUDA(h, cudaMemcpyAsync(f->frame_dev, frame_host, bytes, cudaMemcpyHostToDevice, h->stream));
  const FlowGeom& g = f->geom;
  const dim3 blk(32, 8);
  auto grid = [&](int w, int hh) { return dim3((w + 31) / 32, (hh + 7) / 8); };
  k_flow_level0<<<grid(g.lv[0].w, g.lv[0].h), blk, 0, h->stream>>>(f->frame_dev, H, W, C, f->half, g, f->slot_img(slot));
  SB_CHECK_LAUNCH(h);
  for (int l = 0; l < g.n_levels; ++l) {
    if (l > 0) {
      k_flow_pyrdown<<<grid(g.lv[l].w, g.lv[l].h), blk, 0, h->stream>>>(g, l, f->slot_img(slot));
      SB_CHECK_LAUNCH(h);
    }
    k_flow_finish<<<grid(g.lv[l].w + 2 * g.win, g.lv[l].h + 2 * g.win), blk, 0, h->stream>>>(g, l, f->slot_img(slot),
                                                                                          f->slot_der(slot));
    SB_CHECK_LAUNCH(h);
  }
  f->slot_t[slot] = t;
  f->stamp[slot] = ++f->clock;
  return SB_OK;
}

int sb_flow_shift(sb_handle_t h, int flow_id, int64_t t, int n, const int64_t* ref_t, const float* pts,
                  float* out_pts, int32_t* out_status, float* out_err) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  SbFlow* f = get_flow(h, flow_id);
  if (!f) return sb_fail(h, SB_ERR_INVALID, "sb_flow_shift: no flow %d", flow_id);
  if (n < 0) return sb_fail(h, SB_ERR_INVALID, "sb_flow_shift: n = %d", n);
  if (n == 0) return SB_OK;
  if (!ref_t || !pts || !out_pts || !out_status || !out_err) return sb_fail(h, SB_ERR_INVALID, "sb_flow_shift: null buffer");
  const int cur = f->find(t);
  if (cur < 0) return sb_fail(h, SB_ERR_INVALID, "sb_flow_shift: frame %lld is not held", (long long)t);
  SB_CUDA(h, cudaSetDevice(h->device));
  int rc;
  if (n > f->cap) {
    cudaFree(f->in_dev); cudaFree(f->out_dev); cudaFreeHost(f->in_host); cudaFreeHost(f->out_host);
    f->in_dev = nullptr; f->out_dev = nullptr; f->in_host = nullptr; f->out_host = nullptr; f->cap = 0;
    const int cap = std::max(n, 256);
    if ((rc = sb_dev_alloc(h, &f->in_dev, cap)) || (rc = sb_dev_alloc(h, &f->out_dev, cap))) return rc;
    SB_CUDA(h, cudaHostAlloc((void**)&f->in_host, cap * sizeof(FlowIn), cudaHostAllocDefault));
    SB_CUDA(h, cudaHostAlloc((void**)&f->out_host, cap * sizeof(FlowOut), cudaHostAllocDefault));
    f->cap = cap;
  }
  f->stamp[cur] = ++f->clock;
  for (int i = 0; i < n; ++i) {
    const int s = f->find(ref_t[i]);
    if (s < 0) return sb_fail(h, SB_ERR_INVALID, "sb_flow_shift: reference frame %lld is not held", (long long)ref_t[i]);
    f->stamp[s] = f->clock;
    f->in_host[i] = FlowIn{pts[2 * i], pts[2 * i + 1], s, 0};
  }
  const int area2 = (f->win * f->win + 1) & ~1;
  const size_t smem = (size_t)kFlowWarps * (area2 * sizeof(short) + f->win * f->win * sizeof(short2));
  SB_CUDA(h, cudaMemcpyAsync(f->in_dev, f->in_host, n * sizeof(FlowIn), cudaMemcpyHostToDevice, h->stream));
  k_flow_lk<<<(n + kFlowWarps - 1) / kFlowWarps, kFlowWarps * 32, smem, h->stream>>>(
      f->geom, f->img, f->der, f->img_elems, f->der_elems, cur, f->in_dev, f->out_dev, n);
  SB_CHECK_LAUNCH(h);
  SB_CUDA(h, cudaMemcpyAsync(f->out_host, f->out_dev, n * sizeof(FlowOut), cudaMemcpyDeviceToHost, h->stream));
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  for (int i = 0; i < n; ++i) {
    out_pts[2 * i] = f->out_host[i].x;
    out_pts[2 * i + 1] = f->out_host[i].y;
    out_status[i] = f->out_host[i].status;
    out_err[i] = f->out_host[i].err;
  }
  return SB_OK;
}

int sb_flow_fetch_level(sb_handle_t h, int flow_id, int64_t t, int level, uint8_t* img_out, int16_t* deriv_out,
                        int* out_H, int* out_W, int* out_n_levels) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  SbFlow* f = get_flow(h, flow_id);
  if (!f) return sb_fail(h, SB_ERR_INVALID, "sb_flow_fetch_level: no flow %d", flow_id);
  const int slot = f->find(t);
  if (slot < 0) return sb_fail(h, SB_ERR_INVALID, "sb_flow_fetch_level: frame %lld is not held", (long long)t);
  const FlowGeom& g = f->geom;
  if (level < 0 || level >= g.n_levels)
    return sb_fail(h, SB_ERR_INVALID, "sb_flow_fetch_level: level %d outside 0..%d", level, g.n_levels - 1);
  SB_CUDA(h, cudaSetDevice(h->device));
  const FlowLevel L = g.lv[level];
  const size_t pw = L.w + 2 * g.win, first = (size_t)g.win * pw + g.win;
  if (img_out)
    SB_CUDA(h, cudaMemcpy2DAsync(img_out, L.w, f->slot_img(slot) + L.img_off + first, pw, L.w, L.h, cudaMemcpyDeviceToHost, h->stream));
  if (deriv_out)
    SB_CUDA(h, cudaMemcpy2DAsync(deriv_out, L.w * sizeof(short2), f->slot_der(slot) + L.der_off + first, pw * sizeof(short2),
                                 L.w * sizeof(short2), L.h, cudaMemcpyDeviceToHost, h->stream));
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  if (out_H) *out_H = L.h;
  if (out_W) *out_W = L.w;
  if (out_n_levels) *out_n_levels = g.n_levels;
  return SB_OK;
}

}  // extern "C"
