// Model engine: executes the flat op-list compiled from the reference's backbone + heads graph,
// and the fused predictors (bottom-up / single-instance / centered-instance / centroid) on top.
//
// Reference: sleap/nn/model.py:312-364 (graph topology), sleap/nn/inference.py:2864-3003
// (BottomUpInferenceLayer), :1319-1380 (SingleInstanceInferenceLayer), :1747-1966 (CentroidCrop),
// :2059-2200 (FindInstancePeaks).
#include <algorithm>

#include "sb_common.cuh"
#include "sb_kernels_direct.cuh"
#include "sb_model.h"

using namespace sbd;

namespace {

template <typename T> T* buf_ptr(const SbBuffer& b) { return (T*)b.dev; }

size_t elem_size(const SbModel* m, const SbBuffer& b) { return (b.f32 || m->precision == 1) ? 4 : 2; }

int grid_for(size_t total, int sm) {
  size_t g = (total + 255) / 256;
  size_t cap = (size_t)sm * 16;
  return (int)std::max<size_t>(1, std::min(g, cap));
}

int build_programs(sb_handle_s* h, SbModel* m);   // the last step of sb_model_configure (below, with the op slots)

}  // namespace

void sb_global_scratch_free(SbGlobalScratch& g) {
  for (float* p : {g.part, g.points, g.crop_off}) if (p) cudaFree(p);    // vals lives in the points block
  g = SbGlobalScratch();
}

int sb_global_scratch_alloc(sb_handle_s* h, SbGlobalScratch& g, int B, int H, int C) {
  const int target = (2 * h->sm_count + B - 1) / B;
  g.rpc = std::max(1, (H + target - 1) / target);
  g.chunks = (H + g.rpc - 1) / g.rpc;
  SB_CUDA(h, cudaMalloc((void**)&g.part, (size_t)B * g.chunks * C * 3 * 4));
  SB_CUDA(h, cudaMalloc((void**)&g.points, (size_t)B * C * 3 * 4));
  g.vals = g.points + (size_t)B * C * 2;
  SB_CUDA(h, cudaMalloc((void**)&g.crop_off, (size_t)B * 2 * 4));
  return 0;
}

void sb_models_free(sb_handle_s* h) {
  for (SbModel* m : h->models) {
    if (!m) continue;
    for (auto& b : m->buffers) if (b.dev) cudaFree(b.dev);
    if (m->weights_dev) cudaFree(m->weights_dev);
    if (m->weights_tc_dev) cudaFree(m->weights_tc_dev);
    if (m->frames_dev) cudaFree(m->frames_dev);
    sb_global_scratch_free(m->gs);
    if (m->trk_dev) cudaFree(m->trk_dev);
    for (int i = 0; i < 2; ++i) if (m->trk_host[i]) cudaFreeHost(m->trk_host[i]);
    m->slots.release();
    for (auto& e : m->fwd_events) cudaEventDestroy(e);
    sb_post_ws_free(m->ws);
    sb_gather_free(m);
    sb_topdown_free(m);
    for (auto& p : m->prog) p.clear();
    sb_entry_release(m);
    sb_conv_tc_release(m);
    delete m;
  }
  h->models.clear();
}

SbModel* chain_model(sb_handle_s* h, int id, int kind, const char* what) {
  SbModel* m = (h && id >= 0 && id < (int)h->models.size()) ? h->models[id] : nullptr;
  if (m && (kind == SB_CHAIN_ANY || m->chain == kind)) return m;
  sb_fail(h, SB_ERR_INVALID, "%s", what);
  return nullptr;
}

// Releases the model's post-processing chain and everything sized or attached for it; the only code that does.  The
// device is drained first: post-processing and result copies of earlier steps may still read the workspace.
static int chain_drop(sb_handle_s* h, SbModel* m) {
  SB_CUDA(h, cudaDeviceSynchronize());
  h->post_pending = false;
  sb_post_ws_free(m->ws);
  m->slots.release();                            // staging is sized from the chain's record width
  sb_gather_free(m);                             // window sizes depend on (B, max_instances, n_nodes)
  m->trk = nullptr;                              // its checks (nodes, instance capacity) were made against the old chain
  sb_global_scratch_free(m->gs);
  sb_topdown_free(m);
  m->chain = SB_CHAIN_NONE;
  ++m->chain_gen;
  return 0;
}

int sb_track_records_alloc(sb_handle_s* h, SbModel* m, int B, int I) {
  if (m->trk_B >= B && m->trk_I == I) return SB_OK;
  cudaFree(m->trk_dev); m->trk_dev = nullptr;
  for (int i = 0; i < 2; ++i) { cudaFreeHost(m->trk_host[i]); m->trk_host[i] = nullptr; }
  m->trk_B = 0;
  const size_t n = (size_t)B * sb_track_record_width(I);
  int rc;
  if ((rc = sb_dev_alloc(h, &m->trk_dev, n))) return rc;
  for (int i = 0; i < 2; ++i) SB_CUDA(h, cudaHostAlloc((void**)&m->trk_host[i], n * sizeof(double), cudaHostAllocDefault));
  m->trk_B = B; m->trk_I = I;
  return SB_OK;
}

// The model a per-model configure call sets up: a valid id, non-null params and a configured network
static SbModel* configure_target(sb_handle_s* h, int id, const void* p) {
  SbModel* m = chain_model(h, id, SB_CHAIN_ANY, "bad model id / params");
  if (!m || !p) { sb_fail(h, SB_ERR_INVALID, "bad model id / params"); return nullptr; }
  if (!m->configured) { sb_fail(h, SB_ERR_INVALID, "call sb_model_configure first"); return nullptr; }
  return m;
}

int sb_net_size(sb_handle_s* h, const SbModel* m, int H, int W, int* Hres, int* Wres, int* Hnet, int* Wnet) {
  const SbOp* pre = nullptr;
  for (auto& op : m->ops) if (op.kind() == SB_OPK_PREPROCESS) { pre = &op; break; }
  if (!pre) return sb_fail(h, SB_ERR_INVALID, "model has no preprocess op");
  const float input_scale = pre->input_scale();
  const int pad_stride = std::max(1, pre->pad_stride());
  *Hres = H; *Wres = W;
  if (input_scale != 1.0f) { *Wres = (int)((float)W * input_scale); *Hres = (int)((float)H * input_scale); }
  *Hnet = ((*Hres + pad_stride - 1) / pad_stride) * pad_stride;
  *Wnet = ((*Wres + pad_stride - 1) / pad_stride) * pad_stride;
  return 0;
}

extern "C" {

int sb_load_model(sb_handle_t h, const int32_t* ops, int n_ops, const float* weights, int64_t n_weights,
                  int precision, int* out_model_id) {
  if (!h) return sb_fail(nullptr, SB_ERR_INVALID, "null handle");
  if (!ops || n_ops <= 0 || !weights || n_weights <= 0 || !out_model_id)
    return sb_fail(h, SB_ERR_INVALID, "sb_load_model: bad arguments");
  if (precision < 0 || precision > 2) return sb_fail(h, SB_ERR_INVALID, "precision must be 0 (fp16), 1 (fp32 CUDA cores) or 2 (split fp16 on the tensor cores)");
  SB_CUDA(h, cudaSetDevice(h->device));
  SbModel* m = new SbModel();
  m->precision = precision;
  m->n_weights = n_weights;
  for (int i = 0; i < n_ops; ++i) {
    const int32_t* w = ops + (size_t)i * SB_OP_WORDS;
    if (w[0] == SB_OPK_BUFFER) {
      SbBuffer b;
      b.id = w[1]; b.stride_den = w[2]; b.C = w[3]; b.f32 = w[4]; b.is_input = w[5];
      if (b.id != (int)m->buffers.size()) { delete m; return sb_fail(h, SB_ERR_INVALID, "buffer ids must be dense and ordered"); }
      if (b.stride_den <= 0 || b.C <= 0) { delete m; return sb_fail(h, SB_ERR_INVALID, "bad buffer record"); }
      m->buffers.push_back(b);
    } else {
      SbOp op;
      memcpy(op.w, w, sizeof(op.w));
      const int nb = (int)m->buffers.size();
      auto okbuf = [&](int id) { return id >= 0 && id < nb; };
      if (op.kind() < SB_OPK_CONV || op.kind() > SB_OPK_COPY) { delete m; return sb_fail(h, SB_ERR_INVALID, "op %d: unknown kind %d", i, op.kind()); }
      if (!okbuf(op.out_buf()) || (op.kind() != SB_OPK_PREPROCESS && !okbuf(op.in_buf()))) { delete m; return sb_fail(h, SB_ERR_INVALID, "op %d: bad buffer id", i); }
      if (op.kind() == SB_OPK_ADD && !okbuf(op.in2_buf())) { delete m; return sb_fail(h, SB_ERR_INVALID, "op %d: bad second input", i); }
      if (op.kind() == SB_OPK_CONV && op.residual() && (!okbuf(op.res_buf()) || !okbuf(op.sum_buf()))) {
        delete m; return sb_fail(h, SB_ERR_INVALID, "op %d: bad residual buffer id", i);
      }
      if (op.kind() == SB_OPK_CONV && op.explicit_pad() && (op.pad_top() < 0 || op.pad_left() < 0 || op.pad_top() >= op.k() || op.pad_left() >= op.k())) {
        delete m; return sb_fail(h, SB_ERR_INVALID, "op %d: bad explicit padding", i);
      }
      if (op.kind() == SB_OPK_TCONV && op.k() != 3 && op.k() != 4) { delete m; return sb_fail(h, SB_ERR_INVALID, "op %d: transposed conv kernel %d (3 or 4)", i, op.k()); }
      if (op.kind() == SB_OPK_POOL && op.k() != 0 && op.k() != 3) { delete m; return sb_fail(h, SB_ERR_INVALID, "op %d: bad pool kind", i); }
      if (op.kind() == SB_OPK_PREPROCESS && (op.pre_mode() < SB_PRE_PLAIN || op.pre_mode() > SB_PRE_IMAGENET_CAFFE_GRAY)) {
        delete m; return sb_fail(h, SB_ERR_INVALID, "op %d: bad preprocess mode", i);
      }
      if (op.kind() == SB_OPK_PREPROCESS && std::any_of(m->ops.begin(), m->ops.end(), [](const SbOp& o) { return o.kind() == SB_OPK_PREPROCESS; })) {
        delete m; return sb_fail(h, SB_ERR_INVALID, "op %d: a second preprocess op", i);
      }
      auto okoff = [&](int off, int64_t n) { return off < 0 ? true : (int64_t)off + n <= n_weights; };
      if (op.kind() == SB_OPK_CONV || op.kind() == SB_OPK_TCONV) {
        const int64_t nw = (int64_t)op.k() * op.k() * op.in_C() * op.out_C();
        if (op.w_off() < 0 || !okoff(op.w_off(), nw) || !okoff(op.b_off(), op.out_C()) ||
            !okoff(op.bn_scale_off(), op.out_C()) || !okoff(op.bn_shift_off(), op.out_C())) {
          delete m; return sb_fail(h, SB_ERR_INVALID, "op %d: weight offsets out of range", i);
        }
      }
      m->ops.push_back(op);
    }
  }
  if (m->buffers.empty() || m->ops.empty()) { delete m; return sb_fail(h, SB_ERR_INVALID, "empty model"); }
  cudaError_t e = cudaMalloc((void**)&m->weights_dev, (size_t)n_weights * sizeof(float));
  if (e != cudaSuccess) { delete m; return sb_fail(h, SB_ERR_CUDA, "cudaMalloc weights: %s", cudaGetErrorString(e)); }
  e = cudaMemcpy(m->weights_dev, weights, (size_t)n_weights * sizeof(float), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) { cudaFree(m->weights_dev); delete m; return sb_fail(h, SB_ERR_CUDA, "copy weights: %s", cudaGetErrorString(e)); }
  m->weights_host.assign(weights, weights + n_weights);
  h->models.push_back(m);
  *out_model_id = (int)h->models.size() - 1;
  return SB_OK;
}

int sb_model_configure(sb_handle_t h, int model_id, int max_batch, int H, int W, int C_in) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_ANY, "bad model id");
  if (!m) return SB_ERR_INVALID;
  if (max_batch <= 0 || H <= 0 || W <= 0 || (C_in != 1 && C_in != 3)) return sb_fail(h, SB_ERR_INVALID, "sb_model_configure: bad shape");
  SB_CUDA(h, cudaSetDevice(h->device));
  int Hres, Wres, Hnet, Wnet;                  // the preprocess op defines the net input size
  if (const int rc = sb_net_size(h, m, H, W, &Hres, &Wres, &Hnet, &Wnet)) return rc;
  for (auto& b : m->buffers) {
    if (Hnet % b.stride_den || Wnet % b.stride_den)
      return sb_fail(h, SB_ERR_INVALID, "net input %dx%d not divisible by stride %d (pad_to_stride too small)", Hnet, Wnet, b.stride_den);
  }
  // a reconfigure invalidates everything sized from the old shape: the post-processing chain (its configure call must be
  // repeated; the C-ABI refuses to run a chain the model does not have), then the activation buffers and the plans
  if (const int rc = chain_drop(h, m)) return rc;
  for (auto& b : m->buffers) { if (b.dev) { cudaFree(b.dev); b.dev = nullptr; } }
  if (m->frames_dev) { cudaFree(m->frames_dev); m->frames_dev = nullptr; }
  m->configured = false;
  for (auto& p : m->prog) p.clear();             // the programs refer to the plans
  sb_entry_release(m);
  sb_conv_tc_release(m);
  m->B = max_batch; m->Hin = H; m->Win = W; m->Cin = C_in; m->Hres = Hres; m->Wres = Wres; m->Hnet = Hnet; m->Wnet = Wnet;
  size_t total = 0;
  for (auto& b : m->buffers) {
    b.H = Hnet / b.stride_den; b.W = Wnet / b.stride_den;
    const size_t bytes = (size_t)max_batch * b.H * b.W * b.C * elem_size(m, b);
    cudaError_t e = cudaMalloc(&b.dev, bytes + 256);
    if (e != cudaSuccess) return sb_fail(h, SB_ERR_CUDA, "cudaMalloc buffer %d (%zu B): %s", b.id, bytes, cudaGetErrorString(e));
    total += bytes;
  }
  m->act_bytes = total;
  SB_CUDA(h, cudaMalloc(&m->frames_dev, (size_t)max_batch * H * W * C_in * sizeof(float)));
  int rc = sb_conv_tc_prepare(h, m);
  if (!rc) rc = sb_entry_prepare(h, m);
  if (!rc) rc = sb_conv_tc_autotune(h, m);
  if (!rc) rc = sb_entry_autotune(h, m);
  if (!rc) rc = build_programs(h, m);
  if (rc) return rc;
  m->configured = true;
  return SB_OK;
}

}  // extern "C"

// ------------------------------------------------------------------------------------------
// The slots of the generic ops, in the activation type T of the model's precision.  Precision 2 keeps the preprocessed
// frame in fp32 and its activations as split-fp16 [lo | hi | hi] channel planes (sb_kernels_direct.cuh).
namespace {

template <typename TO>
SbLaunchFn preprocess_entry(const SbModel* m, const SbOp& op, const SbBuffer& ob) {
  const int Hin = m->Hin, Win = m->Win, Cin = m->Cin, Hres = m->Hres, Wres = m->Wres;
  const int resize = op.input_scale() != 1.0f;
  int mode_ch = 0;
  if (Cin == 3 && (ob.C == 1 || op.pre_mode() == SB_PRE_IMAGENET_CAFFE_GRAY)) mode_ch = 1;
  if (Cin == 1 && ob.C == 3) mode_ch = 2;
  const int imagenet = op.pre_mode() != SB_PRE_PLAIN;
  return [=](sb_handle_s* h, const void* frames_dev, int frames_are_u8, int B) {
    const size_t total = (size_t)B * ob.H * ob.W * ob.C;
    if (frames_are_u8)
      k_preprocess<unsigned char, TO><<<grid_for(total, h->sm_count), 256, 0, h->stream>>>(
          (const unsigned char*)frames_dev, Hin, Win, Cin, (TO*)ob.dev, ob.H, ob.W, ob.C, Hres, Wres, resize, mode_ch, 1, total, imagenet);
    else
      k_preprocess<float, TO><<<grid_for(total, h->sm_count), 256, 0, h->stream>>>(
          (const float*)frames_dev, Hin, Win, Cin, (TO*)ob.dev, ob.H, ob.W, ob.C, Hres, Wres, resize, mode_ch, 0, total, imagenet);
    SB_CHECK_LAUNCH(h);
    return 0;
  };
}

template <typename TI, typename TO>
int conv_entry(sb_handle_s* h, const SbModel* m, const SbOp& op, int osplit, SbLaunchFn& slot) {
  const SbBuffer& ib = m->buffers[op.in_buf()];
  const SbBuffer& ob = m->buffers[op.out_buf()];
  const int k = op.k(), st = op.stride();
  const int tot_h = std::max((ob.H - 1) * st + k - ib.H, 0), tot_w = std::max((ob.W - 1) * st + k - ib.W, 0);
  const int pad_top = op.explicit_pad() ? op.pad_top() : tot_h / 2, pad_left = op.explicit_pad() ? op.pad_left() : tot_w / 2;
  const float* W = m->weights_dev + op.w_off();
  const float* bias = op.b_off() >= 0 ? m->weights_dev + op.b_off() : nullptr;
  const float* bs = (op.flags() & SB_OPF_BN) ? m->weights_dev + op.bn_scale_off() : nullptr;
  const float* bh = (op.flags() & SB_OPF_BN) ? m->weights_dev + op.bn_shift_off() : nullptr;
  const int in_tile = (DC_TILE - 1) * st + k;
  const size_t sm = ((size_t)in_tile * in_tile * DC_CK + (size_t)k * k * DC_CK * DC_CO) * sizeof(float);
  const dim3 g(((ob.W + DC_TILE - 1) / DC_TILE) * ((ob.H + DC_TILE - 1) / DC_TILE), (op.out_C() + DC_CO - 1) / DC_CO);
  const int relu = (op.flags() & SB_OPF_RELU) ? 1 : 0;
  auto kern = k_conv_direct<TI, TO>;
  if (sm > 48 * 1024) {          // raised, never lowered: other ops and models launch this instantiation with their own sizes
    cudaFuncAttributes fa;
    SB_CUDA(h, cudaFuncGetAttributes(&fa, kern));
    if ((int)sm > fa.maxDynamicSharedSizeBytes) SB_CUDA(h, cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
  }
  slot = [=](sb_handle_s* h, const void*, int, int B) {
    kern<<<dim3(g.x, g.y, B), 256, sm, h->stream>>>((const TI*)ib.dev, ib.H, ib.W, ib.C, op.in_coff(), op.in_C(), (TO*)ob.dev, ob.H, ob.W,
                                                    ob.C, op.out_coff(), op.out_C(), W, bias, bs, bh, k, st, pad_top, pad_left, relu, osplit);
    SB_CHECK_LAUNCH(h);
    return 0;
  };
  return 0;
}

// The slot of a generic op: one that has no tensor-core plan and that the input stage does not cover.
template <typename T>
int op_entry_t(sb_handle_s* h, const SbModel* m, const SbOp& op, SbLaunchFn& slot) {
  const bool split = m->precision == 2;
  const SbBuffer& ob = m->buffers[op.out_buf()];
  const SbBuffer ib = op.kind() == SB_OPK_PREPROCESS ? SbBuffer() : m->buffers[op.in_buf()];
  const SbBuffer ib2 = op.kind() == SB_OPK_ADD ? m->buffers[op.in2_buf()] : SbBuffer();
  // POOL, UPSAMPLE, ADD in precision 2: the record carries the physical channel count (3C); the split kernels work on
  // logical channels
  const int C = split ? op.in_C() / 3 : op.in_C();
  const int relu = (op.flags() & SB_OPF_RELU) ? 1 : 0;
  const float* W = m->weights_dev + op.w_off();
  const float* bias = op.b_off() >= 0 ? m->weights_dev + op.b_off() : nullptr;
  switch (op.kind()) {
    case SB_OPK_PREPROCESS:
      if (op.pre_mode() != SB_PRE_PLAIN && ob.C != 3) return sb_fail(h, SB_ERR_INVALID, "ImageNet preprocessing needs a 3-channel network input");
      slot = (ob.f32 && sizeof(T) == 2) ? preprocess_entry<float>(m, op, ob) : preprocess_entry<T>(m, op, ob);
      return 0;
    case SB_OPK_CONV: {
      const int osplit = (split && !ob.f32) ? op.out_C() : 0;
      if (ib.f32 && sizeof(T) == 2) {              // precision 2: first conv straight from the fp32 preprocessed frame
        if (ob.f32) return sb_fail(h, SB_ERR_INVALID, "conv from the fp32 input buffer to an fp32 head is not supported in precision 2");
        return conv_entry<float, __half>(h, m, op, osplit, slot);
      }
      if (ob.f32 && sizeof(T) == 2) return conv_entry<T, float>(h, m, op, 0, slot);
      return conv_entry<T, T>(h, m, op, osplit, slot);
    }
    case SB_OPK_TCONV:
      slot = [=](sb_handle_s* h, const void*, int, int B) {
        dim3 g((ob.H * ob.W + 255) / 256, (op.out_C() + DC_CO - 1) / DC_CO, B);
        k_tconv_direct<T, T><<<g, 256, 0, h->stream>>>((const T*)ib.dev, ib.H, ib.W, ib.C, op.in_coff(), op.in_C(), (T*)ob.dev, ob.C,
                                                       op.out_coff(), op.out_C(), W, bias, relu, split ? op.out_C() : 0, op.k());
        SB_CHECK_LAUNCH(h);
        return 0;
      };
      return 0;
    case SB_OPK_POOL:
      slot = [=](sb_handle_s* h, const void*, int, int B) {
        const size_t total = (size_t)B * ob.H * ob.W * C;
        const int grid = grid_for(total, h->sm_count);
        if (op.k() == 3) {                      // ResNet stem: zero padding 1, 3x3 window, stride 2
          if (split)
            k_maxpool3s2_split<<<grid, 256, 0, h->stream>>>((const __half*)ib.dev, ib.H, ib.W, ib.C, op.in_coff(), C, (__half*)ob.dev, ob.H,
                                                            ob.W, ob.C, op.out_coff(), total);
          else
            k_maxpool3s2<T><<<grid, 256, 0, h->stream>>>((const T*)ib.dev, ib.H, ib.W, ib.C, op.in_coff(), C, (T*)ob.dev, ob.H, ob.W, ob.C,
                                                         op.out_coff(), total);
        } else if (split)
          k_maxpool2_split<<<grid, 256, 0, h->stream>>>((const __half*)ib.dev, ib.H, ib.W, ib.C, op.in_coff(), C, (__half*)ob.dev, ob.H, ob.W,
                                                        ob.C, op.out_coff(), total);
        else
          k_maxpool2<T><<<grid, 256, 0, h->stream>>>((const T*)ib.dev, ib.H, ib.W, ib.C, op.in_coff(), C, (T*)ob.dev, ob.H, ob.W, ob.C,
                                                     op.out_coff(), total);
        SB_CHECK_LAUNCH(h);
        return 0;
      };
      return 0;
    case SB_OPK_UPSAMPLE:
      slot = [=](sb_handle_s* h, const void*, int, int B) {
        const size_t total = (size_t)B * ob.H * ob.W * C;
        const int bilinear = (op.flags() & SB_OPF_BILINEAR) ? 1 : 0;
        if (split)
          k_upsample2_split<<<grid_for(total, h->sm_count), 256, 0, h->stream>>>((const __half*)ib.dev, ib.H, ib.W, ib.C, op.in_coff(), C,
                                                                                 (__half*)ob.dev, ob.C, op.out_coff(), bilinear, total);
        else
          k_upsample2<T><<<grid_for(total, h->sm_count), 256, 0, h->stream>>>((const T*)ib.dev, ib.H, ib.W, ib.C, op.in_coff(), C,
                                                                              (T*)ob.dev, ob.C, op.out_coff(), bilinear, total);
        SB_CHECK_LAUNCH(h);
        return 0;
      };
      return 0;
    case SB_OPK_ADD:
      slot = [=](sb_handle_s* h, const void*, int, int B) {
        const size_t npix = (size_t)B * ob.H * ob.W;
        if (split)
          k_add_split<<<grid_for(npix * C, h->sm_count), 256, 0, h->stream>>>((const __half*)ib.dev, ib.C, op.in_coff(), (const __half*)ib2.dev,
                                                                              ib2.C, op.in2_coff(), (__half*)ob.dev, ob.C, op.out_coff(), C, npix, relu);
        else
          k_add<T><<<grid_for(npix * C, h->sm_count), 256, 0, h->stream>>>((const T*)ib.dev, ib.C, op.in_coff(), (const T*)ib2.dev, ib2.C,
                                                                           op.in2_coff(), (T*)ob.dev, ob.C, op.out_coff(), C, npix, relu);
        SB_CHECK_LAUNCH(h);
        return 0;
      };
      return 0;
    case SB_OPK_COPY:
      slot = [=](sb_handle_s* h, const void*, int, int B) {
        const size_t npix = (size_t)B * ob.H * ob.W;
        k_copy<T><<<grid_for(npix * op.in_C(), h->sm_count), 256, 0, h->stream>>>((const T*)ib.dev, ib.C, op.in_coff(), (T*)ob.dev, ob.C,
                                                                                  op.out_coff(), op.in_C(), npix);
        SB_CHECK_LAUNCH(h);
        return 0;
      };
      return 0;
    default:
      return sb_fail(h, SB_ERR_INVALID, "unknown op kind %d", op.kind());
  }
}

// Both programs, one slot per op: the input stage's slots first, then each tensor-core conv (and the POOL or ADD slot it
// absorbs), then the generic ops.  Also the per-op kinds and the buffers the production program may not store.
int build_programs(sb_handle_s* h, SbModel* m) {
  const size_t n = m->ops.size();
  m->op_kind.assign(n, 0);
  for (size_t oi = 0; oi < n; ++oi)
    if (m->ops[oi].kind() == SB_OPK_CONV || m->ops[oi].kind() == SB_OPK_TCONV) m->op_kind[oi] = m->tc_plans[oi] ? 1 : 2;
  m->buf_elided.assign(m->buffers.size(), 0);
  for (int all_stores = 0; all_stores < 2; ++all_stores) {
    m->prog[all_stores].assign(n, nullptr);
    std::vector<char> taken(n, 0);
    sb_entry_build(m, all_stores, taken);
    for (size_t oi = 0; oi < n; ++oi) {
      if (taken[oi]) continue;
      if (m->tc_plans[oi]) {
        const SbTcEntry e = sb_conv_tc_entry(m, (int)oi, all_stores);
        m->prog[all_stores][oi] = e.run;
        if (e.absorbs >= 0) taken[e.absorbs] = 1;
        if (e.elides_out) m->buf_elided[m->ops[oi].out_buf()] = 1;
        continue;
      }
      const int rc = m->precision == 1 ? op_entry_t<float>(h, m, m->ops[oi], m->prog[all_stores][oi])
                                       : op_entry_t<__half>(h, m, m->ops[oi], m->prog[all_stores][oi]);
      if (rc) return rc;
    }
  }
  return 0;
}

// One forward pass of `prog`: per op its profiling event, the wait before the first op that overwrites a head buffer the
// post-processing stream may still read, then its slot.
int run_program(sb_handle_s* h, SbModel* m, const std::vector<SbLaunchFn>& prog, const void* frames_dev, int frames_are_u8, int B) {
  cudaStream_t s = h->stream;
  for (size_t oi = 0; oi < prog.size(); ++oi) {
    if (!m->prof_events.empty()) cudaEventRecord(m->prof_events[oi], s);
    if ((int)oi == m->guard_op && h->post_pending) SB_CUDA(h, cudaStreamWaitEvent(s, h->post_done_ev, 0));
    if (prog[oi])
      if (const int rc = prog[oi](h, frames_dev, frames_are_u8, B)) return rc;
  }
  if (!m->prof_events.empty()) cudaEventRecord(m->prof_events[prog.size()], s);
  return 0;
}

}  // namespace

int sb_run_ops(sb_handle_s* h, SbModel* m, const void* frames_dev, int frames_are_u8, int B, bool all_stores) {
  if (!m->configured) return sb_fail(h, SB_ERR_INVALID, "model not configured");
  if (B <= 0 || B > m->B) return sb_fail(h, SB_ERR_INVALID, "batch %d exceeds configured max %d", B, m->B);
  const bool timed = m->fwd_timing && 2 * (m->fwd_n + 1) <= (int)m->fwd_events.size();
  if (timed) cudaEventRecord(m->fwd_events[2 * m->fwd_n], h->stream);
  const int rc = run_program(h, m, m->prog[all_stores], frames_dev, frames_are_u8, B);
  if (timed) { cudaEventRecord(m->fwd_events[2 * m->fwd_n + 1], h->stream); ++m->fwd_n; }
  return rc;
}

__global__ void k_half_to_float(const __half* __restrict__ in, float* __restrict__ out, size_t n) {
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < n; t += (size_t)gridDim.x * blockDim.x)
    out[t] = __half2float(in[t]);
}

static int upload_frames(sb_handle_s* h, SbModel* m, const void* images_host, int is_u8, int B) {
  const size_t bytes = (size_t)B * m->Hin * m->Win * m->Cin * (is_u8 ? 1 : 4);
  SB_CUDA(h, cudaMemcpyAsync(m->frames_dev, images_host, bytes, cudaMemcpyHostToDevice, h->stream));
  return 0;
}

extern "C" {

int sb_model_forward(sb_handle_t h, int model_id, const void* images_host, int images_are_u8, int B,
                     int n_outputs, const int32_t* output_buffer_ids, float** out_host_ptrs) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_ANY, "bad model id");
  if (!m) return SB_ERR_INVALID;
  SB_CUDA(h, cudaSetDevice(h->device));
  if (!m->configured) return sb_fail(h, SB_ERR_INVALID, "model not configured");
  if (B <= 0 || B > m->B) return sb_fail(h, SB_ERR_INVALID, "bad batch");
  int rc = upload_frames(h, m, images_host, images_are_u8, B);
  if (rc) return rc;
  bool all_stores = false;                               // a tensor nobody reads inside the graph is only written on request
  for (int i = 0; i < n_outputs; ++i) {
    const int id = output_buffer_ids[i];
    if (id >= 0 && id < (int)m->buffers.size() && m->buf_elided[id]) all_stores = true;
  }
  if ((rc = sb_run_ops(h, m, m->frames_dev, images_are_u8, B, all_stores))) return rc;
  for (int i = 0; i < n_outputs; ++i) {
    const int id = output_buffer_ids[i];
    if (id < 0 || id >= (int)m->buffers.size()) return sb_fail(h, SB_ERR_INVALID, "bad output buffer id %d", id);
    SbBuffer& b = m->buffers[id];
    const size_t n = (size_t)B * b.H * b.W * b.C;
    if (elem_size(m, b) == 4) {
      SB_CUDA(h, cudaMemcpyAsync(out_host_ptrs[i], b.dev, n * 4, cudaMemcpyDeviceToHost, h->stream));
    } else {
      float* tmp = nullptr;
      SB_CUDA(h, cudaMalloc((void**)&tmp, n * 4));
      k_half_to_float<<<grid_for(n, h->sm_count), 256, 0, h->stream>>>((const __half*)b.dev, tmp, n);
      h->gpu_launches++;
      cudaError_t e = cudaMemcpyAsync(out_host_ptrs[i], tmp, n * 4, cudaMemcpyDeviceToHost, h->stream);
      cudaStreamSynchronize(h->stream);
      cudaFree(tmp);
      if (e != cudaSuccess) return sb_fail(h, SB_ERR_CUDA, "copy out: %s", cudaGetErrorString(e));
    }
  }
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  return SB_OK;
}

// Per-op device timing of one forward pass (CUDA events on the launching stream); used by
// bench.py for the roofline of the conv kernels.  out_ms[i] = duration of op i; out_kind[i] =
// 0 other, 1 tensor-core conv, 2 CUDA-core conv; out_flops[i] = 2*MACs of the op for batch B.
int sb_model_profile_ops(sb_handle_t h, int model_id, const uint8_t* frames_dev, int B, int cap, float* out_ms,
                         int32_t* out_kind, double* out_flops, int32_t* out_n_ops) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_ANY, "model not configured");
  if (!m || !m->configured) return sb_fail(h, SB_ERR_INVALID, "model not configured");
  SB_CUDA(h, cudaSetDevice(h->device));
  const int n = (int)m->ops.size();
  if (cap < n) return sb_fail(h, SB_ERR_INVALID, "capacity %d < n_ops %d", cap, n);
  m->prof_events.resize(n + 1);
  for (auto& e : m->prof_events) SB_CUDA(h, cudaEventCreate(&e));
  int rc = sb_run_ops(h, m, frames_dev, 1, B);
  cudaStreamSynchronize(h->stream);
  for (int i = 0; i < n && !rc; ++i) {
    cudaEventElapsedTime(&out_ms[i], m->prof_events[i], m->prof_events[i + 1]);
    const SbOp& op = m->ops[i];
    out_kind[i] = m->op_kind[i]; out_flops[i] = 0.0;
    if (op.kind() == SB_OPK_CONV || op.kind() == SB_OPK_TCONV) {
      const SbBuffer& ib = m->buffers[op.in_buf()];
      const SbBuffer& ob = m->buffers[op.out_buf()];
      const double pix = op.kind() == SB_OPK_TCONV ? (double)ib.H * ib.W : (double)ob.H * ob.W;
      out_flops[i] = 2.0 * op.k() * op.k() * op.in_C() * op.out_C() * pix * B;
    }
  }
  for (auto& e : m->prof_events) cudaEventDestroy(e);
  m->prof_events.clear();
  *out_n_ops = n;
  return rc;
}

int sb_model_forward_times(sb_handle_t h, int model_id, int enable, int cap, float* out_ms, int32_t* out_n) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_ANY, "bad model id");
  if (!m) return SB_ERR_INVALID;
  SB_CUDA(h, cudaSetDevice(h->device));
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  int n = 0;
  for (; n < m->fwd_n && n < cap && out_ms; ++n)
    SB_CUDA(h, cudaEventElapsedTime(&out_ms[n], m->fwd_events[2 * n], m->fwd_events[2 * n + 1]));
  if (out_n) *out_n = n;
  m->fwd_n = 0;
  if (enable && m->fwd_events.empty()) {
    m->fwd_events.resize(2 * 1024);
    for (auto& e : m->fwd_events) SB_CUDA(h, cudaEventCreate(&e));
  }
  m->fwd_timing = enable != 0;
  return SB_OK;
}

}  // extern "C"

// ---------------------------------- bottom-up ------------------------------------------------
// A model's bottom-up step runs one post-processing chain: the PAF chain (sb_bottomup_configure) or the multi-class
// chain (sb_multiclass_configure).  Both share the workspace, the result records, the pinned staging, the copy stream
// and the slot events; what differs is the record width and the kernels queued after the network.

// The first op that overwrites one of the head buffers the post-processing reads (-1: none, or SB_DISABLE_POST_OVERLAP):
// the network of the next step waits for the previous step's post-processing right before it.
static int post_guard_op(const SbModel* m, int b0, int b1, int b2) {
  if (getenv("SB_DISABLE_POST_OVERLAP")) return -1;
  for (size_t i = 0; i < m->ops.size(); ++i) {
    const int ob = m->ops[i].out_buf();
    if (ob == b0 || ob == b1 || (b2 >= 0 && ob == b2)) return (int)i;
  }
  return -1;
}

// Floats per frame of the chain's result block: its records, or for the global chain points and values (the block is
// [B][C][2] points | [B][C] values at the configured B, one copy of the whole block)
static size_t record_width(const SbModel* m) {
  if (m->chain == SB_CHAIN_GLOBAL) return (size_t)m->buffers[m->gl.cms_buffer].C * 3;
  return m->chain == SB_CHAIN_CLASS ? sb_class_record_width(m->mc.n_classes, m->mc.n_nodes) : sb_record_width(m->bu.max_instances, m->bu.n_nodes);
}

// One map a chain reads: device pointer and NHWC shape (a head buffer, or a from-maps call's upload)
struct SbMap {
  const float* dev;
  int H, W, C;
};
static SbMap head_map(const SbModel* m, int buf) {
  const SbBuffer& b = m->buffers[buf];
  return {(const float*)b.dev, b.H, b.W, b.C};
}
static const float* head_offsets(const SbModel* m, int buf) { return buf >= 0 ? (const float*)m->buffers[buf].dev : nullptr; }

// A head buffer id a configure call names: in range, an f32 head output of C channels
static bool f32_head(const SbModel* m, int buf, int C) {
  return buf >= 0 && buf < (int)m->buffers.size() && m->buffers[buf].f32 && m->buffers[buf].C == C;
}

// The PAF chain's parameters, checked by sb_bottomup_configure and sb_bottomup_from_maps alike (not the buffer ids),
// with the shared memory max_node_peaks gives its kernels (on the handle's device, which must be current)
static int check_paf_params(sb_handle_s* h, const sb_bottomup_params* p) {
  if (p->n_nodes <= 0 || p->n_edges <= 0 || !p->edges) return sb_fail(h, SB_ERR_INVALID, "bad skeleton");
  if (p->n_sorted > p->n_edges || p->max_peaks_per_sample <= 0 || p->max_node_peaks <= 0 || p->max_instances <= 0)
    return sb_fail(h, SB_ERR_INVALID, "bad capacities");
  for (int e = 0; e < 2 * p->n_edges; ++e)
    if (p->edges[e] < 0 || p->edges[e] >= p->n_nodes) return sb_fail(h, SB_ERR_INVALID, "edge node index out of range");
  return sb_check_paf_smem(h, p->n_nodes, p->n_edges, p->max_node_peaks);
}

// The multi-class chain's parameters, checked by sb_multiclass_configure and sb_multiclass_from_maps alike, with the
// shared memory max_node_peaks and n_classes give k_class_group (on the handle's device, which must be current)
static int check_class_params(sb_handle_s* h, const sb_multiclass_params* p) {
  if (p->n_classes < 1 || p->n_classes > SB_MAX_CLASSES)
    return sb_fail(h, SB_ERR_INVALID, "%d classes (1 to %d)", p->n_classes, SB_MAX_CLASSES);
  if (p->cm_output_stride <= 0 || p->class_maps_output_stride <= 0 || !(p->input_scale > 0.f) || p->max_peaks_per_sample <= 0 ||
      p->max_node_peaks <= 0)
    return sb_fail(h, SB_ERR_INVALID, "bad strides / input scale / capacities");
  return sb_check_class_smem(h, p->max_node_peaks, p->n_classes);
}

// ---- host copies of the results (sb_common.cuh) ----
void sb_split_records(const float* rec, int B, size_t width, std::initializer_list<SbRecField> floats,
                      std::initializer_list<int32_t*> ints) {
  for (int b = 0; b < B; ++b) {
    const float* r = rec + (size_t)b * width;
    for (const SbRecField& f : floats) {
      if (f.dst) memcpy(f.dst + (size_t)b * f.n, r, f.n * sizeof(float));
      r += f.n;
    }
    for (int32_t* d : ints) {
      if (d) d[b] = (int32_t)*r;
      ++r;
    }
  }
}

int sb_graph_download(sb_handle_s* h, const SbPostWs& ws, int B, SbGraphHost& g) {
  const size_t nodes = (size_t)B * ws.C, K = ws.max_node_peaks;
  g.n_peaks.resize(B); g.node_cnt.resize(nodes); g.node_peaks.resize(nodes * K);
  g.score_mat.resize((size_t)B * ws.n_edges * K * K);
  SB_CUDA(h, cudaMemcpy(g.n_peaks.data(), ws.n_peaks, (size_t)B * 4, cudaMemcpyDeviceToHost));
  SB_CUDA(h, cudaMemcpy(g.node_cnt.data(), ws.node_cnt, g.node_cnt.size() * 4, cudaMemcpyDeviceToHost));
  SB_CUDA(h, cudaMemcpy(g.node_peaks.data(), ws.node_peaks, g.node_peaks.size() * 4, cudaMemcpyDeviceToHost));
  SB_CUDA(h, cudaMemcpy(g.score_mat.data(), ws.score_mat, g.score_mat.size() * 4, cudaMemcpyDeviceToHost));
  return 0;
}

int sb_graph_flatten(sb_handle_s* h, const SbPostWs& ws, const SbGraphHost& g, const int* edges_host, int B, int cap,
                     int32_t* edge_inds, int32_t* edge_peak_inds, float* line_scores, int32_t* cand_offsets) {
  const int C = ws.C, K = ws.max_node_peaks, E = ws.n_edges;
  int tc = 0;
  for (int b = 0; b < B; ++b) {
    cand_offsets[b] = tc;
    for (int e = 0; e < E; ++e) {
      const int sn = edges_host[2 * e], dn = edges_host[2 * e + 1];
      const int ns = std::min(g.node_cnt[(size_t)b * C + sn], K), nd = std::min(g.node_cnt[(size_t)b * C + dn], K);
      for (int i = 0; i < ns; ++i)
        for (int j = 0; j < nd; ++j) {
          if (tc >= cap) return sb_fail(h, SB_ERR_INVALID, "candidate capacity %d exceeded", cap);
          edge_inds[tc] = e;
          edge_peak_inds[2 * tc] = g.node_peaks[((size_t)b * C + sn) * K + i];
          edge_peak_inds[2 * tc + 1] = g.node_peaks[((size_t)b * C + dn) * K + j];
          line_scores[tc] = g.score_mat[((size_t)b * E + e) * K * K + (size_t)i * nd + j];
          ++tc;
        }
    }
  }
  cand_offsets[B] = tc;
  return SB_OK;
}

// ---------------------------------- the slots of the streamed steps ----------------------------
int SbSlots::alloc(sb_handle_s* h, size_t frame_bytes, size_t stage_floats) {
  if (!copy_stream) SB_CUDA(h, cudaStreamCreateWithFlags(&copy_stream, cudaStreamNonBlocking));
  for (int i = 0; i < 2; ++i) {
    for (cudaEvent_t* e : {&h2d_done[i], &frames_free[i], &result[i]})
      if (!*e) SB_CUDA(h, cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    if (!frames[i]) SB_CUDA(h, cudaMalloc(&frames[i], frame_bytes));
    if (!stage[i]) SB_CUDA(h, cudaHostAlloc((void**)&stage[i], stage_floats * sizeof(float), cudaHostAllocDefault));
  }
  return 0;
}

int SbSlots::check_submit(sb_handle_s* h, const char* what, int slot, int B, int max_B, const void* frames_host) const {
  if (slot < 0 || slot > 1 || !frames_host || B <= 0 || B > max_B) return sb_fail(h, SB_ERR_INVALID, "%s: bad slot / batch", what);
  if (slot_B[slot]) return sb_fail(h, SB_ERR_INVALID, "%s: slot %d holds a batch that was not collected", what, slot);
  return 0;
}

int SbSlots::upload(sb_handle_s* h, int slot, const void* frames_host, size_t bytes, std::initializer_list<Copy> more) {
  if (slot_seq[slot]) SB_CUDA(h, cudaStreamWaitEvent(copy_stream, frames_free[slot], 0));
  SB_CUDA(h, cudaMemcpyAsync(frames[slot], frames_host, bytes, cudaMemcpyHostToDevice, copy_stream));
  for (const Copy& c : more) SB_CUDA(h, cudaMemcpyAsync(c.dst, c.src, c.bytes, cudaMemcpyHostToDevice, copy_stream));
  SB_CUDA(h, cudaEventRecord(h2d_done[slot], copy_stream));
  return 0;
}

int SbSlots::check_collect(sb_handle_s* h, const char* what, int slot, int B) const {
  if (slot < 0 || slot > 1 || !slot_B[slot]) return sb_fail(h, SB_ERR_INVALID, "%s: slot %d holds no submitted batch", what, slot);
  if (B != slot_B[slot]) return sb_fail(h, SB_ERR_INVALID, "%s: slot %d holds a batch of %d frames, not %d", what, slot, slot_B[slot], B);
  if (slot_B[1 - slot] && slot_seq[1 - slot] < slot_seq[slot])
    return sb_fail(h, SB_ERR_INVALID, "%s: slot %d was submitted first; collect batches in submit order", what, 1 - slot);
  return 0;
}

int SbSlots::collect(sb_handle_s* h, int slot) {
  const int B = slot_B[slot];
  slot_B[slot] = 0;
  SB_CUDA(h, cudaEventSynchronize(result[slot]));
  done_B[slot] = B;
  return 0;
}

int SbSlots::check_read(sb_handle_s* h, const char* what, int slot, int B) const {
  if (slot < 0 || slot > 1 || B <= 0 || done_B[slot] != B)
    return sb_fail(h, SB_ERR_INVALID, "%s: slot %d holds no collected batch of %d frames", what, slot, B);
  return 0;
}

int SbSlots::check_idle(sb_handle_s* h, const char* what) const {
  if (busy()) return sb_fail(h, SB_ERR_INVALID, "%s: a batch was submitted and not collected; collect it first", what);
  return 0;
}

void SbSlots::release() {
  for (int i = 0; i < 2; ++i) {
    if (frames[i]) cudaFree(frames[i]);
    if (stage[i]) cudaFreeHost(stage[i]);
    for (cudaEvent_t e : {h2d_done[i], frames_free[i], result[i]}) if (e) cudaEventDestroy(e);
  }
  if (copy_stream) cudaStreamDestroy(copy_stream);
  *this = SbSlots();
}

extern "C" {

int sb_bottomup_configure(sb_handle_t h, int model_id, const sb_bottomup_params* p) {
  SbModel* m = configure_target(h, model_id, p);
  if (!m) return SB_ERR_INVALID;
  SB_CUDA(h, cudaSetDevice(h->device));
  if (int rc = check_paf_params(h, p)) return rc;
  if (!f32_head(m, p->cms_buffer, p->n_nodes) || !f32_head(m, p->pafs_buffer, 2 * p->n_edges))
    return sb_fail(h, SB_ERR_INVALID, "cms / pafs buffers must be f32 head outputs of n_nodes / 2 * n_edges channels");
  if (p->offsets_buffer >= 0 && !f32_head(m, p->offsets_buffer, 2 * p->n_nodes)) return sb_fail(h, SB_ERR_INVALID, "bad offsets buffer");
  int rc = chain_drop(h, m);
  if (rc) return rc;
  const SbBuffer& cb = m->buffers[p->cms_buffer];
  if ((rc = sb_post_ws_alloc(h, m->ws, m->B, cb.H, cb.W, cb.C, p->max_peaks_per_sample, p->max_node_peaks, p->max_instances, p->n_edges)))
    return rc;
  SB_CUDA(h, cudaMemcpy(m->ws.edges_dev, p->edges, (size_t)p->n_edges * 2 * sizeof(int), cudaMemcpyHostToDevice));
  if (p->n_sorted > 0)
    SB_CUDA(h, cudaMemcpy(m->ws.sorted_edges_dev, p->sorted_edge_inds, (size_t)p->n_sorted * sizeof(int), cudaMemcpyHostToDevice));
  m->ws.n_sorted = p->n_sorted;
  m->bu = *p;
  m->bu.edges = nullptr; m->bu.sorted_edge_inds = nullptr;
  m->bu_edges.assign(p->edges, p->edges + 2 * p->n_edges);
  m->guard_op = post_guard_op(m, p->cms_buffer, p->pafs_buffer, p->offsets_buffer);
  m->chain = SB_CHAIN_PAF;
  return SB_OK;
}

int sb_multiclass_configure(sb_handle_t h, int model_id, const sb_multiclass_params* p) {
  SbModel* m = configure_target(h, model_id, p);
  if (!m) return SB_ERR_INVALID;
  SB_CUDA(h, cudaSetDevice(h->device));
  if (int rc = check_class_params(h, p)) return rc;
  if (!f32_head(m, p->cms_buffer, p->n_nodes) || !f32_head(m, p->class_maps_buffer, p->n_classes))
    return sb_fail(h, SB_ERR_INVALID, "cms / class-map buffers must be f32 head outputs of n_nodes / n_classes channels");
  if (p->offsets_buffer >= 0 && !f32_head(m, p->offsets_buffer, 2 * p->n_nodes)) return sb_fail(h, SB_ERR_INVALID, "bad offsets buffer");
  int rc = chain_drop(h, m);
  if (rc) return rc;
  const SbBuffer& cb = m->buffers[p->cms_buffer];
  if ((rc = sb_post_ws_alloc(h, m->ws, m->B, cb.H, cb.W, cb.C, p->max_peaks_per_sample, p->max_node_peaks, 1, 0))) return rc;
  m->ws.node_lists = true;
  const size_t nrec = (size_t)m->B * sb_class_record_width(p->n_classes, p->n_nodes);
  if ((rc = sb_dev_alloc(h, &m->ws.records, nrec))) return rc;
  m->ws.bytes += nrec * sizeof(float);
  m->mc = *p;
  m->guard_op = post_guard_op(m, p->cms_buffer, p->class_maps_buffer, p->offsets_buffer);
  m->chain = SB_CHAIN_CLASS;
  return SB_OK;
}

static size_t stage_floats(const SbModel* m) {          // [world][B][width] when the exchange is connected
  return (size_t)(m->gather.connected ? m->gather.world : 1) * m->B * record_width(m);
}

// One D2H copy of a batch's results into pinned `dst`: the rank's own records, or -- exchange connected -- the whole gather
// window of the step just pushed (device-side wait for the peers, copy, acknowledge; all on stream rs).
static int queue_result_copy(sb_handle_s* h, SbModel* m, int B, cudaStream_t rs, float* dst, int counts_slot) {
  if (m->gather.connected)
    return sb_gather_queue_collect(h, m, m->gather.step - 1, B, dst, m->gather.counts_dev + counts_slot * SB_GATHER_MAX_WORLD, rs);
  // the global chain's values sit at the configured batch's offset of its block, so the whole block comes over (B <= m->B)
  const bool global = m->chain == SB_CHAIN_GLOBAL;
  SB_CUDA(h, cudaMemcpyAsync(dst, global ? m->gs.points : m->ws.records, (global ? m->B : B) * record_width(m) * sizeof(float),
                             cudaMemcpyDeviceToHost, rs));
  return 0;
}
static const float* own_slice(const SbModel* m, const float* staged, int B) {
  return staged + (m->gather.connected ? (size_t)m->gather.rank * B * record_width(m) : 0);
}
static int check_exchange(sb_handle_s* h, SbModel* m) {
  if (m->gather.connected && *m->gather.status_host != 0) {
    const int st = *m->gather.status_host;
    *m->gather.status_host = 0;
    return sb_fail(h, SB_ERR_CUDA, "record exchange timed out (%s): a peer rank stopped pushing or consuming",
                   st == SB_GATHER_TIMEOUT_ARRIVE ? "waiting for arrivals" : "waiting for acknowledgements");
  }
  return 0;
}

// A PAF-chain record: peaks | peak values | instance scores | n_valid | flags
static void split_paf_records(const SbModel* m, const float* rec, int B, float* out_instance_peaks, float* out_instance_peak_vals,
                              float* out_instance_scores, int32_t* out_n_valid, int32_t* out_flags) {
  const size_t I = m->bu.max_instances, C = m->bu.n_nodes;
  sb_split_records(rec, B, record_width(m), {{out_instance_peaks, I * C * 2}, {out_instance_peak_vals, I * C}, {out_instance_scores, I}},
                   {out_n_valid, out_flags});
}

// The PAF chain: local peaks, PAF scoring and matching, grouping into ws's instance arrays and records (and, gx given,
// every peer's gather window).
static int bottomup_post_kernels(sb_handle_s* h, const sb_bottomup_params& p, SbPostWs& ws, const SbMap& cms, const SbMap& pafs,
                                 const float* off, int B, const SbGatherDev* gx = nullptr) {
  SbPeakParams pp{p.peak_threshold, p.refinement, p.integral_patch_size, (float)p.cm_output_stride, 1.0f};
  int rc = sbk_local_peaks(h, cms.dev, off, B, cms.H, cms.W, cms.C, pp, ws);
  if (rc) return rc;
  const float max_len = p.max_edge_length_ratio * (float)std::max(std::max(pafs.H, pafs.W), pafs.C) * (float)p.paf_output_stride;
  if ((rc = sbk_score_match(h, pafs.dev, B, pafs.H, pafs.W, pafs.C, p.n_line_points, p.paf_output_stride, max_len,
                            p.dist_penalty_weight, ws))) return rc;
  return sbk_group(h, B, p.n_nodes, p.min_instance_peaks, p.min_line_scores, p.input_scale, ws, gx);
}

// The multi-class chain: local peaks with their per-node lists, then the identity grouping into the records.
static int multiclass_post_kernels(sb_handle_s* h, const sb_multiclass_params& p, SbPostWs& ws, const SbMap& cms,
                                   const SbMap& cls, const float* off, int B) {
  SbPeakParams pp{p.peak_threshold, p.refinement, p.integral_patch_size, (float)p.cm_output_stride, 1.0f};
  int rc = sbk_local_peaks(h, cms.dev, off, B, cms.H, cms.W, cms.C, pp, ws);
  if (rc) return rc;
  return sbk_class_group(h, cls.dev, B, cls.H, cls.W, cls.C, (float)p.class_maps_output_stride, p.input_scale, ws);
}

// The step's chain on the head buffers: the global peaks (plus the device crop offsets crop_off, when given), the
// multi-class one, or the PAF one with the record exchange pushed from k_group's epilogue when connected, else the
// attached tracker after it.
static int step_post_kernels(sb_handle_s* h, SbModel* m, int B, const float* crop_off) {
  if (m->chain == SB_CHAIN_GLOBAL) {
    const sb_global_params& p = m->gl;
    const SbBuffer& cb = m->buffers[p.cms_buffer];
    const SbGlobalScratch& g = m->gs;
    SbPeakParams pp{p.peak_threshold, p.refinement, p.integral_patch_size, (float)p.output_stride, p.input_scale};
    return sbk_global_peaks(h, (const float*)cb.dev, head_offsets(m, p.offsets_buffer), B, cb.H, cb.W, cb.C, pp, crop_off, g.part,
                            g.chunks, g.rpc, g.points, g.vals);
  }
  if (m->chain == SB_CHAIN_CLASS) {
    const sb_multiclass_params& p = m->mc;
    return multiclass_post_kernels(h, p, m->ws, head_map(m, p.cms_buffer), head_map(m, p.class_maps_buffer),
                                   head_offsets(m, p.offsets_buffer), B);
  }
  const sb_bottomup_params& p = m->bu;
  const SbMap cms = head_map(m, p.cms_buffer), pafs = head_map(m, p.pafs_buffer);
  const float* off = head_offsets(m, p.offsets_buffer);
  if (m->gather.connected) {
    const SbGatherDev gx = sb_gather_dev(m, (unsigned long long)m->gather.step);
    const int rc = bottomup_post_kernels(h, p, m->ws, cms, pafs, off, B, &gx);
    if (!rc) m->gather.step++;
    return rc;
  }
  if (const int rc = bottomup_post_kernels(h, p, m->ws, cms, pafs, off, B)) return rc;
  if (!m->trk) return 0;
  if (B > m->trk_B) return sb_fail(h, SB_ERR_INVALID, "attached tracker was sized for %d frames per step, not %d", m->trk_B, B);
  return sbk_track_step(h, m->trk, B, m->ws.inst_peaks, m->ws.inst_vals, m->ws.inst_scores, m->ws.n_inst, p.max_instances,
                        m->trk_cut, m->trk_h, m->trk_w, m->trk_dev);
}

// A multi-class record: points | values | class probabilities | flags
static void split_class_records(const sb_multiclass_params& p, const float* rec, int B, float* out_points, float* out_vals,
                                float* out_class_probs, int32_t* out_flags) {
  const size_t n1 = (size_t)p.n_classes * p.n_nodes;
  sb_split_records(rec, B, sb_class_record_width(p.n_classes, p.n_nodes), {{out_points, n1 * 2}, {out_vals, n1}, {out_class_probs, n1}},
                   {out_flags});
}

// The track records of a batch go to the host with its result records, on the same stream.
static int queue_track_copy(sb_handle_s* h, SbModel* m, int B, cudaStream_t rs, int which) {
  if (!m->trk) return 0;
  SB_CUDA(h, cudaMemcpyAsync(m->trk_host[which], m->trk_dev, (size_t)B * sb_track_record_width(m->trk_I) * sizeof(double),
                             cudaMemcpyDeviceToHost, rs));
  return 0;
}

// The configured chain's post-processing of this batch (peak finding, then PAF scoring / matching /
// grouping or the identity grouping) on the handle's post-processing
// stream: it only depends on the head outputs, so it overlaps the network of the next batch
// (run_ops waits on post_done_ev right before it overwrites a head buffer).  Without the overlap
// (SB_DISABLE_POST_OVERLAP: no guard op) it still runs there, so that work a caller queues on the
// post-processing stream stays behind it, and the handle's stream waits for it at once.
static int bottomup_post(sb_handle_s* h, SbModel* m, int B, const float* crop_off = nullptr) {
  cudaStream_t main_stream = h->stream;
  SB_CUDA(h, cudaEventRecord(h->fwd_done_ev, main_stream));
  SB_CUDA(h, cudaStreamWaitEvent(h->post_stream, h->fwd_done_ev, 0));
  h->stream = h->post_stream;
  int rc = step_post_kernels(h, m, B, crop_off);
  cudaError_t e = cudaEventRecord(h->post_done_ev, h->post_stream);
  h->stream = main_stream;
  if (rc) return rc;
  if (e != cudaSuccess) return sb_fail(h, SB_ERR_CUDA, "event record: %s", cudaGetErrorString(e));
  if (m->guard_op < 0) SB_CUDA(h, cudaStreamWaitEvent(main_stream, h->post_done_ev, 0));
  else h->post_pending = true;
  return 0;
}

static const char* const kNoPaf = "bottom-up predictor not configured";
static const char* const kNoClass = "multi-class predictor not configured";

int sb_infer_bottomup_dev(sb_handle_t h, int model_id, const uint8_t* frames_dev, int B) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_PAF, kNoPaf);
  if (!m) return SB_ERR_INVALID;
  SB_CUDA(h, cudaSetDevice(h->device));
  int rc = sb_run_ops(h, m, frames_dev, 1, B);
  if (rc) return rc;
  return bottomup_post(h, m, B);
}

// The streamed steps of the chain: submit batch i + 1 (its upload runs on the slots' copy stream) while batch i computes,
// then collect batch i; ONE D2H copy per batch brings the per-frame records into the slot's staging.  A synchronous call
// is one step into slot 0 and its collect.

static int slots_alloc(sb_handle_s* h, SbModel* m) {
  return m->slots.alloc(h, (size_t)m->B * m->Hin * m->Win * m->Cin, stage_floats(m));
}

// Queues the step of B frames at frames_dev into `slot`: network, post-processing (crop_off: the global chain's device
// crop offsets, or nullptr), the result and track copies into the slot's staging, its events.  The batch is then submitted.
static int queue_step(sb_handle_s* h, SbModel* m, const void* frames_dev, int frames_are_u8, int B, int slot, const float* crop_off) {
  SbSlots& sl = m->slots;
  int rc = sb_run_ops(h, m, frames_dev, frames_are_u8, B);
  if (rc) return rc;
  SB_CUDA(h, cudaEventRecord(sl.frames_free[slot], h->stream));
  if ((rc = bottomup_post(h, m, B, crop_off))) return rc;
  cudaStream_t rs = h->post_pending ? h->post_stream : h->stream;
  if ((rc = queue_result_copy(h, m, B, rs, sl.stage[slot], 1 + slot))) return rc;
  if ((rc = queue_track_copy(h, m, B, rs, slot))) return rc;
  SB_CUDA(h, cudaEventRecord(sl.result[slot], rs));
  sl.submitted(slot, B);
  return SB_OK;
}

static int step_submit(sb_handle_s* h, SbModel* m, const uint8_t* frames_host, int B, int slot, const char* what) {
  SbSlots& sl = m->slots;
  int rc = sl.check_submit(h, what, slot, B, m->B, frames_host);
  if (rc) return rc;
  SB_CUDA(h, cudaSetDevice(h->device));
  if ((rc = slots_alloc(h, m)) || (rc = sl.upload(h, slot, frames_host, (size_t)B * m->Hin * m->Win * m->Cin))) return rc;
  SB_CUDA(h, cudaStreamWaitEvent(h->stream, sl.h2d_done[slot], 0));
  return queue_step(h, m, sl.frames[slot], 1, B, slot, nullptr);
}

// Blocks until the records of the batch submitted into `slot` are in its pinned staging.
static int step_collect(sb_handle_s* h, SbModel* m, int slot, int B, const char* what) {
  int rc = m->slots.check_collect(h, what, slot, B);
  if (rc || (rc = m->slots.collect(h, slot))) return rc;
  return check_exchange(h, m);
}

// A synchronous call: the uint8 or float32 frames (and the global chain's crop offsets, when given) uploaded on the
// handle's stream into frames_dev, the step queued into slot 0, then slot 0 collected.
static int step_call(sb_handle_s* h, SbModel* m, const void* frames_host, int frames_are_u8, int B, const float* crop_off_host,
                     const char* what) {
  if (B <= 0 || B > m->B) return sb_fail(h, SB_ERR_INVALID, "%s: bad batch", what);
  int rc = m->slots.check_idle(h, what);
  if (rc) return rc;
  SB_CUDA(h, cudaSetDevice(h->device));
  if ((rc = slots_alloc(h, m)) || (rc = upload_frames(h, m, frames_host, frames_are_u8, B))) return rc;
  if (crop_off_host)
    SB_CUDA(h, cudaMemcpyAsync(m->gs.crop_off, crop_off_host, (size_t)B * 2 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
  if ((rc = queue_step(h, m, m->frames_dev, frames_are_u8, B, 0, crop_off_host ? m->gs.crop_off : nullptr))) return rc;
  return step_collect(h, m, 0, B, what);
}

int sb_infer_bottomup(sb_handle_t h, int model_id, const uint8_t* frames_host, int B, float* out_instance_peaks,
                      float* out_instance_peak_vals, float* out_instance_scores, int32_t* out_n_valid,
                      int32_t* out_flags) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_PAF, kNoPaf);
  if (!m) return SB_ERR_INVALID;
  if (const int rc = step_call(h, m, frames_host, 1, B, nullptr, "sb_infer_bottomup")) return rc;
  split_paf_records(m, own_slice(m, m->slots.stage[0], B), B, out_instance_peaks, out_instance_peak_vals, out_instance_scores,
                    out_n_valid, out_flags);
  return SB_OK;
}

int sb_infer_multiclass(sb_handle_t h, int model_id, const void* frames_host, int frames_are_u8, int B, float* out_points,
                        float* out_vals, float* out_class_probs, int32_t* out_flags) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_CLASS, kNoClass);
  if (!m) return SB_ERR_INVALID;
  if (!frames_host || !out_points || !out_vals || !out_class_probs) return sb_fail(h, SB_ERR_INVALID, "sb_infer_multiclass: null argument");
  if (const int rc = step_call(h, m, frames_host, frames_are_u8 ? 1 : 0, B, nullptr, "sb_infer_multiclass")) return rc;
  split_class_records(m->mc, m->slots.stage[0], B, out_points, out_vals, out_class_probs, out_flags);
  return SB_OK;
}

// The stream post-processing runs on (consumers such as the NCCL gather can be queued behind it).
int sb_get_post_stream(sb_handle_t h, void** out_stream) {
  if (!h || !out_stream) return sb_fail(h, SB_ERR_INVALID, "null argument");
  *out_stream = (void*)h->post_stream;
  return SB_OK;
}

int sb_bottomup_submit(sb_handle_t h, int model_id, const uint8_t* frames_host, int B, int slot) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_PAF, kNoPaf);
  return m ? step_submit(h, m, frames_host, B, slot, "sb_bottomup_submit") : SB_ERR_INVALID;
}

int sb_bottomup_collect(sb_handle_t h, int model_id, int slot, int B, float* out_instance_peaks,
                        float* out_instance_peak_vals, float* out_instance_scores, int32_t* out_n_valid,
                        int32_t* out_flags) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_PAF, kNoPaf);
  if (!m) return SB_ERR_INVALID;
  if (const int rc = step_collect(h, m, slot, B, "sb_bottomup_collect")) return rc;
  split_paf_records(m, own_slice(m, m->slots.stage[slot], B), B, out_instance_peaks, out_instance_peak_vals, out_instance_scores,
                    out_n_valid, out_flags);
  return SB_OK;
}

int sb_multiclass_submit(sb_handle_t h, int model_id, const uint8_t* frames_host, int B, int slot) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_CLASS, kNoClass);
  return m ? step_submit(h, m, frames_host, B, slot, "sb_multiclass_submit") : SB_ERR_INVALID;
}

int sb_multiclass_collect(sb_handle_t h, int model_id, int slot, int B, float* out_points, float* out_vals,
                          float* out_class_probs, int32_t* out_flags) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_CLASS, kNoClass);
  if (!m) return SB_ERR_INVALID;
  if (const int rc = step_collect(h, m, slot, B, "sb_multiclass_collect")) return rc;
  split_class_records(m->mc, m->slots.stage[slot], B, out_points, out_vals, out_class_probs, out_flags);
  return SB_OK;
}

int sb_bottomup_gathered(sb_handle_t h, int model_id, int slot, int B, float* out_records, int32_t* out_counts) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_PAF, "sb_bottomup_gathered: exchange not connected");
  if (!m || !m->gather.connected) return sb_fail(h, SB_ERR_INVALID, "sb_bottomup_gathered: exchange not connected");
  if (!out_records) return sb_fail(h, SB_ERR_INVALID, "sb_bottomup_gathered: bad slot");
  if (const int rc = m->slots.check_read(h, "sb_bottomup_gathered", slot, B)) return rc;
  memcpy(out_records, m->slots.stage[slot], (size_t)m->gather.world * B * sb_record_width(m->bu.max_instances, m->bu.n_nodes) * sizeof(float));
  if (out_counts)
    for (int r = 0; r < m->gather.world; ++r) out_counts[r] = m->gather.counts_host[(1 + slot) * SB_GATHER_MAX_WORLD + r];
  return SB_OK;
}

int sb_bottomup_attach_tracker(sb_handle_t h, int model_id, int tracker_id, int max_instances, double img_h, double img_w) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_PAF, kNoPaf);
  if (!m) return SB_ERR_INVALID;
  SB_CUDA(h, cudaSetDevice(h->device));
  if (h->post_pending) SB_CUDA(h, cudaStreamSynchronize(h->post_stream));
  if (tracker_id < 0) { m->trk = nullptr; return SB_OK; }
  SbTracker* t = sb_tracker_get(h, tracker_id);
  if (!t) return sb_fail(h, SB_ERR_INVALID, "sb_bottomup_attach_tracker: no tracker %d on this handle", tracker_id);
  if (m->gather.connected)
    return sb_fail(h, SB_ERR_UNSUPPORTED, "sb_bottomup_attach_tracker: the record exchange is connected (one rank only)");
  if (sb_tracker_nodes(t) != m->bu.n_nodes || sb_tracker_max_instances(t) < m->bu.max_instances)
    return sb_fail(h, SB_ERR_INVALID, "sb_bottomup_attach_tracker: tracker of %d nodes / %d instances, predictor of %d / %d",
                   sb_tracker_nodes(t), sb_tracker_max_instances(t), m->bu.n_nodes, m->bu.max_instances);
  if (!(img_h > 0) || !(img_w > 0)) return sb_fail(h, SB_ERR_INVALID, "sb_bottomup_attach_tracker: image %g x %g", img_h, img_w);
  if (const int rc = sb_track_records_alloc(h, m, m->B, sb_tracker_max_instances(t))) return rc;
  m->trk = t; m->trk_cut = max_instances < 0 ? -1 : max_instances; m->trk_h = img_h; m->trk_w = img_w;
  return SB_OK;
}

int sb_bottomup_tracks(sb_handle_t h, int model_id, int slot, int B, double* out_tracks) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_PAF, "sb_bottomup_tracks: no tracker attached");
  if (!m || !m->trk) return sb_fail(h, SB_ERR_INVALID, "sb_bottomup_tracks: no tracker attached");
  if (slot < 0 || slot > 1 || B <= 0 || B > m->trk_B || !out_tracks) return sb_fail(h, SB_ERR_INVALID, "sb_bottomup_tracks: bad slot / batch");
  if (const int rc = m->slots.check_read(h, "sb_bottomup_tracks", slot, B)) return rc;
  memcpy(out_tracks, m->trk_host[slot], (size_t)B * sb_track_record_width(m->trk_I) * sizeof(double));
  return SB_OK;
}

int sb_bottomup_device_tracks(sb_handle_t h, int model_id, int B, double* out_tracks) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_PAF, "sb_bottomup_device_tracks: no tracker attached");
  if (!m || !m->trk) return sb_fail(h, SB_ERR_INVALID, "sb_bottomup_device_tracks: no tracker attached");
  if (B <= 0 || B > m->trk_B || !out_tracks) return sb_fail(h, SB_ERR_INVALID, "sb_bottomup_device_tracks: bad batch");
  SB_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t rs = h->post_pending ? h->post_stream : h->stream;
  SB_CUDA(h, cudaMemcpyAsync(out_tracks, m->trk_dev, (size_t)B * sb_track_record_width(m->trk_I) * sizeof(double),
                             cudaMemcpyDeviceToHost, rs));
  SB_CUDA(h, cudaStreamSynchronize(rs));
  return SB_OK;
}

int sb_bottomup_device_records(sb_handle_t h, int model_id, float** records_dev) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_PAF, kNoPaf);
  if (!m || !records_dev) return sb_fail(h, SB_ERR_INVALID, kNoPaf);
  *records_dev = m->ws.records;
  return SB_OK;
}

// The peaks and PAF candidates of the step that wrote ws, flattened per frame into the caller's arrays
static int fetch_graph_ws(sb_handle_s* h, const SbPostWs& ws, const int* edges_host, int B, int cap_peaks, float* peaks,
                          float* peak_vals, int32_t* peak_channel_inds, int32_t* peak_offsets, int cap_cands,
                          int32_t* edge_inds, int32_t* edge_peak_inds, float* line_scores, int32_t* cand_offsets) {
  SbGraphHost g;
  SB_CUDA(h, cudaStreamSynchronize(h->stream));
  SB_CUDA(h, cudaStreamSynchronize(h->post_stream));
  if (const int rc = sb_graph_download(h, ws, B, g)) return rc;
  const int MP = ws.max_peaks;
  int tp = 0;
  for (int b = 0; b < B; ++b) {
    const int n = g.n_peaks[b];
    peak_offsets[b] = tp;
    if (tp + n > cap_peaks) return sb_fail(h, SB_ERR_INVALID, "peak capacity exceeded");
    if (n > 0) {
      SB_CUDA(h, cudaMemcpy(peaks + 2 * (size_t)tp, ws.peaks + (size_t)b * MP * 2, (size_t)n * 8, cudaMemcpyDeviceToHost));
      SB_CUDA(h, cudaMemcpy(peak_vals + tp, ws.peak_vals + (size_t)b * MP, (size_t)n * 4, cudaMemcpyDeviceToHost));
      SB_CUDA(h, cudaMemcpy(peak_channel_inds + tp, ws.peak_ch + (size_t)b * MP, (size_t)n * 4, cudaMemcpyDeviceToHost));
    }
    tp += n;
  }
  peak_offsets[B] = tp;
  return sb_graph_flatten(h, ws, g, edges_host, B, cap_cands, edge_inds, edge_peak_inds, line_scores, cand_offsets);
}

int sb_bottomup_fetch_graph(sb_handle_t h, int model_id, int B, int cap_peaks, float* peaks, float* peak_vals,
                            int32_t* peak_channel_inds, int32_t* peak_offsets, int cap_cands, int32_t* edge_inds,
                            int32_t* edge_peak_inds, float* line_scores, int32_t* cand_offsets) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_PAF, kNoPaf);
  if (!m) return SB_ERR_INVALID;
  SB_CUDA(h, cudaSetDevice(h->device));
  return fetch_graph_ws(h, m->ws, m->bu_edges.data(), B, cap_peaks, peaks, peak_vals, peak_channel_inds, peak_offsets,
                        cap_cands, edge_inds, edge_peak_inds, line_scores, cand_offsets);
}

int sb_bottomup_from_maps(sb_handle_t h, const sb_bottomup_params* p, const float* cms_host, int B, int H, int W,
                          const float* pafs_host, int Hp, int Wp, const float* offsets_host,
                          float* out_instance_peaks, float* out_instance_peak_vals, float* out_instance_scores,
                          int32_t* out_n_valid, int32_t* out_flags, int cap_peaks, float* peaks, float* peak_vals,
                          int32_t* peak_channel_inds, int32_t* peak_offsets, int cap_cands, int32_t* edge_inds,
                          int32_t* edge_peak_inds, float* line_scores, int32_t* cand_offsets) {
  if (!h || !p) return sb_fail(h, SB_ERR_INVALID, "null handle / params");
  if (!cms_host || !pafs_host || !out_instance_peaks || !out_instance_peak_vals || !out_instance_scores || !out_n_valid)
    return sb_fail(h, SB_ERR_INVALID, "sb_bottomup_from_maps: null argument");
  if (B <= 0 || H <= 0 || W <= 0 || Hp <= 0 || Wp <= 0) return sb_fail(h, SB_ERR_INVALID, "sb_bottomup_from_maps: bad shape");
  SB_CUDA(h, cudaSetDevice(h->device));
  int rc = check_paf_params(h, p);
  if (rc) return rc;
  const int C = p->n_nodes, C2 = 2 * p->n_edges;
  SbScratch s(h);
  if ((rc = sb_post_ws_alloc(h, s.ws, B, H, W, C, p->max_peaks_per_sample, p->max_node_peaks, p->max_instances, p->n_edges))) return rc;
  SbMap cms{nullptr, H, W, C}, pafs{nullptr, Hp, Wp, C2};
  const float* off = nullptr;
  const size_t ncm = (size_t)B * H * W * C;
  if ((rc = s.upload(cms_host, ncm, &cms.dev)) || (rc = s.upload(pafs_host, (size_t)B * Hp * Wp * C2, &pafs.dev)) ||
      (rc = s.upload(offsets_host, 2 * ncm, &off, true)) || (rc = s.to_dev(s.ws.edges_dev, p->edges, (size_t)p->n_edges * 2)))
    return rc;
  if (p->n_sorted > 0 && (rc = s.to_dev(s.ws.sorted_edges_dev, p->sorted_edge_inds, (size_t)p->n_sorted))) return rc;
  s.ws.n_sorted = p->n_sorted;
  if ((rc = bottomup_post_kernels(h, *p, s.ws, cms, pafs, off, B))) return rc;
  const SbPostWs& ws = s.ws;
  const size_t I = p->max_instances;
  if ((rc = s.to_host(out_instance_peaks, ws.inst_peaks, B * I * C * 2)) || (rc = s.to_host(out_instance_peak_vals, ws.inst_vals, B * I * C)) ||
      (rc = s.to_host(out_instance_scores, ws.inst_scores, B * I)) || (rc = s.to_host(out_n_valid, ws.n_inst, (size_t)B)) ||
      (rc = s.to_host(out_flags, ws.flags, (size_t)B, true)) || (rc = s.sync()))
    return rc;
  if (peaks)
    return fetch_graph_ws(h, ws, p->edges, B, cap_peaks, peaks, peak_vals, peak_channel_inds, peak_offsets, cap_cands,
                          edge_inds, edge_peak_inds, line_scores, cand_offsets);
  return SB_OK;
}

int sb_multiclass_from_maps(sb_handle_t h, const sb_multiclass_params* p, const float* cms_host, int B, int H, int W,
                            const float* class_logits_host, int Hc, int Wc, const float* offsets_host, float* out_points,
                            float* out_vals, float* out_class_probs, int32_t* out_flags) {
  if (!h || !p) return sb_fail(h, SB_ERR_INVALID, "null handle / params");
  if (!cms_host || !class_logits_host || !out_points || !out_vals || !out_class_probs)
    return sb_fail(h, SB_ERR_INVALID, "sb_multiclass_from_maps: null argument");
  if (B <= 0 || H <= 0 || W <= 0 || Hc <= 0 || Wc <= 0 || p->n_nodes <= 0) return sb_fail(h, SB_ERR_INVALID, "sb_multiclass_from_maps: bad shape");
  SB_CUDA(h, cudaSetDevice(h->device));
  int rc = check_class_params(h, p);
  if (rc) return rc;
  const int C = p->n_nodes, NC = p->n_classes;
  SbScratch s(h);
  if ((rc = sb_post_ws_alloc(h, s.ws, B, H, W, C, p->max_peaks_per_sample, p->max_node_peaks, 1, 0))) return rc;
  s.ws.node_lists = true;
  std::vector<float> rec((size_t)B * sb_class_record_width(NC, C));
  if ((rc = sb_dev_alloc(h, &s.ws.records, rec.size()))) return rc;
  SbMap cms{nullptr, H, W, C}, cls{nullptr, Hc, Wc, NC};
  const float* off = nullptr;
  const size_t ncm = (size_t)B * H * W * C;
  if ((rc = s.upload(cms_host, ncm, &cms.dev)) || (rc = s.upload(class_logits_host, (size_t)B * Hc * Wc * NC, &cls.dev)) ||
      (rc = s.upload(offsets_host, 2 * ncm, &off, true)) || (rc = multiclass_post_kernels(h, *p, s.ws, cms, cls, off, B)) ||
      (rc = s.to_host(rec.data(), s.ws.records, rec.size())) || (rc = s.sync()))
    return rc;
  split_class_records(*p, rec.data(), B, out_points, out_vals, out_class_probs, out_flags);
  return SB_OK;
}

// ---------------------------------- global peaks (single / centered instance) ----------------
static const char* const kNoGlobal = "global-peak predictor not configured";

// The points and values of the first B frames of the global chain's block staged in `slot`
static void split_global(const SbModel* m, int slot, int B, float* out_points, float* out_vals) {
  const size_t C = m->buffers[m->gl.cms_buffer].C;
  memcpy(out_points, m->slots.stage[slot], (size_t)B * C * 2 * sizeof(float));
  memcpy(out_vals, m->slots.stage[slot] + (size_t)m->B * C * 2, (size_t)B * C * sizeof(float));
}

int sb_global_configure(sb_handle_t h, int model_id, const sb_global_params* p) {
  SbModel* m = configure_target(h, model_id, p);
  if (!m) return SB_ERR_INVALID;
  SB_CUDA(h, cudaSetDevice(h->device));
  const int nb = (int)m->buffers.size();
  if (p->cms_buffer < 0 || p->cms_buffer >= nb || !m->buffers[p->cms_buffer].f32) return sb_fail(h, SB_ERR_INVALID, "bad cms buffer");
  if (p->offsets_buffer >= nb) return sb_fail(h, SB_ERR_INVALID, "bad offsets buffer");
  const SbBuffer& cb = m->buffers[p->cms_buffer];
  if (cb.C > 256) return sb_fail(h, SB_ERR_UNSUPPORTED, "more than 256 confidence-map channels");
  int rc = chain_drop(h, m);
  if (rc || (rc = sb_global_scratch_alloc(h, m->gs, m->B, cb.H, cb.C))) return rc;
  m->gl = *p;
  m->guard_op = post_guard_op(m, p->cms_buffer, p->cms_buffer, p->offsets_buffer);
  m->chain = SB_CHAIN_GLOBAL;
  return SB_OK;
}

int sb_infer_global(sb_handle_t h, int model_id, const void* images_host, int images_are_u8, int B,
                    const float* crop_offsets_host, float* out_points, float* out_vals) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_GLOBAL, kNoGlobal);
  if (!m) return SB_ERR_INVALID;
  if (const int rc = step_call(h, m, images_host, images_are_u8 ? 1 : 0, B, crop_offsets_host, "sb_infer_global")) return rc;
  split_global(m, 0, B, out_points, out_vals);
  return SB_OK;
}

// The double-buffered form of sb_infer_global (uint8 frames, no crop offsets): the points | values block comes back in
// one copy.
int sb_global_submit(sb_handle_t h, int model_id, const uint8_t* frames_host, int B, int slot) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_GLOBAL, kNoGlobal);
  return m ? step_submit(h, m, frames_host, B, slot, "sb_global_submit") : SB_ERR_INVALID;
}

int sb_global_collect(sb_handle_t h, int model_id, int slot, int B, float* out_points, float* out_vals) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_GLOBAL, kNoGlobal);
  if (!m) return SB_ERR_INVALID;
  if (!out_points || !out_vals) return sb_fail(h, SB_ERR_INVALID, "sb_global_collect: null argument");
  if (const int rc = step_collect(h, m, slot, B, "sb_global_collect")) return rc;
  split_global(m, slot, B, out_points, out_vals);
  return SB_OK;
}

// ---------------------------------- centroids (top-down stage 1) ------------------------------
int sb_centroid_configure(sb_handle_t h, int model_id, const sb_centroid_params* p) {
  SbModel* m = configure_target(h, model_id, p);
  if (!m) return SB_ERR_INVALID;
  SB_CUDA(h, cudaSetDevice(h->device));
  const int nb = (int)m->buffers.size();
  if (p->cms_buffer < 0 || p->cms_buffer >= nb || !m->buffers[p->cms_buffer].f32) return sb_fail(h, SB_ERR_INVALID, "bad cms buffer");
  if (p->offsets_buffer >= nb) return sb_fail(h, SB_ERR_INVALID, "bad offsets buffer");
  int rc = chain_drop(h, m);
  if (rc) return rc;
  const SbBuffer& cb = m->buffers[p->cms_buffer];
  if ((rc = sb_post_ws_alloc(h, m->ws, m->B, cb.H, cb.W, cb.C, p->max_peaks_per_sample, 1, 1, 0))) return rc;
  m->ce = *p;
  m->chain = SB_CHAIN_CENTROID;
  return SB_OK;
}

int sb_infer_centroids(sb_handle_t h, int model_id, const void* images_host, int images_are_u8, int B,
                       float* out_centroids, float* out_vals, int32_t* out_sample_inds, int32_t* out_n,
                       int32_t* out_flags) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_CENTROID, "centroid predictor not configured");
  if (!m) return SB_ERR_INVALID;
  SB_CUDA(h, cudaSetDevice(h->device));
  if (B <= 0 || B > m->B) return sb_fail(h, SB_ERR_INVALID, "bad batch");
  if (sb_topdown_busy(m))      // the pending instance stage reads this workspace's flags
    return sb_fail(h, SB_ERR_INVALID, "sb_infer_centroids: a top-down batch was submitted and not collected; collect it first");
  int rc = upload_frames(h, m, images_host, images_are_u8, B);
  if (rc) return rc;
  if ((rc = sb_run_ops(h, m, m->frames_dev, images_are_u8, B))) return rc;
  const sb_centroid_params& p = m->ce;
  SbBuffer& cb = m->buffers[p.cms_buffer];
  SbPeakParams pp{p.peak_threshold, p.refinement, p.integral_patch_size, (float)p.output_stride, p.input_scale};
  if ((rc = sbk_local_peaks(h, (const float*)cb.dev, head_offsets(m, p.offsets_buffer), B, cb.H, cb.W, cb.C, pp, m->ws))) return rc;
  return sb_peaks_to_host(h, m->ws, B, out_centroids, out_vals, nullptr, out_sample_inds, out_n, out_flags);
}

}  // extern "C"
