// Multi-GPU exchange of the per-frame result records over NVLink peer memory (SURVEY 8e).
//
// The reference is single-GPU (sleap/nn/system.py:29-46); frames are independent, so ranks own contiguous frame
// shards and the ONE exchange step of the path is an all-gather of fixed-size instance records
// (sleap/nn/inference.py:3230-3343 consumes them to build LabeledFrames).  Instead of a collective call after the
// grouping kernel, the grouping kernel's epilogue (k_group, sb_post.cu) stores each frame's record straight into the
// gather window of EVERY peer through CUDA-IPC mapped pointers (NVSwitch: every peer at full bandwidth), then the last
// CTA publishes a per-(generation, source rank) arrival word with system-scope release.  No rank ever waits for another
// inside its step: the windows are G generations deep and a consumer (device kernel or host collect) acknowledges a
// generation back to every producer, which only blocks a producer that has run G steps ahead of the slowest consumer.
//
// Window of one rank (one cudaMalloc, exported with cudaIpcGetMemHandle):
//   float  data  [G][world][Bmax][width]      records written by rank r into slot [gen][r]
//   u64    arrive[G][world]                   ((step + 1) << 8) | B   written by rank r after its records
//   u64    ack   [world]                      steps consumed by rank r (written by r into every peer's window)
//   u32    done                               local: CTAs of the current k_group launch that finished their stores
#include <algorithm>

#include "sb_common.cuh"
#include "sb_model.h"

namespace {

__device__ __forceinline__ unsigned long long ld_acquire_sys(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long gtime_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Waits (bounded) until every source rank's records of `step` have arrived in this rank's window; optionally
// acknowledges the generation to every producer.  One warp; lane r watches rank r.
__global__ void k_gather_wait(SbGatherDev g, unsigned long long step, int do_ack, unsigned long long timeout_ns, int* counts_out) {
  const int r = threadIdx.x;
  const int gen = (int)(step % (unsigned long long)g.G);
  bool ok = true;
  if (r < g.world) {
    const unsigned long long* a = g.arrive[g.rank] + (size_t)gen * g.world + r;
    const unsigned long long t0 = gtime_ns();
    unsigned long long v;
    while (((v = ld_acquire_sys(a)) >> 8) < step + 1) {
      if (gtime_ns() - t0 > timeout_ns) { ok = false; break; }
      __nanosleep(200);
    }
    if (counts_out) counts_out[r] = ok ? (int)(v & 0xff) : -1;
  }
  ok = __all_sync(0xffffffffu, ok);
  if (!ok && r == 0) atomicExch(g.status, SB_GATHER_TIMEOUT_ARRIVE);
  __threadfence_system();
  if (do_ack && r < g.world) st_release_sys(g.ack[r] + g.rank, step + 1);
}

__global__ void k_gather_ack(SbGatherDev g, unsigned long long step) {
  const int r = threadIdx.x;
  __threadfence_system();
  if (r < g.world) st_release_sys(g.ack[r] + g.rank, step + 1);
}

}  // namespace

static size_t win_data_bytes(const SbGather& g) { return (size_t)g.G * g.world * g.Bmax * g.width * sizeof(float); }
static size_t win_bytes(const SbGather& g) {
  return win_data_bytes(g) + ((size_t)g.G * g.world + g.world) * sizeof(unsigned long long) + 64;
}

void sb_gather_free(SbModel* m) {
  SbGather& g = m->gather;
  for (int r = 0; r < g.world; ++r)
    if (g.peer[r] && r != g.rank) cudaIpcCloseMemHandle(g.peer[r]);
  if (g.local) cudaFree(g.local);
  if (g.status_host) cudaFreeHost(g.status_host);
  if (g.counts_host) cudaFreeHost(g.counts_host);
  g = SbGather();
}

// Device-side view of the exchange for one step (passed by value to k_group / the wait kernels).
SbGatherDev sb_gather_dev(const SbModel* m, unsigned long long step) {
  const SbGather& g = m->gather;
  SbGatherDev d;
  memset(&d, 0, sizeof(d));
  d.on = g.connected ? 1 : 0;
  d.rank = g.rank; d.world = g.world; d.G = g.G; d.Bmax = g.Bmax; d.width = g.width; d.step = step;
  const size_t data_b = win_data_bytes(g);
  for (int r = 0; r < g.world; ++r) {
    char* base = (char*)g.peer[r];
    d.data[r] = (float*)base;
    d.arrive[r] = (unsigned long long*)(base + data_b);
    d.ack[r] = d.arrive[r] + (size_t)g.G * g.world;
  }
  d.done = (unsigned int*)((char*)g.local + data_b + ((size_t)g.G * g.world + g.world) * sizeof(unsigned long long));
  d.status = g.status_dev;
  d.timeout_ns = g.timeout_ns;
  return d;
}

int sb_gather_queue_collect(sb_handle_s* h, SbModel* m, long long step, int B, float* host_dst, int* counts_dev, cudaStream_t s) {
  SbGather& g = m->gather;
  const SbGatherDev d = sb_gather_dev(m, (unsigned long long)step);
  k_gather_wait<<<1, 32, 0, s>>>(d, (unsigned long long)step, 0, g.timeout_ns, counts_dev);
  SB_CHECK_LAUNCH(h);
  const float* src = (const float*)g.local + (size_t)(step % g.G) * g.world * g.Bmax * g.width;
  SB_CUDA(h, cudaMemcpy2DAsync(host_dst, (size_t)B * g.width * sizeof(float), src, (size_t)g.Bmax * g.width * sizeof(float),
                               (size_t)B * g.width * sizeof(float), g.world, cudaMemcpyDeviceToHost, s));
  k_gather_ack<<<1, 32, 0, s>>>(d, (unsigned long long)step);
  SB_CHECK_LAUNCH(h);
  g.consumed = std::max(g.consumed, step + 1);
  return 0;
}

extern "C" {

int sb_gather_init(sb_handle_t h, int model_id, int rank, int world, int generations, void* out_ipc_handle) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_PAF, "sb_gather_init: bottom-up predictor not configured");
  if (!m) return SB_ERR_INVALID;
  if (world < 1 || world > SB_GATHER_MAX_WORLD || rank < 0 || rank >= world || generations < 2 || generations > 64 || !out_ipc_handle)
    return sb_fail(h, SB_ERR_INVALID, "sb_gather_init: bad arguments (world <= %d, 2 <= generations <= 64)", SB_GATHER_MAX_WORLD);
  if (m->B > 255) return sb_fail(h, SB_ERR_UNSUPPORTED, "sb_gather_init: more than 255 frames per rank and step");
  SB_CUDA(h, cudaSetDevice(h->device));
  SB_CUDA(h, cudaDeviceSynchronize());
  sb_gather_free(m);
  SbGather& g = m->gather;
  g.rank = rank; g.world = world; g.G = generations; g.Bmax = m->B;
  g.width = sb_record_width(m->bu.max_instances, m->bu.n_nodes);
  g.timeout_ns = 5ull * 1000 * 1000 * 1000;
  SB_CUDA(h, cudaMalloc(&g.local, win_bytes(g)));
  SB_CUDA(h, cudaMemset(g.local, 0, win_bytes(g)));
  SB_CUDA(h, cudaHostAlloc((void**)&g.status_host, sizeof(int), cudaHostAllocMapped));
  SB_CUDA(h, cudaHostAlloc((void**)&g.counts_host, sizeof(int) * SB_GATHER_MAX_WORLD * 3, cudaHostAllocMapped));   // [collect | slot 0 | slot 1]
  *g.status_host = 0;
  SB_CUDA(h, cudaHostGetDevicePointer((void**)&g.status_dev, g.status_host, 0));
  SB_CUDA(h, cudaHostGetDevicePointer((void**)&g.counts_dev, g.counts_host, 0));
  g.peer[rank] = g.local;
  cudaIpcMemHandle_t hd;
  SB_CUDA(h, cudaIpcGetMemHandle(&hd, g.local));
  static_assert(sizeof(hd) == SB_IPC_HANDLE_BYTES, "CUDA IPC handle size");
  memcpy(out_ipc_handle, &hd, sizeof(hd));
  SB_CUDA(h, cudaDeviceSynchronize());
  return SB_OK;
}

int sb_gather_connect(sb_handle_t h, int model_id, const void* all_ipc_handles) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_ANY, "bad model id");
  if (!m || !m->gather.local || !all_ipc_handles) return sb_fail(h, SB_ERR_INVALID, "sb_gather_connect: call sb_gather_init first");
  SB_CUDA(h, cudaSetDevice(h->device));
  SbGather& g = m->gather;
  for (int r = 0; r < g.world; ++r) {
    if (r == g.rank) continue;
    cudaIpcMemHandle_t hd;
    memcpy(&hd, (const char*)all_ipc_handles + (size_t)r * SB_IPC_HANDLE_BYTES, sizeof(hd));
    cudaError_t e = cudaIpcOpenMemHandle(&g.peer[r], hd, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      g.peer[r] = nullptr;
      return sb_fail(h, SB_ERR_CUDA, "cudaIpcOpenMemHandle(rank %d): %s", r, cudaGetErrorString(e));
    }
  }
  g.connected = true;
  g.step = 0;
  g.consumed = 0;
  m->slots.release();                              // host staging now holds [world][B][width] windows
  return SB_OK;
}

int sb_gather_enabled(sb_handle_t h, int model_id) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_ANY, "bad model id");
  return (m && m->gather.connected) ? 1 : 0;
}

// Device consumer of step `step`: queued on the post-processing stream behind whatever was submitted so far; waits
// for all ranks' records of that step (bounded), then acknowledges the generation.  The window of the step stays
// readable by later work on that stream until `generations` more steps have been pushed by every rank.
int sb_gather_consume_dev(sb_handle_t h, int model_id, int64_t step) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_ANY, "bad model id");
  if (!m || !m->gather.connected) return sb_fail(h, SB_ERR_INVALID, "sb_gather_consume_dev: exchange not connected");
  if (step < 0) step = m->gather.consumed;        // next unconsumed step
  if (step >= m->gather.step) return sb_fail(h, SB_ERR_INVALID, "sb_gather_consume_dev: step %lld was not pushed", (long long)step);
  SB_CUDA(h, cudaSetDevice(h->device));
  k_gather_wait<<<1, 32, 0, h->post_stream>>>(sb_gather_dev(m, (unsigned long long)step), (unsigned long long)step, 1, m->gather.timeout_ns, nullptr);
  SB_CHECK_LAUNCH(h);
  m->gather.consumed = std::max(m->gather.consumed, (long long)step + 1);
  return SB_OK;
}

int sb_gather_window(sb_handle_t h, int model_id, int64_t step, float** out_dev_ptr, int64_t* out_floats) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_ANY, "bad model id");
  if (!m || !m->gather.local || !out_dev_ptr) return sb_fail(h, SB_ERR_INVALID, "sb_gather_window: exchange not initialised");
  const SbGather& g = m->gather;
  *out_dev_ptr = (float*)g.local + (size_t)(step % g.G) * g.world * g.Bmax * g.width;
  if (out_floats) *out_floats = (int64_t)g.world * g.Bmax * g.width;
  return SB_OK;
}

// Host consumer: blocks until the records of `step` from every rank are in out_records_host
// ([world][B][width] float32, rank-major = frame order for contiguous shards); out_counts[r] = frames rank r pushed.
int sb_gather_collect(sb_handle_t h, int model_id, int64_t step, int B, float* out_records_host, int32_t* out_counts) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_ANY, "bad model id");
  if (!m || !m->gather.connected || !out_records_host) return sb_fail(h, SB_ERR_INVALID, "sb_gather_collect: exchange not connected");
  SbGather& g = m->gather;
  if (step < 0 || step >= g.step) return sb_fail(h, SB_ERR_INVALID, "sb_gather_collect: step %lld was not pushed", (long long)step);
  if (B <= 0 || B > g.Bmax) return sb_fail(h, SB_ERR_INVALID, "sb_gather_collect: bad batch");
  SB_CUDA(h, cudaSetDevice(h->device));
  cudaStream_t s = h->post_stream;
  int rc = sb_gather_queue_collect(h, m, step, B, out_records_host, g.counts_dev, s);
  if (rc) return rc;
  SB_CUDA(h, cudaStreamSynchronize(s));
  if (out_counts) for (int r = 0; r < g.world; ++r) out_counts[r] = g.counts_host[r];
  if (*g.status_host != 0) {
    const int st = *g.status_host;
    *g.status_host = 0;
    return sb_fail(h, SB_ERR_CUDA, "record exchange timed out (%s): a peer rank stopped pushing or consuming",
                   st == SB_GATHER_TIMEOUT_ARRIVE ? "waiting for arrivals" : "waiting for acknowledgements");
  }
  return SB_OK;
}

int sb_gather_status(sb_handle_t h, int model_id, int32_t* out_status, int64_t* out_steps_pushed, int64_t* out_steps_consumed) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_ANY, "bad model id");
  if (!m || !m->gather.local) return sb_fail(h, SB_ERR_INVALID, "sb_gather_status: exchange not initialised");
  if (out_status) *out_status = *m->gather.status_host;
  if (out_steps_pushed) *out_steps_pushed = m->gather.step;
  if (out_steps_consumed) *out_steps_consumed = m->gather.consumed;
  return SB_OK;
}

int sb_gather_close(sb_handle_t h, int model_id) {
  SbModel* m = chain_model(h, model_id, SB_CHAIN_ANY, "bad model id");
  if (!m) return sb_fail(h, SB_ERR_INVALID, "bad model id");
  SB_CUDA(h, cudaSetDevice(h->device));
  SB_CUDA(h, cudaDeviceSynchronize());
  sb_gather_free(m);
  return SB_OK;
}

}  // extern "C"
