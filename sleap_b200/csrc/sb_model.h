// Internal model structures (op-list, buffers) shared by sb_model.cu, sb_entry.cu, sb_conv_tc.cu and sb_conv01.cu.
// The int32 record layout must match sleap_b200/nn/oplist.py.
#pragma once
#include <functional>
#include <initializer_list>
#include <vector>

#include "sb_common.cuh"

enum {
  SB_OPK_BUFFER = 0,
  SB_OPK_CONV = 1,
  SB_OPK_TCONV = 2,
  SB_OPK_POOL = 3,
  SB_OPK_UPSAMPLE = 4,
  SB_OPK_ADD = 5,
  SB_OPK_PREPROCESS = 6,
  SB_OPK_COPY = 7,
};
enum { SB_OPF_RELU = 1, SB_OPF_BN = 2, SB_OPF_BILINEAR = 8, SB_OPF_FUSED_POOL = 16, SB_OPF_EXPLICIT_PAD = 32,
       SB_OPF_FUSED_ADD = 64, SB_OPF_RESIDUAL = 128 };
// PREPROCESS modes: IMAGENET_CAFFE(_GRAY) = pretrained ResNet trained on colour (grayscale) frames; _GRAY converts
// colour frames to gray before tile_channels
enum { SB_PRE_PLAIN = 0, SB_PRE_IMAGENET_CAFFE = 1, SB_PRE_IMAGENET_CAFFE_GRAY = 2 };

struct SbOp {
  int32_t w[SB_OP_WORDS];
  int kind() const { return w[0]; }
  int in_buf() const { return w[1]; }
  int in_coff() const { return w[2]; }
  int in_C() const { return w[3]; }
  int in2_buf() const { return w[4]; }
  int in2_coff() const { return w[5]; }
  int out_buf() const { return w[6]; }
  int out_coff() const { return w[7]; }
  int out_C() const { return w[8]; }
  int k() const { return w[9]; }
  int stride() const { return w[10]; }
  int flags() const { return w[11]; }
  int w_off() const { return w[12]; }
  int b_off() const { return w[13]; }
  int bn_scale_off() const { return w[14]; }
  int bn_shift_off() const { return w[15]; }
  // CONV: w[18] = buffer of a fused 2x2 max-pool output (-1: none), w[19] = its channel offset;
  //       the POOL op that follows carries flag SB_OPF_FUSED_POOL and is skipped when the conv
  //       ran on the tensor-core path.
  int pool_buf() const { return w[18]; }
  int pool_coff() const { return w[19]; }
  // CONV with SB_OPF_EXPLICIT_PAD: w[16] / w[17] = top / left zero padding (otherwise TF SAME, derived from the shapes)
  bool explicit_pad() const { return (w[11] & SB_OPF_EXPLICIT_PAD) != 0; }
  int pad_top() const { return w[16]; }
  int pad_left() const { return w[17]; }
  // CONV with SB_OPF_RESIDUAL: the ADD op right after it (flag SB_OPF_FUSED_ADD) sums this conv's output and the
  // shortcut slice (w[20], w[21]) into the sum slice (w[22], w[23]); the tensor-core path does it in the epilogue and
  // the ADD op is then skipped
  bool residual() const { return (w[11] & SB_OPF_RESIDUAL) != 0; }
  int res_buf() const { return w[20]; }
  int res_coff() const { return w[21]; }
  int sum_buf() const { return w[22]; }
  int sum_coff() const { return w[23]; }
  // PREPROCESS: w[16] = float bits of input_scale, w[17] = pad_to_stride, w[19] = SB_PRE_* mode
  float input_scale() const { float f; memcpy(&f, &w[16], 4); return f; }
  int pad_stride() const { return w[17]; }
  int pre_mode() const { return w[19]; }
};

struct SbBuffer {
  int id = 0, stride_den = 1, C = 0, f32 = 0, is_input = 0;
  int H = 0, W = 0;
  void* dev = nullptr;
};

struct SbConvTcPlan;  // sb_conv_tc.cu
struct SbConv01Plan;  // sb_conv01.cu
struct SbTopdown;     // sb_topdown.cu

// One op's slot of a program: its launches for a batch of B frames (the frames feed the input stage), everything else
// fixed at configure time.  An empty slot launches nothing: its op runs inside a neighbour's launch.
using SbLaunchFn = std::function<int(sb_handle_s* h, const void* frames_dev, int frames_are_u8, int B)>;

// The input stage (sb_entry.cu): how a forward pass gets from the raw frame to the first activation the op loop reads.
// Resolved and timed once by sb_model_configure, which then fills the slots it covers in both programs.
enum {
  SB_ENTRY_GENERIC = 0,    // k_preprocess as an ordinary op, then the op loop
  SB_ENTRY_DIRECT,         // k_conv_first: the first conv on the CUDA cores, preprocessing fused
  SB_ENTRY_FRAME_VIEW,     // k_first_view of the frame, then the first conv as a Toeplitz GEMM on the tensor cores
  SB_ENTRY_BUFFER_VIEW,    // k_preprocess, k_first_view of its one-channel output, then the Toeplitz GEMM
  SB_ENTRY_STEM_VIEW,      // k_s2d_view of the frame, then the 7x7 stride-2 stem as a 4x4 GEMM on the tensor cores
};
struct SbEntryPlan {
  int route = SB_ENTRY_GENERIC;
  int pre_op = -1;                 // the PREPROCESS op when the first conv's launch preprocesses the frame (an empty slot)
  int conv_op = -1;                // the first conv, unless the route is generic
  int conv1_op = -1;               // conv1 when the fused first block won: in the production program, k_conv01 runs in
                                   // conv_op's slot and the slots of conv1 and its pool are empty
  SbConv01Plan* conv01 = nullptr;  // fused first encoder block k_conv01 over conv_op and conv_op + 1 (sb_conv01.cu)
  __half* view = nullptr;          // view routes: the [B][view_H][view_W][16] fp16 view the GEMM reads
  float* view_bias = nullptr;      // Toeplitz view: the bias replicated over the 8 pixels of a group
  int view_H = 0, view_W = 0;
  int pre_mode = SB_PRE_PLAIN;     // stem view: the PREPROCESS mode k_s2d_view applies
};

// The post-processing chain a model runs after its network (include/sleap_b200.h): one at a time.  Every configure call,
// sb_model_configure's included, drops the previous chain with its tracker and record exchange.  The fused top-down
// pipeline is a layer over a centroid chain and a global chain, valid while neither model's chain_gen moves.
enum { SB_CHAIN_ANY = -1, SB_CHAIN_NONE = 0, SB_CHAIN_PAF, SB_CHAIN_CLASS, SB_CHAIN_GLOBAL, SB_CHAIN_CENTROID };

// The two slots of a streamed (submit / collect) step and the rules of the streamed steps (include/sleap_b200.h): a
// submit goes into a slot that holds no batch; a collect takes a slot's batch with its B, oldest first; a slot read
// takes the batch last collected from that slot with its B; a synchronous call runs one batch into slot 0 and collects it,
// and is refused while a batch is submitted and not collected.  A check that fails returns SB_ERR_INVALID with `what`
// before its message and changes nothing.  Buffers, stream and events are allocated by the first submit or synchronous
// call after release().
struct SbSlots {
  cudaStream_t copy_stream = nullptr;
  void* frames[2] = {nullptr, nullptr};            // device uint8 frames of the slot's batch
  float* stage[2] = {nullptr, nullptr};            // pinned result staging
  // h2d_done: the slot's upload landed; frames_free: the last read of its frames is done; result: its results are staged
  cudaEvent_t h2d_done[2] = {nullptr, nullptr}, frames_free[2] = {nullptr, nullptr}, result[2] = {nullptr, nullptr};
  int slot_B[2] = {0, 0};                          // frames of the batch the slot holds (submitted, not collected; 0: none)
  int done_B[2] = {0, 0};                          // frames of the batch last collected from the slot (0: none)
  unsigned long long slot_seq[2] = {0, 0}, seq = 0;   // submit number of the slot's last batch (0: none since allocation)

  int alloc(sb_handle_s* h, size_t frame_bytes, size_t stage_floats);
  int check_submit(sb_handle_s* h, const char* what, int slot, int B, int max_B, const void* frames_host) const;
  // The batch's frames (`bytes`), then the copies `more`, into `slot` on the copy stream once the work that last read
  // the slot's frames is done; h2d_done[slot] marks their end.  The caller makes its stream wait on it.
  struct Copy { void* dst; const void* src; size_t bytes; };
  int upload(sb_handle_s* h, int slot, const void* frames_host, size_t bytes, std::initializer_list<Copy> more = {});
  void submitted(int slot, int B) { slot_B[slot] = B; done_B[slot] = 0; slot_seq[slot] = ++seq; }
  void drop(int slot) { slot_B[slot] = 0; }        // a submitted batch whose work could not be queued
  int check_collect(sb_handle_s* h, const char* what, int slot, int B) const;
  int collect(sb_handle_s* h, int slot);           // waits for result[slot]; the slot is free again
  int check_read(sb_handle_s* h, const char* what, int slot, int B) const;
  bool busy() const { return slot_B[0] || slot_B[1]; }
  int check_idle(sb_handle_s* h, const char* what) const;   // refuses a synchronous call while busy()
  void release();
};

struct SbModel {
  int precision = 0;  // 0: fp16 activations + tensor-core convs; 1: fp32 CUDA-core path
  std::vector<SbOp> ops;
  std::vector<SbBuffer> buffers;
  std::vector<float> weights_host;
  float* weights_dev = nullptr;
  void* weights_tc_dev = nullptr;   // fp16 [tap][Cout][Cin] copies for the tensor-core path
  int64_t n_weights = 0;
  bool configured = false;
  int B = 0, Hin = 0, Win = 0, Cin = 0, Hres = 0, Wres = 0, Hnet = 0, Wnet = 0;
  size_t act_bytes = 0;
  void* frames_dev = nullptr;
  std::vector<SbConvTcPlan*> tc_plans;  // per op (nullptr = direct path)
  // The forward pass, one slot per op, built at the end of sb_model_configure: prog[0] is the production program (stores
  // nobody reads inside the network elided, fused POOL and ADD slots empty, k_conv01 where it won), prog[1] stores every
  // tensor (a fused residual ADD and the first block's convs as their own launches) for a forward that asks for one of them
  std::vector<SbLaunchFn> prog[2];
  std::vector<int> op_kind;             // per op, as sb_model_profile_ops reports it
  std::vector<char> buf_elided;         // per buffer: the production program may not store it
  std::vector<cudaEvent_t> prof_events; // non-empty only inside sb_model_profile_ops
  std::vector<cudaEvent_t> fwd_events;  // sb_model_forward_times: (start, end) pairs around every forward pass
  int fwd_n = 0;                        // pairs recorded since the last read
  bool fwd_timing = false;
  // post-processing chain: `chain` says which of the parameter structs bu / mc / gl / ce is live; chain_gen counts the
  // drops (sb_topdown_configure records it)
  int chain = SB_CHAIN_NONE;
  unsigned chain_gen = 0;
  SbPostWs ws;
  sb_bottomup_params bu{};
  std::vector<int> bu_edges;
  sb_multiclass_params mc{};
  int guard_op = -1;                       // first op that overwrites a head buffer the post-processing stream may still read
  // the steps of the chain (sb_infer_bottomup / _multiclass / _global into slot 0, and the streamed sb_bottomup_*,
  // sb_multiclass_*, sb_global_*), staging the chain's records
  SbSlots slots;
  sb_global_params gl{};
  SbGlobalScratch gs;
  sb_centroid_params ce{};
  SbTopdown* td = nullptr;                 // fused top-down pipeline (sb_topdown_configure), held by its centroid model
  SbEntryPlan entry;                       // input stage (sb_entry.cu)
  SbGather gather;                         // peer-memory exchange of the result records (sb_gather.cu)
  // device tracker run after the grouping kernel (sb_bottomup_attach_tracker, sb_track.cu) or, on a top-down pipeline's
  // centroid model, after its record kernel (sb_topdown_attach_tracker); its per-frame track records
  // ([B][sb_track_record_width] doubles) live beside the result records and travel with the result copy
  SbTracker* trk = nullptr;
  int trk_B = 0, trk_I = 0, trk_cut = -1;
  double trk_h = 1.0, trk_w = 1.0;
  double* trk_dev = nullptr;
  double* trk_host[2] = {nullptr, nullptr};   // pinned: slots 0 / 1
};

// The network input of H x W frames as sb_model_configure plans it: resized by the PREPROCESS op's input_scale
// (Hres x Wres), then padded to its pad_to_stride (Hnet x Wnet).  Fails for a model without a PREPROCESS op.
int sb_net_size(sb_handle_s* h, const SbModel* m, int H, int W, int* Hres, int* Wres, int* Hnet, int* Wnet);

// one forward pass: the production program, or the all-stores one
int sb_run_ops(sb_handle_s* h, SbModel* m, const void* frames_dev, int frames_are_u8, int B, bool all_stores = false);

// Model `id` of the handle when its chain is `kind` (SB_CHAIN_ANY: any chain); otherwise fails with `what`, nullptr
SbModel* chain_model(sb_handle_s* h, int id, int kind, const char* what);

void sb_topdown_free(SbModel* m);        // sb_topdown.cu
bool sb_topdown_busy(const SbModel* m);  // the model's top-down pipeline holds a submitted batch not yet collected

// Sizes the model's track records (trk_dev, trk_host) for B frames of a tracker of I instances; keeps larger ones
int sb_track_records_alloc(sb_handle_s* h, SbModel* m, int B, int I);

// record exchange (sb_gather.cu)
SbGatherDev sb_gather_dev(const SbModel* m, unsigned long long step);
void sb_gather_free(SbModel* m);
// queues on `s`: wait for every rank's records of `step`, copy the [world][B][width] window to host_dst, acknowledge
int sb_gather_queue_collect(sb_handle_s* h, SbModel* m, long long step, int B, float* host_dst, int* counts_dev, cudaStream_t s);

// tensor-core conv path (sb_conv_tc.cu)
int sb_conv_tc_prepare(sb_handle_s* h, SbModel* m);      // after buffers are allocated
int sb_conv_tc_autotune(sb_handle_s* h, SbModel* m);     // launch forms of every plan, the input stage's included
void sb_conv_tc_release(SbModel* m);
// The slot of op `op_index` (which has a plan) in the production program or, all_stores, in the all-stores program
struct SbTcEntry {
  SbLaunchFn run;
  int absorbs = -1;         // the op after it (a fused POOL, or a fused residual ADD in production) whose slot is empty
  bool elides_out = false;  // its own output is not stored
};
SbTcEntry sb_conv_tc_entry(const SbModel* m, int op_index, bool all_stores);
// A stride-1 R x S convolution over a [B][H][W][16] fp16 view that is not an op-list buffer, as the plan of op
// `op_index`: output pixel (y, x) takes tap (r, s) from view pixel (y + dy0 + r, x + dx0 + s), with the weights
// w[r * S + s] ([R * S][Cout][16]).  Leaves the op without a plan where the view is smaller than one TMA box.
struct SbTcView {
  SbBuffer in;                     // the view (C = 16)
  SbBuffer out;                    // the output tensor as the GEMM sees it (C = its row pitch)
  int Cout = 0, out_coff = 0;
  int R = 0, S = 0, dy0 = 0, dx0 = 0;
  const float *bias = nullptr, *bn_scale = nullptr, *bn_shift = nullptr;
  int relu = 0;
};
int sb_conv_tc_view_prepare(sb_handle_s* h, SbModel* m, int op_index, const SbTcView& v, const std::vector<float>& w);
void sb_conv_tc_drop(SbModel* m, int op_index);          // frees the op's plan
// configure-time timing: the time of run() in ms, 4 synchronised runs, the first dropped, the minimum of the others
int sb_time_min(sb_handle_s* h, const char* what, float& best, const std::function<int()>& run);

// input stage (sb_entry.cu)
int sb_entry_prepare(sb_handle_s* h, SbModel* m);       // after sb_conv_tc_prepare: route, views, fused block
int sb_entry_autotune(sb_handle_s* h, SbModel* m);      // after sb_conv_tc_autotune: direct vs view, fused vs separate
// fills the slots the input stage covers in m->prog[all_stores], marks them (and the fused block's pool) in `taken`;
// flags the fused block's two tensors in m->buf_elided
void sb_entry_build(SbModel* m, bool all_stores, std::vector<char>& taken);
void sb_entry_release(SbModel* m);

// fused first encoder block, run by the input stage (sb_conv01.cu)
int sb_conv01_prepare(sb_handle_s* h, SbModel* m, int conv0_op, int conv1_op);   // sets m->entry.conv01
void sb_conv01_release(SbModel* m);
int sb_conv01_launch(sb_handle_s* h, const SbConv01Plan* pl, const void* frames_dev, int frames_are_u8, int B);

// programmatic dependent launch for the conv kernels (sb_conv_tc.cu); SB_DISABLE_PDL=1 switches it off
bool sb_pdl_on();

// Launches `kernel` (args: pointers to its arguments, as for cudaLaunchKernelExC) with programmatic stream
// serialization while sb_pdl_on(): its CTAs may start while the kernel before it on the stream drains.
inline cudaError_t sb_launch_pdl(const void* kernel, dim3 grid, dim3 block, size_t smem, cudaStream_t stream, void** args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = sb_pdl_on() ? 1 : 0;
  return cudaLaunchKernelExC(&cfg, kernel, args);
}
