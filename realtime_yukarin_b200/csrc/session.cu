// session.cu -- one audio stream's encode -> convert -> decode chain kept resident in HBM and run as a
// three-stage software pipeline on three CUDA streams.
//
// Semantics = the reference's three StreamWrapper-driven stages as the workers run them
// (realtime_voice_conversion/worker/{encode,convert,decode}_worker.py with stream/*.py): stage input chunk j
// is added at start_time = extra + j*T and step k processes [k*T - extra, k*T + T + extra), i.e. window item i
// of step k is item k*n - 2e + i of the stage's input sequence, silent where that is negative (SURVEY A.9a,
// verified against the reference's BaseStream.fetch).  Instead of Python segment lists each stage keeps its
// last window on the device and slides it by one chunk per step:
//   wave window      (n_wave + 2 e_wave samples)                                -> WORLD analysis -> trim
//   feature window   (n_feat + 2 e_conv frames of f0/ap/mc/voiced + aligned samples) -> gate, stage 1, stage 2 -> trim
//   converted window (n_feat + 2 e_dec frames of f0/ap/sp)                      -> realtime synthesizer -> NaN scrub
//
// Pipelining = what run.py does with three OS processes and queues (run.py:58-93), done with streams and events:
//   stream E: slide wave (+ input resampler)                                                           of chunk k+1
//   stream A: DIO/StoneMask (or CREPE), then CheapTrick || D4C (two branches of one graph)             of chunk k+1
//   stream C: head (slide features, silence gate), then stage-1 U-Net (+f0 map), mc2sp                 of chunk k
//   stream C2: stage-2 U-Net (the wgmma layers)                                                     of chunk k-1
//   stream D: slide converted features, synthesizer add/plan/pulse/overlap-add, NaN scrub             of chunk k-2
// Inter-stage buffers are double-buffered (index = step parity), except the stage-1 -> stage-2 -> decode hand-off set, which has three
// slots (index = step % 3) so that stage 1 of a chunk does not wait for stage 2 of the chunk two steps before; events order
// producer/consumer and guard reuse.
// The effective-frame count that selects the stage-1 plan (T_eff + 128 - T_eff % 128) is read on the device by a
// conditional graph node, so the host never waits inside a step.
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <array>
#include <numeric>
#include <vector>

#include "../../include/ryk.h"
#include "engine.h"
#include "features.h"
#include "synth.h"
#include "unet.h"

namespace ryk {

constexpr int kRing = 8;          // event / output-slot ring (pipeline depth is bounded by the buffer guards below)
constexpr int kHandoff = 3;       // slots of the stage-1 -> stage-2 -> decode hand-off buffers (cv_*), h = step % kHandoff
constexpr int kHandoffGraphs = 6; // graphs that read or write both a parity buffer and a hand-off slot: one per step % 6 = (b, h)

// One captured stage of a step (see run_graph).  Destroying it drops the executable graph.
struct StageGraph {
  cudaGraphExec_t exec = nullptr; long long launches = 0;       // launches: kernel nodes of the graph (one launch runs them all)
  StageGraph() = default;
  StageGraph(const StageGraph&) = delete;
  StageGraph& operator=(const StageGraph&) = delete;
  ~StageGraph() { reset(); }
  void reset() { if (exec) cudaGraphExecDestroy(exec); exec = nullptr; launches = 0; }
};
// The stage graphs of the chunks of one parity, in step order.
struct ParityGraphs {
  StageGraph gate;         // stream E: wave slides (the "gate" stage of RYK_STAGE_TIMES; the silence gate itself runs in s1_head)
  StageGraph analysis;     // stream A: DIO/Harvest + StoneMask, then CheapTrick || D4C
  StageGraph s1_head;      // stream C: feature-window slides + silence gate (mask / index / count of the step)
  StageGraph s2_layers;    // single session: stage-2 layers 1..14
  StageGraph synth;        // stream D: synthesizer + NaN scrub
};
// The stage graphs that touch the hand-off slot h as well as parity buffers, for the chunks of one step % 6 (b = j & 1, h = j % 3).
struct HandoffGraphs {
  // stream C: the rest of stage 1 with the padded-length bucket chosen ON THE DEVICE = {k_set_bucket -> SWITCH conditional node whose
  // body i is the stage-1 sequence for the padded length 128 i (0: no effective frame)}; built at session creation, no host sync
  StageGraph s1;
  StageGraph s2_pro;       // stage-2 prologue (single session: + layer 0; group member: into the group's batched input)
  StageGraph s2_epi;       // stage-2 epilogue (single session: layer 15 +; group member: from the group's batched output)
  StageGraph dec_slide;    // stream D: decode-window slides
};
// Events of one ring slot r = step % kRing.  Null until created, so a partly built session can be freed.
struct StepEvents {
  cudaEvent_t gate = nullptr;      // wave slides of step r done (stream E)
  cudaEvent_t enc = nullptr;       // analysis of step r done
  cudaEvent_t cslide = nullptr;    // head of stage 1 of step r done: enc_*[b] and cw_wave[g] consumed
  cudaEvent_t s1 = nullptr;        // stage 1 of step r done
  cudaEvent_t pro = nullptr;       // stage-2 prologue of step r done (group members only)
  cudaEvent_t conv = nullptr;      // stage 2 of step r done
  cudaEvent_t dslide = nullptr;    // the converted features of step r sit in the decode window
  cudaEvent_t dec = nullptr;       // output of step r staged (after the copies the entry point appends to stream D)
  std::array<cudaEvent_t*, 8> all() { return {&gate, &enc, &cslide, &s1, &pro, &conv, &dslide, &dec}; }
};
struct Group;
struct Session {
  // optional per-stage device timing (RYK_STAGE_TIMES=1): [stage E1,E2,S1,S2,D][begin/end][ring]
  cudaEvent_t tev[5][2][kRing]; bool stage_times = false;
  // plan-cache owner ids (activation buffers are private to the session): stage 1, and stage 2 of even / odd chunks
  int s1_owner = 0, s2_owner[2] = {0, 0};
  float* d_colmin[2] = {nullptr, nullptr};
  Group* group = nullptr; int slot = 0;        // member of a batched stage-2 group (config 5), else nullptr
  Voice* voice = nullptr; int voice_id = 0;    // the voice the session converts into (fixed for its lifetime)
  ryk_session_config cfg;
  SptkMats sptk;                   // the engine's sp2mc / mc2sp matrices of cfg's (order, alpha, fft_length), captured in the graphs
  int hop, rate, n_wave, n_feat, e_wave, e_enc_frames, e_conv, e_dec;
  int Lw, Tw, Td, nb, C;
  int Tp;                          // stage-2 padded length: Tw rounded up to the next multiple of 128 (always > Tw)
  long long step = 0;              // chunks submitted
  long long collected = 0;         // chunks collected through the host API
  cudaStream_t sE = nullptr, sC = nullptr, sD = nullptr;     // gate | stage 1 | decode
  // stage 2 of even / odd chunks on two streams with two activation plans (a group member uses only the first): the latency-bound
  // bottleneck layers (c4-d2: 30 % of a forward's time, a few CTAs each) of one chunk overlap the GPU-filling layers of its neighbour
  cudaStream_t sC2s[2] = {nullptr, nullptr};
  cudaStream_t sA[2] = {nullptr, nullptr};   // WORLD analysis of even / odd chunks: two chunks' analyses may be in flight
  cudaStream_t sA_side = nullptr;            // D4C branch of the analysis graphs while they are captured; never used at step time
  std::array<cudaStream_t, 7> streams() const { return {sE, sA[0], sA[1], sC, sC2s[0], sC2s[1], sD}; }
  StepEvents ev[kRing];
  // sliding windows, double-buffered by step parity
  float* wave_win[2];
  float *cw_f0[2], *cw_ap[2], *cw_mc[2], *cw_wave[2]; uint8_t* cw_voiced[2];
  float *dw_f0[2], *dw_ap[2], *dw_sp[2];
  // inter-stage buffers, double-buffered by step parity
  float *enc_f0[2], *enc_sp[2], *enc_ap[2], *enc_mc[2]; uint8_t* enc_voiced[2];
  double* d_mse; uint8_t* d_mask[2]; int* d_index[2]; int* d_count[2];
  // the hand-off set: written by stage 1 (and cv_sp_out by the stage-2 epilogue), read by stage 2 and the decode slide; slot = step % 3
  float *cv_mc_out[kHandoff], *cv_f0_out[kHandoff], *cv_ap_out[kHandoff], *cv_sp_out[kHandoff]; uint8_t* cv_voiced_out[kHandoff];
  float* cv_sp_mid[kHandoff];
  double* dec_f0_f64;
  int max_blocks;
  // host-API staging rings (pinned host + device), slot = step % kRing
  float* d_chunk[kRing]; float* h_in[kRing];
  double* d_out[kRing]; double* h_out[kRing];
  int* d_n_out[kRing]; int* h_n[kRing];
  float* d_chunk_fixed = nullptr;      // the chunk the (captured) encode graph reads
  double* d_out_fixed[2];              // blocks written by the (captured) decode graph, by parity
  int* d_n_fixed[2];
  ParityGraphs graphs[2];
  HandoffGraphs hgraphs[kHandoffGraphs];
  Synth* synth = nullptr;
  DioPlan* dio[2] = {nullptr, nullptr};     // one analysis plan per chunk parity (owned), f0 methods 0 and 1
  CrepePlan* crepe[2] = {nullptr, nullptr}; // f0 method 2: one CREPE forward per chunk parity (owned) in place of DIO/Harvest
  // Device rates (ryk_session_set_input_rate / _output_rate): chunks arrive at in.rate and outputs leave at out.rate; analysis, the
  // U-Nets and synthesis stay at cfg.fs.  rate 0 = that side runs at fs (no resampler).
  struct RateSide {
    int rate = 0, up = 1, down = 1, n_taps = 0;
    int hist = 0;                                 // input: history window (chunk + left support); output: kept synthesizer samples
    double* d_h = nullptr;
    ResampleState* d_st = nullptr;                // [2] by step parity
  } in, out;
  int n_in = 0;                    // samples per pushed chunk (n_wave without an input resampler)
  int delay_in = 0;                // leading zeros of the model-rate input (model samples)
  int max_out = 0;                 // most output samples one step can return
  float* in_win[2] = {nullptr, nullptr};      // input history windows (in.hist device-rate samples)
  float* d_chunk_model = nullptr;             // the step's resampled chunk (n_wave model-rate samples)
  double* out_hist[2] = {nullptr, nullptr};   // kept synthesizer samples (out.hist)
  double* d_rout_fixed[2] = {nullptr, nullptr}; int* d_rn_fixed[2] = {nullptr, nullptr};   // device-rate output of a step, by parity
  // The session's f0 map (ryk_session_set_f0_map / _f0_follow) and the statistics of its speaker (ryk_session_f0_measure).  The captured
  // stage-1 graphs read *d_f0_map; f0_map_sync brings it up to date on stream C in front of a step's stage 1.
  F0Map f0_map = {};               // what the next submitted step uses (follow mode: its input side is the fallback)
  bool f0_dirty = false;           // f0_map changed since the last submitted step
  bool f0_measure = false;         // the head of stage 1 ends with k_f0_measure
  bool f0_reset = false;           // the statistics restart at the next submitted step
  F0Map* d_f0_map = nullptr; F0Stats* d_f0_stats = nullptr;
  F0Map* h_f0_map = nullptr;       // pinned staging, slot = step % kRing
  std::vector<void*> allocs, pinned;
};

// Several sessions on one GPU sharing ONE batched stage-2 forward per step (BASELINE config 5: 8 streams per GPU,
// stage-2 input (B, 1, Tp, 512)).  Everything else (analysis, gate, stage 1, synthesis) stays per stream: those
// stages carry per-stream state and data-dependent lengths, and they are a small share of the SM time.
// Members may join and leave between steps (ryk_group_add / _remove): group_rebuild then builds p2 anew around the new member list.
struct Group {
  std::vector<Session*> members;               // in slot order: member i reads and writes batch item i of p2
  std::vector<Voice*> voices;                  // the members' distinct voices in the order of their first member; p2 lives on voices[0]
  int owner = 0;                               // plan-cache owner id of p2
  UNetPlan* p2 = nullptr;                      // stage-2 plan at batch = members.size(), member i on the weights of its voice
  cudaStream_t sG = nullptr;
  cudaEvent_t ev_fwd[kRing] = {};              // batched forward of step r done
  long long step = 0, collected = 0;
  StageGraph fwd_graph;
};

// dst = [old[shift..L), new[0..shift)] row-wise (rows of `row` elements)
template <typename T>
__global__ void k_slide(const T* __restrict__ old_, const T* __restrict__ new_, T* __restrict__ dst, size_t L, size_t shift, size_t row) {
  size_t total = L * row;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    size_t r = i / row;
    dst[i] = r + shift < L ? old_[i + shift * row] : new_[i - (L - shift) * row];
  }
}

// several windows slid by one launch (blockIdx.y = window): dst = [old[shift..L), new[0..shift)] in units of `elem` bytes
struct SlideDesc { const void* old_; const void* new_; void* dst; size_t L, shift, row; int elem; };
struct SlideBatch { SlideDesc d[5]; int n; };
__global__ void k_slide_multi(SlideBatch b) {
  const SlideDesc& d = b.d[blockIdx.y];
  size_t total = d.L * d.row;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    size_t r = i / d.row;
    bool keep = r + d.shift < d.L;
    size_t src = keep ? i + d.shift * d.row : i - (d.L - d.shift) * d.row;
    if (d.elem == 4) ((uint32_t*)d.dst)[i] = keep ? ((const uint32_t*)d.old_)[src] : ((const uint32_t*)d.new_)[src];
    else ((uint8_t*)d.dst)[i] = keep ? ((const uint8_t*)d.old_)[src] : ((const uint8_t*)d.new_)[src];
  }
}

template <typename T>
__global__ void k_fill_rows(T* __restrict__ dst, size_t rows, size_t row, T first, T rest) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < rows * row; i += (size_t)gridDim.x * blockDim.x)
    dst[i] = (i % row == 0) ? first : rest;
}

__global__ void k_f32_to_f64(const float* __restrict__ a, double* __restrict__ b, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) b[i] = (double)a[i];
}

// ---- output re-blocker + silence gate (SURVEY 8(f) rank 2; realtime_voice_conversion/worker/decode_worker.py:38-59) ----
// The reference's decode worker concatenates the synthesizer blocks into `wave_fragment`, cuts one out_audio_chunk off its
// front whenever enough samples are queued (at most one per step) and drops the chunk when its mean STFT power is below
// -output_silent_threshold dB.  Here the fragment lives in HBM (ping-pong buffers), the sample count of a step is read from
// device memory (no host sync) and the gate kernels (world_synth.cu) are predicated on the device-side "chunk emitted" flag.
struct ReblockState { int len, sel, overflow; };
struct Reblock {
  int chunk = 0, max_in = 0, cap = 0, n_fft = 2048, hop = 512;
  double threshold_db = 80.0;
  ReblockState* d_state = nullptr;
  double* d_frag[2] = {nullptr, nullptr};
  double* d_scratch = nullptr;
  double* d_chunk[kRing]; int* d_nvalid[kRing]; int* d_status[kRing]; double* d_power[kRing];
  double* h_chunk[kRing]; int* h_status[kRing]; double* h_power[kRing]; int* h_overflow[kRing];
  cudaEvent_t ev[kRing];
  double* d_stage_in = nullptr; int* d_stage_n = nullptr;     // staging for the host-buffer entry point
  long long pushed = 0;
  std::vector<void*> allocs, pinned;
};

static void reblock_free(Reblock* R) {
  if (!R) return;
  for (int i = 0; i < kRing; ++i) if (R->ev[i]) cudaEventDestroy(R->ev[i]);
  for (void* p : R->allocs) cudaFree(p);
  for (void* p : R->pinned) cudaFreeHost(p);
  delete R;
}

__global__ void __launch_bounds__(1024) k_reblock(ReblockState* __restrict__ st, double* __restrict__ frag0, double* __restrict__ frag1, int cap,
                                                 const double* __restrict__ in, const int* __restrict__ n_in_p, int max_in, int chunk,
                                                 double* __restrict__ out, int* __restrict__ n_valid) {
  __shared__ int sh_len, sh_sel;
  if (threadIdx.x == 0) { sh_len = st->len; sh_sel = st->sel; }
  __syncthreads();
  const int len = sh_len, sel = sh_sel;
  int n_in = *n_in_p;
  if (n_in < 0) n_in = 0;
  int clamped = 0;
  if (n_in > max_in) { n_in = max_in; clamped = 1; }
  double* cur = sel ? frag1 : frag0;
  double* nxt = sel ? frag0 : frag1;
  const int new_len = len + n_in;
  if (new_len >= chunk) {
    int rest = new_len - chunk, over = 0;
    if (rest > cap) { rest = cap; over = 1; }
    for (int i = threadIdx.x; i < chunk; i += blockDim.x) out[i] = i < len ? cur[i] : in[i - len];
    for (int j = threadIdx.x; j < rest; j += blockDim.x) { const int i = chunk + j; nxt[j] = i < len ? cur[i] : in[i - len]; }
    if (threadIdx.x == 0) { st->len = rest; st->sel = sel ^ 1; st->overflow |= over | clamped; *n_valid = chunk; }
  } else {
    for (int i = threadIdx.x; i < n_in; i += blockDim.x) cur[len + i] = in[i];
    if (threadIdx.x == 0) { st->len = new_len; st->overflow |= clamped; *n_valid = 0; }
  }
}

// NaN -> 0 on the produced samples (decode_stream.py:38) and publish the sample count
__global__ void k_scrub(double* __restrict__ y, const SynthState* __restrict__ st, int block, int max_samples, int* __restrict__ n_out) {
  int n = st->blocks_out * block;
  if (n > max_samples) n = max_samples;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) { double v = y[i]; if (v != v) y[i] = 0.0; }
  if (blockIdx.x == 0 && threadIdx.x == 0) *n_out = n;
}

template <typename T>
static int slide(const T* old_, const T* new_, T* dst, size_t L, size_t shift, size_t row, cudaStream_t st) {
  size_t total = L * row;
  if (total == 0) return 0;
  int blocks = (int)((total + 255) / 256); if (blocks > 2368) blocks = 2368;
  k_slide<T><<<blocks, 256, 0, st>>>(old_, new_, dst, L, shift, row);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

static int slide_batch(SlideBatch& b, cudaStream_t st) {
  size_t mx = 0;
  for (int i = 0; i < b.n; ++i) { size_t t = b.d[i].L * b.d[i].row; if (t > mx) mx = t; }
  if (mx == 0) return 0;
  int blocks = (int)((mx + 255) / 256); if (blocks > 592) blocks = 592;
  k_slide_multi<<<dim3(blocks, b.n), 256, 0, st>>>(b);
  RYK_CUDA(cudaGetLastError());
  return 0;
}
template <typename T>
static void slide_add(SlideBatch& b, const T* old_, const T* new_, T* dst, size_t L, size_t shift, size_t row) {
  SlideDesc& d = b.d[b.n++];
  d.old_ = old_; d.new_ = new_; d.dst = dst; d.L = L; d.shift = shift; d.row = row; d.elem = (int)sizeof(T);
}

static Session* get_session(Engine* e, int id) { return (id >= 0 && id < (int)e->sessions.size()) ? e->sessions[id] : nullptr; }

static void session_free(Session* s) {
  if (!s) return;
  for (cudaStream_t st : s->streams()) if (st) { cudaStreamSynchronize(st); cudaStreamDestroy(st); }
  if (s->sA_side) cudaStreamDestroy(s->sA_side);
  for (StepEvents& ev : s->ev)
    for (cudaEvent_t* p : ev.all()) if (*p) cudaEventDestroy(*p);
  if (s->stage_times) for (int a = 0; a < 5; ++a) for (int w = 0; w < 2; ++w) for (int i = 0; i < kRing; ++i) cudaEventDestroy(s->tev[a][w][i]);
  for (void* p : s->allocs) cudaFree(p);
  for (void* p : s->pinned) cudaFreeHost(p);
  for (DioPlan* p : s->dio) dio_plan_free(p);
  for (CrepePlan* p : s->crepe) crepe_plan_free(p);
  synth_destroy(s->synth);
  delete s;                                       // drops the stage graphs
}

static void group_free(Group* G) {
  if (!G) return;
  if (G->sG) { cudaStreamSynchronize(G->sG); cudaStreamDestroy(G->sG); }
  for (int i = 0; i < kRing; ++i) if (G->ev_fwd[i]) cudaEventDestroy(G->ev_fwd[i]);
  for (Session* m : G->members) {
    m->group = nullptr;
    for (HandoffGraphs& hg : m->hgraphs) {        // the captured stage-2 prologue / epilogue graphs point into the group's plan
      hg.s2_pro.reset();
      hg.s2_epi.reset();
    }
  }
  delete G;
}

void session_destroy_all(Engine* e) {
  for (Reblock* R : e->reblocks) reblock_free(R);
  e->reblocks.clear();
  for (Group* G : e->groups) group_free(G);
  e->groups.clear();
  for (Session* s : e->sessions) session_free(s);
  e->sessions.clear();
}

// make every session stream wait for what is already queued on the engine's main stream
int session_streams_fork(Engine* e, cudaEvent_t ev) {
  for (Session* s : e->sessions) {
    if (!s) continue;
    for (cudaStream_t st : s->streams()) RYK_CUDA(cudaStreamWaitEvent(st, ev, 0));
  }
  for (Group* G : e->groups) if (G) RYK_CUDA(cudaStreamWaitEvent(G->sG, ev, 0));
  return 0;
}
// make the engine's main stream wait for everything queued on the session streams
int session_streams_join(Engine* e) {
  for (Session* s : e->sessions) {
    if (!s) continue;
    for (cudaStream_t st : s->streams()) {
      cudaEvent_t ev;
      RYK_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
      RYK_CUDA(cudaEventRecord(ev, st));
      RYK_CUDA(cudaStreamWaitEvent(e->stream, ev, 0));
      RYK_CUDA(cudaEventDestroy(ev));
    }
  }
  for (Group* G : e->groups) {
    if (!G) continue;
    cudaEvent_t ev;
    RYK_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    RYK_CUDA(cudaEventRecord(ev, G->sG));
    RYK_CUDA(cudaStreamWaitEvent(e->stream, ev, 0));
    RYK_CUDA(cudaEventDestroy(ev));
  }
  return 0;
}

// ---- CUDA-graph cache ---------------------------------------------------------------------------------
// Every stage of a step is a fixed kernel sequence over fixed buffers (selected by chunk parity, and for stage 1 by the
// padded effective length), so each variant is stream-captured once and replayed: a step costs ~6 graph launches on
// the host instead of ~90 kernel launches (the host was the bottleneck at 0.75 ms of launch overhead per 0.78 ms step).

// Kernel nodes of a graph, or -1 on a CUDA error.  cuFFT's kernels and cluster and programmatic launches are kernel nodes; memset and
// memcpy nodes are not.  A conditional node is not either: its bodies are counted on their own (stage1_build_switch).
static int graph_kernels(cudaGraph_t graph) {
  size_t n = 0;
  RYK_CUDA(cudaGraphGetNodes(graph, nullptr, &n));
  std::vector<cudaGraphNode_t> nodes(n);
  RYK_CUDA(cudaGraphGetNodes(graph, nodes.data(), &n));
  int kernels = 0;
  for (cudaGraphNode_t node : nodes) {
    cudaGraphNodeType type;
    if (cudaGraphNodeGetType(node, &type) != cudaSuccess) {
      // the CUDA 12.9 runtime under a 13.0 driver cannot name a conditional node's type (cudaErrorUnknown); kernel nodes always resolve.
      // Clear the error so that no later cudaGetLastError reports it.
      (void)cudaGetLastError();
      continue;
    }
    kernels += type == cudaGraphNodeTypeKernel;
  }
  return kernels;
}

// instantiate graph into g, count its kernels, destroy graph
static int stage_graph_init(StageGraph& g, cudaGraph_t graph) {
  const int kernels = graph_kernels(graph);
  if (kernels < 0) return -1;
  RYK_CUDA(cudaGraphInstantiate(&g.exec, graph, 0));
  RYK_CUDA(cudaGraphDestroy(graph));
  g.launches = kernels;
  return 0;
}

// every launch of a stage graph adds its kernel nodes to e->launches
static int stage_graph_launch(Engine* e, const StageGraph& g, cudaStream_t st) {
  RYK_CUDA(cudaGraphLaunch(g.exec, st));
  e->launches += g.launches;
  return 0;
}

// capture body() on stream st into g
template <typename F>
static int capture_graph(StageGraph& g, cudaStream_t st, F&& body) {
  cudaGraph_t graph = nullptr;
  RYK_CUDA(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
  int rc = body();
  cudaError_t err = cudaStreamEndCapture(st, &graph);
  if (rc) return rc;
  RYK_CUDA(err);
  return stage_graph_init(g, graph);
}

// run_graph captures body() on stream st into g on first use and replays g.
template <typename F>
static int run_graph(Engine* e, StageGraph& g, cudaStream_t st, F&& body) {
  if (!g.exec && capture_graph(g, st, body)) return -1;
  return stage_graph_launch(e, g, st);
}

// The same for a graph of step k that has a copy per hand-off slot (member `which` of s->hgraphs[k % 6]; body(h) enqueues the copy of
// slot h).  The first step of a parity captures the copies of all three slots and uploads the two it does not launch, so the steps
// after the first two pay for no capture or upload, as with the graphs kept per parity.
template <typename F>
static int run_handoff_graph(Engine* e, Session* s, long long k, StageGraph HandoffGraphs::*which, cudaStream_t st, F&& body) {
  StageGraph& g = s->hgraphs[k % kHandoffGraphs].*which;
  if (!g.exec)
    for (int j = (int)(k & 1); j < kHandoffGraphs; j += 2) {
      StageGraph& gj = s->hgraphs[j].*which;
      if (gj.exec) continue;
      if (capture_graph(gj, st, [&]() -> int { return body(j % kHandoff); })) return -1;
      if (&gj != &g) RYK_CUDA(cudaGraphUpload(gj.exec, st));
    }
  return stage_graph_launch(e, g, st);
}

struct BucketKernels { int n[16]; };     // kernel nodes of each body of a stage-1 SWITCH

// value of the SWITCH node = padded effective length / 128 (count[1] / 128), 0 when no frame is effective (count[0] == 0); the kernels
// of the selected body go to the engine's device launch counter (other sessions' setters may add at the same time)
__global__ void k_set_bucket(cudaGraphConditionalHandle handle, const int* __restrict__ count, int n_buckets, BucketKernels kernels,
                             unsigned long long* __restrict__ launches) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    int v = count[0] > 0 ? count[1] / 128 : 0;
    if (v < 0 || v >= n_buckets) v = n_buckets - 1;        // cannot happen (count[1] <= Tw + 128); keeps the node in range
    cudaGraphSetConditional(handle, (unsigned)v);
    atomicAdd(launches, (unsigned long long)kernels.n[v]);
  }
}

static int stage1_body(Engine* e, Session* s, int b, int h, int tp1);

// Build the stage-1 graph of the chunks of step % 6 = j with a device-side switch over the padded-length buckets (CUDA conditional
// nodes, 12.8+).
static int stage1_build_switch(Engine* e, Session* s, int j) {
  const int b = j & 1, h = j % kHandoff;
  const int n_buckets = s->Tp / 128 + 1;
  RYK_CHECK(n_buckets <= 16, "window too long for the stage-1 graph table");
  cudaGraph_t graph = nullptr;
  RYK_CUDA(cudaGraphCreate(&graph, 0));
  cudaGraphConditionalHandle handle;
  RYK_CUDA(cudaGraphConditionalHandleCreate(&handle, graph, 0, cudaGraphCondAssignDefault));
  // node 1: the setter (its body table is filled in once the bodies are captured)
  cudaGraphNode_t set_node = nullptr;
  const int* cnt = s->d_count[b];
  int nb_ = n_buckets;
  BucketKernels kernels = {};
  void* args[5] = {(void*)&handle, (void*)&cnt, (void*)&nb_, (void*)&kernels, (void*)&e->d_launches};
  cudaKernelNodeParams kp = {};
  kp.func = (void*)k_set_bucket; kp.gridDim = dim3(1); kp.blockDim = dim3(32); kp.sharedMemBytes = 0; kp.kernelParams = args; kp.extra = nullptr;
  RYK_CUDA(cudaGraphAddKernelNode(&set_node, graph, nullptr, 0, &kp));
  // node 2: SWITCH
  cudaGraphNodeParams cp = {};
  cp.type = cudaGraphNodeTypeConditional;
  cp.conditional.handle = handle;
  cp.conditional.type = cudaGraphCondTypeSwitch;
  cp.conditional.size = (unsigned)n_buckets;
  cudaGraphNode_t sw = nullptr;
  RYK_CUDA(cudaGraphAddNode(&sw, graph, &set_node, 1, &cp));
  for (int i = 0; i < n_buckets; ++i) {
    cudaGraph_t body = cp.conditional.phGraph_out[i];
    RYK_CUDA(cudaStreamBeginCaptureToGraph(s->sC, body, nullptr, nullptr, 0, cudaStreamCaptureModeThreadLocal));
    int rc = stage1_body(e, s, b, h, i * 128);
    cudaGraph_t out = nullptr;
    cudaError_t err = cudaStreamEndCapture(s->sC, &out);
    if (rc) return rc;
    RYK_CUDA(err);
    kernels.n[i] = graph_kernels(body);
    if (kernels.n[i] < 0) return -1;
  }
  RYK_CUDA(cudaGraphKernelNodeSetParams(set_node, &kp));
  if (stage_graph_init(s->hgraphs[j].s1, graph)) return -1;
  RYK_CUDA(cudaGraphUpload(s->hgraphs[j].s1.exec, s->sC));     // the first step of each copy does not pay for the upload
  return 0;
}

// The head of stage 1 of a chunk of parity b: slide the feature window by the analysis outputs and run the silence gate on the
// chunk's wave window (mask / index / count[b], which only stage 1 reads).  It is all of stage 1 that the next chunks of this parity
// wait for: once it ran, their analysis may overwrite enc_*[b] and their wave slide cw_wave[g].
static int stage1_head(Engine* e, Session* s, int b) {
  const int f = b, g = b ^ 1, pe = s->e_enc_frames;
  const ryk_session_config& c = s->cfg;
  SlideBatch sb; sb.n = 0;
  slide_add<float>(sb, s->cw_f0[f], s->enc_f0[b] + pe, s->cw_f0[g], s->Tw, s->n_feat, 1);
  slide_add<float>(sb, s->cw_ap[f], s->enc_ap[b] + (size_t)pe * s->nb, s->cw_ap[g], s->Tw, s->n_feat, s->nb);
  slide_add<float>(sb, s->cw_mc[f], s->enc_mc[b] + (size_t)pe * s->C, s->cw_mc[g], s->Tw, s->n_feat, s->C);
  slide_add<uint8_t>(sb, s->cw_voiced[f], s->enc_voiced[b] + pe, s->cw_voiced[g], s->Tw, s->n_feat, 1);
  if (slide_batch(sb, s->sC)) return -1;
  if (gate_mask_run(e, s->cw_wave[g], s->Tw * s->hop, c.fft_length, s->hop, c.threshold_db, s->Tw, s->d_mse, s->d_mask[b], s->d_index[b],
                    s->d_count[b], s->sC)) return -1;
  // the chunk's own frames: over a stream they tile the input, every 5 ms frame exactly once
  if (s->f0_measure && f0_measure_run(s->enc_f0[b] + pe, s->enc_voiced[b] + pe, s->n_feat, s->d_f0_stats, s->d_f0_map, s->sC)) return -1;
  return 0;
}

// In front of stage 1 of step k on stream C: restart the speaker statistics and copy the f0 map into the block the stage-1 graphs read,
// when either was asked for since the previous step.  Stage 1 of every step runs on stream C in step order, so the steps already
// submitted keep the map they were submitted with and step k is the first to see the new one; the host does not wait and no kernel runs.
// The copy reads pinned slot k % kRing when the stream reaches it; that slot was last used by step k - kRing, whose copy ended before
// the head of its stage 1 did (the wait returns at once unless the host is a whole ring ahead of the device).
static int f0_map_sync(Session* s, long long k) {
  if (s->f0_reset) {
    RYK_CUDA(cudaMemsetAsync(s->d_f0_stats, 0, sizeof(F0Stats), s->sC));
    s->f0_reset = false;
  }
  if (!s->f0_dirty) return 0;
  const int r = (int)(k % kRing);
  if (k >= kRing) RYK_CUDA(cudaEventSynchronize(s->ev[r].cslide));
  s->h_f0_map[r] = s->f0_map;
  RYK_CUDA(cudaMemcpyAsync(s->d_f0_map, s->h_f0_map + r, sizeof(F0Map), cudaMemcpyHostToDevice, s->sC));
  s->f0_dirty = false;
  return 0;
}

// The rest of stage 1 of a chunk of parity b and hand-off slot h: (gather ->) 1-D U-Net at padded length tp1 (0: no effective frame,
// voice_changer.py:32-35 skips the net) -> scatter into the silent template + f0 map, mc2sp.  Enqueued on stream C while it is captured
// as one body of the chunk's SWITCH graph; every body is captured when the session is created so that no chunk ever pays for a capture
// in the middle of a stream.
static int stage1_body(Engine* e, Session* s, int b, int h, int tp1) {
  const int g = b ^ 1;
  const ryk_session_config& c = s->cfg;
  const float* d_y = nullptr;
  if (tp1 > 0) {
    UNetPlan* p1 = nullptr;
    if (unet_get_plan(e, s->voice->stage1, 1, 1, tp1, e->precision, &p1, s->s1_owner)) return -1;
    if (stage1_prologue_run(s->voice, s->cw_mc[g], s->d_index[b], s->d_count[b], s->C, (float*)p1->d_in, tp1, s->sC)) return -1;
    if (unet_forward(e, p1, s->sC)) return -1;
    d_y = (const float*)p1->d_out;
  }
  if (stage1_epilogue_run(s->voice, d_y, s->d_index[b], s->d_mask[b], s->d_count[b], s->Tw, s->C, s->cw_f0[g], s->cw_ap[g], s->cw_voiced[g], s->nb,
                          kSilentMc0, s->cv_mc_out[h], s->cv_f0_out[h], s->cv_ap_out[h], s->cv_voiced_out[h], s->d_f0_map, s->sC)) return -1;
  return mc2sp_run(e, s->sptk.d_H, s->cv_mc_out[h], s->Tw, c.order, c.fft_length, 1e-16, s->cv_sp_mid[h], nullptr, s->sC);
}

// Step k = s->step is enqueued in three parts so that a group can interleave its members:
//   front: streams E and C (analysis, gate, stage 1, mc2sp) and the stage-2 prologue
//   mid:   the stage-2 U-Net forward (single session: on its own stream C2; group: one batched forward on the group stream)
//   back:  stage-2 epilogue and stream D (synthesizer); results land in s->d_out_fixed[b] / s->d_n_fixed[b]; s->step advances.
// In each part b = k & 1 selects the inter-stage buffer set; the sliding windows are read from [f] = [b] and written to [g] = [b ^ 1];
// h = k % 3 is the hand-off slot, hgraphs[k % 6] the graphs that touch it, and r = k % kRing the event slot.

// stage 2 of a single session alternates its stream (and plan) by chunk parity; a group member always uses the first stream
static cudaStream_t s2_stream(const Session* s, int b) { return s->sC2s[s->group ? 0 : b]; }
// The decode slide reads only the chunk's frames [e_conv, e_conv + n_feat) of the converted window, so stage 2 computes only the
// decoder rows those frames depend on; the prologue pads rows [Tw, Tp) with one row, so the encoder computes one copy of the rows
// that depend only on it.
static int s2_plan(Engine* e, const Session* s, int b, UNetPlan** p2) {
  return unet_get_plan(e, s->voice->stage2, 1, s->Tp, 512, e->precision, p2, s->s2_owner[b], s->e_conv, s->n_feat, false, s->Tw);
}

// begin (which = 0) / end (1) of a stage in the RYK_STAGE_TIMES timeline
static int stage_time(Session* s, int stage, int which, int r, cudaStream_t st) {
  if (s->stage_times) RYK_CUDA(cudaEventRecord(s->tev[stage][which][r], st));
  return 0;
}

static int session_front(Engine* e, Session* s, const float* d_chunk_user) {
  const long long k = s->step;
  const int b = (int)(k & 1), f = b, g = b ^ 1, r = (int)(k % kRing);
  const ryk_session_config& c = s->cfg;
  const int pe = s->e_enc_frames;
  cudaStream_t sC2 = s2_stream(s, b);
  float* d_colmin = s->d_colmin[s->group ? 0 : b];
  ParityGraphs& pg = s->graphs[b];

  // ================= stream E: wave slides =================
  RYK_CUDA(cudaMemcpyAsync(s->d_chunk_fixed, d_chunk_user, sizeof(float) * s->n_in, cudaMemcpyDeviceToDevice, s->sE));
  if (k >= 2) {
    RYK_CUDA(cudaStreamWaitEvent(s->sE, s->ev[(k - 2) % kRing].cslide, 0));  // cw_wave[g]: last read by the silence gate in the head of stage 1 of k-2
    RYK_CUDA(cudaStreamWaitEvent(s->sE, s->ev[(k - 2) % kRing].enc, 0));     // wave_win[g]: last read by the analysis of k-2
  }
  if (stage_time(s, 0, 0, r, s->sE)) return -1;
  if (run_graph(e, pg.gate, s->sE, [&]() -> int {
        const float* chunk = s->d_chunk_fixed;
        if (s->in.rate) {            // device rate -> fs in front of the wave slide
          if (slide<float>(s->in_win[f], s->d_chunk_fixed, s->in_win[g], s->in.hist, s->n_in, 1, s->sE)) return -1;
          if (resample_stream_in_run(e, s->in_win[g], s->in.hist, s->n_in, s->delay_in, s->in.up, s->in.down, s->in.d_h, s->in.n_taps,
                                     s->in.d_st + f, s->in.d_st + g, s->d_chunk_model, s->n_wave, s->sE)) return -1;
          chunk = s->d_chunk_model;
        }
        if (slide<float>(s->wave_win[f], chunk, s->wave_win[g], s->Lw, s->n_wave, 1, s->sE)) return -1;
        return slide<float>(s->cw_wave[f], s->wave_win[g] + (size_t)pe * s->hop, s->cw_wave[g], (size_t)s->Tw * s->hop, (size_t)s->n_feat * s->hop, 1, s->sE);
      })) return -1;
  if (stage_time(s, 0, 1, r, s->sE)) return -1;
  RYK_CUDA(cudaEventRecord(s->ev[r].gate, s->sE));

  // ================= stream A[b]: WORLD analysis (the chunks of one parity share a plan and a stream) =================
  cudaStream_t sA = s->sA[b];
  RYK_CUDA(cudaStreamWaitEvent(sA, s->ev[r].gate, 0));
  if (k >= 2) RYK_CUDA(cudaStreamWaitEvent(sA, s->ev[(k - 2) % kRing].cslide, 0));   // enc_*[b] consumed by stage 1 of k-2
  if (stage_time(s, 1, 0, r, sA)) return -1;
  if (run_graph(e, pg.analysis, sA, [&]() -> int {
        const double* d_f0 = nullptr;
        if (s->crepe[b]) {
          if (crepe_plan_run(e, s->crepe[b], s->wave_win[g], sA)) return -1;
          d_f0 = crepe_plan_f0(s->crepe[b]);
        } else {
          if (dio_stonemask_run(e, s->dio[b], s->wave_win[g], sA)) return -1;
          d_f0 = dio_plan_f0(s->dio[b]);
        }
        const int n_enc = s->Lw / s->hop;
        return spectral_analysis_run(e, s->wave_win[g], s->Lw, c.fs, c.frame_period_ms, d_f0, n_enc, c.fft_length, c.order, s->sptk.d_G,
                                     s->enc_sp[b], s->enc_ap[b], s->enc_mc[b], s->enc_f0[b], s->enc_voiced[b], sA, s->sA_side);
      })) return -1;
  if (stage_time(s, 1, 1, r, sA)) return -1;
  RYK_CUDA(cudaEventRecord(s->ev[r].enc, sA));

  // ================= stream C: stage 1 (head: feature slides + silence gate; then U-Net, f0 map, mc2sp) =================
  // mask / index / count[b] are written by the head and read by the SWITCH graph, both on stream C: no guard between steps needed
  // (nor for the f0 map: the host's copy, the measuring kernel in the head and the epilogue in the SWITCH graph are all on stream C;
  // the copy goes before the head so that it cannot overwrite what this step's measurement writes in follow mode)
  if (f0_map_sync(s, k)) return -1;
  RYK_CUDA(cudaStreamWaitEvent(s->sC, s->ev[r].enc, 0));                       // (the analysis of step r waited for its wave slides)
  if (stage_time(s, 2, 0, r, s->sC)) return -1;
  if (run_graph(e, pg.s1_head, s->sC, [&]() -> int { return stage1_head(e, s, b); })) return -1;
  // the next chunks of this parity wait only for the head, so stage 1's U-Net is off the gate -> analysis -> stage 1 recurrence
  RYK_CUDA(cudaEventRecord(s->ev[r].cslide, s->sC));
  // three hand-off slots: stage 1 rewrites what step k-3 handed on, so it runs beside stage 2 of k-2 (and k-1)
  if (k >= kHandoff) {
    RYK_CUDA(cudaStreamWaitEvent(s->sC, s->ev[(k - 3) % kRing].dslide, 0));   // cv_{f0,ap}_out[h] consumed by decode k-3
    RYK_CUDA(cudaStreamWaitEvent(s->sC, s->ev[(k - 3) % kRing].conv, 0));     // cv_sp_mid[h] consumed by stage 2 of k-3
  }
  if (stage_graph_launch(e, s->hgraphs[k % kHandoffGraphs].s1, s->sC)) return -1;   // counts the setter; k_set_bucket counts the body
  if (stage_time(s, 2, 1, r, s->sC)) return -1;
  RYK_CUDA(cudaEventRecord(s->ev[r].s1, s->sC));

  // ================= stream C2: stage-2 prologue =================
  RYK_CUDA(cudaStreamWaitEvent(sC2, s->ev[r].s1, 0));
  if (k >= kHandoff) RYK_CUDA(cudaStreamWaitEvent(sC2, s->ev[(k - 3) % kRing].dslide, 0));  // cv_sp_out[h] consumed by decode k-3
  if (stage_time(s, 3, 0, r, sC2)) return -1;
  if (s->group) {
    Group* G = s->group;
    if (G->step >= 1) RYK_CUDA(cudaStreamWaitEvent(sC2, G->ev_fwd[(G->step - 1) % kRing], 0));   // batched input read by forward k-1
    float* dst = (float*)G->p2->d_in + (size_t)s->slot * s->Tp * 512;
    if (run_handoff_graph(e, s, k, &HandoffGraphs::s2_pro, sC2, [&](int h) -> int {
          return sr_prologue_run(e, s->cv_sp_mid[h], s->Tw, s->Tp, s->nb, dst, sC2, d_colmin);
        })) return -1;
    RYK_CUDA(cudaEventRecord(s->ev[r].pro, sC2));
  } else {
    UNetPlan* p2 = nullptr;
    if (s2_plan(e, s, b, &p2)) return -1;
    if (run_handoff_graph(e, s, k, &HandoffGraphs::s2_pro, sC2, [&](int h) -> int {
          if (sr_prologue_run(e, s->cv_sp_mid[h], s->Tw, s->Tp, s->nb, (float*)p2->d_in, sC2, d_colmin)) return -1;
          return unet_forward(e, p2, sC2, 0, 0);
        })) return -1;
  }
  return 0;
}

// single session: stage-2 layers 1..14 (the wgmma layers) on the session's own stream
static int session_mid_single(Engine* e, Session* s) {
  const int b = (int)(s->step & 1);
  cudaStream_t sC2 = s2_stream(s, b);
  UNetPlan* p2 = nullptr;
  if (s2_plan(e, s, b, &p2)) return -1;
  cudaEvent_t pe0 = nullptr, pe1 = nullptr;
  if (e->profile) { RYK_CUDA(cudaEventCreate(&pe0)); RYK_CUDA(cudaEventCreate(&pe1)); RYK_CUDA(cudaEventRecord(pe0, sC2)); }
  if (run_graph(e, s->graphs[b].s2_layers, sC2, [&]() -> int { return unet_forward(e, p2, sC2, 1, 14); })) return -1;
  if (e->profile) { RYK_CUDA(cudaEventRecord(pe1, sC2)); e->prof_events.emplace_back(pe0, pe1); }
  return 0;
}

static int session_back(Engine* e, Session* s) {
  const long long k = s->step;
  const int b = (int)(k & 1), f = b, g = b ^ 1, r = (int)(k % kRing);
  const ryk_session_config& c = s->cfg;
  const int pc = s->e_conv;
  cudaStream_t sC2 = s2_stream(s, b);
  ParityGraphs& pg = s->graphs[b];
  if (s->group) {
    Group* G = s->group;
    RYK_CUDA(cudaStreamWaitEvent(sC2, G->ev_fwd[G->step % kRing], 0));
    const float* src = (const float*)G->p2->d_out + (size_t)s->slot * s->Tp * 512;
    if (run_handoff_graph(e, s, k, &HandoffGraphs::s2_epi, sC2, [&](int h) -> int {
          return sr_epilogue_run(e, src, s->Tw, s->nb, s->cv_sp_out[h], sC2, pc, pc + s->n_feat);
        })) return -1;
  } else {
    UNetPlan* p2 = nullptr;
    if (s2_plan(e, s, b, &p2)) return -1;
    if (run_handoff_graph(e, s, k, &HandoffGraphs::s2_epi, sC2, [&](int h) -> int {
          if (unet_forward(e, p2, sC2, 15, 15)) return -1;
          return sr_epilogue_run(e, (const float*)p2->d_out, s->Tw, s->nb, s->cv_sp_out[h], sC2, pc, pc + s->n_feat);
        })) return -1;
  }
  if (stage_time(s, 3, 1, r, sC2)) return -1;
  RYK_CUDA(cudaEventRecord(s->ev[r].conv, sC2));

  // ================= stream D: realtime synthesizer =================
  RYK_CUDA(cudaStreamWaitEvent(s->sD, s->ev[r].conv, 0));
  if (stage_time(s, 4, 0, r, s->sD)) return -1;
  if (synth_host_advance(e, s->synth, s->Td, s->sD)) return -1;
  const int max_blocks = s->max_blocks;
  if (run_handoff_graph(e, s, k, &HandoffGraphs::dec_slide, s->sD, [&](int h) -> int {
        SlideBatch sb; sb.n = 0;
        slide_add<float>(sb, s->dw_f0[f], s->cv_f0_out[h] + pc, s->dw_f0[g], s->Td, s->n_feat, 1);
        slide_add<float>(sb, s->dw_ap[f], s->cv_ap_out[h] + (size_t)pc * s->nb, s->dw_ap[g], s->Td, s->n_feat, s->nb);
        slide_add<float>(sb, s->dw_sp[f], s->cv_sp_out[h] + (size_t)pc * s->nb, s->dw_sp[g], s->Td, s->n_feat, s->nb);
        if (slide_batch(sb, s->sD)) return -1;
        k_f32_to_f64<<<(s->Td + 127) / 128, 128, 0, s->sD>>>(s->dw_f0[g], s->dec_f0_f64, s->Td);
        RYK_CUDA(cudaGetLastError());
        return 0;
      })) return -1;
  // the converted features of this hand-off slot are free again as soon as they sit in the decode window
  RYK_CUDA(cudaEventRecord(s->ev[r].dslide, s->sD));
  if (run_graph(e, pg.synth, s->sD, [&]() -> int {
        if (synth_add_kernel(e, s->synth, s->dec_f0_f64, s->Td, s->dw_sp[g], s->dw_ap[g], s->sD)) return -1;
        if (synth_drain_async(e, s->synth, s->d_out_fixed[b], max_blocks, s->sD)) return -1;
        k_scrub<<<8, 256, 0, s->sD>>>(s->d_out_fixed[b], s->synth->dev.state, c.vocoder_buffer_size, max_blocks * c.vocoder_buffer_size, s->d_n_fixed[b]);
        RYK_CUDA(cudaGetLastError());
        if (!s->out.rate) return 0;
        // fs -> device rate: the outputs whose filter support the synthesizer has produced; the rest waits for the next step
        return resample_stream_out_run(e, s->out_hist[f], s->out_hist[g], s->out.hist, s->d_out_fixed[b], s->d_n_fixed[b], s->out.up, s->out.down,
                                       s->out.d_h, s->out.n_taps, s->out.d_st + f, s->out.d_st + g, s->d_rout_fixed[b], s->max_out,
                                       s->d_rn_fixed[b], s->sD);
      })) return -1;
  if (stage_time(s, 4, 1, r, s->sD)) return -1;
  // ev[r].dec is recorded by stage_out after the copies it appends to stream D
  s->step++;
  return 0;
}

static int session_enqueue(Engine* e, Session* s, const float* d_chunk_user) {
  int rc = session_front(e, s, d_chunk_user);
  if (!rc) rc = session_mid_single(e, s);
  if (!rc) rc = session_back(e, s);
  return rc;
}

// One step of every member + the batched stage-2 forward between their front and back halves.
static int group_enqueue(Engine* e, Group* G, const float* const* d_chunks) {
  const int r = (int)(G->step % kRing);
  for (size_t i = 0; i < G->members.size(); ++i)
    if (session_front(e, G->members[i], d_chunks[i])) return -1;
  for (Session* m : G->members) {
    RYK_CUDA(cudaStreamWaitEvent(G->sG, m->ev[m->step % kRing].pro, 0));
    if (m->step >= 1) RYK_CUDA(cudaStreamWaitEvent(G->sG, m->ev[(m->step - 1) % kRing].conv, 0));   // batched output read by epilogue k-1
  }
  cudaEvent_t pe0 = nullptr, pe1 = nullptr;
  if (e->profile) { RYK_CUDA(cudaEventCreate(&pe0)); RYK_CUDA(cudaEventCreate(&pe1)); RYK_CUDA(cudaEventRecord(pe0, G->sG)); }
  if (run_graph(e, G->fwd_graph, G->sG, [&]() -> int { return unet_forward(e, G->p2, G->sG, 0, 15); })) return -1;
  if (e->profile) { RYK_CUDA(cudaEventRecord(pe1, G->sG)); e->prof_events.emplace_back(pe0, pe1); }
  RYK_CUDA(cudaEventRecord(G->ev_fwd[r], G->sG));
  for (Session* m : G->members)
    if (session_back(e, m)) return -1;
  G->step++;
  return 0;
}

// ---- host-API staging shared by sessions and groups (ring slot r = step % kRing) ----
// host chunk -> pinned slot -> s->d_chunk[r] on stream E
static int stage_in(Session* s, int r, const float* wave) {
  memcpy(s->h_in[r], wave, sizeof(float) * s->n_in);
  RYK_CUDA(cudaMemcpyAsync(s->d_chunk[r], s->h_in[r], sizeof(float) * s->n_in, cudaMemcpyHostToDevice, s->sE));
  return 0;
}

// the samples a step of parity b returns and their count: the synthesizer's blocks, or their device-rate resampling
static double* step_out(Session* s, int b) { return s->out.rate ? s->d_rout_fixed[b] : s->d_out_fixed[b]; }
static int* step_n_out(Session* s, int b) { return s->out.rate ? s->d_rn_fixed[b] : s->d_n_fixed[b]; }

// after a step of s was enqueued: copy its samples and sample count to out / n_out (kind: to the host ring or to device buffers) behind
// the decode stream and record ev[r].dec.  r is the caller's ring slot (the session's step, or the group's step for a member); the
// output buffers are those of the parity of the session's own step, which differs from the group's for a member that joined at a
// group step of the other parity.
static int stage_out(Session* s, int r, double* out, int* n_out, cudaMemcpyKind kind) {
  const int b = (int)((s->step - 1) & 1);
  RYK_CUDA(cudaMemcpyAsync(n_out, step_n_out(s, b), sizeof(int), kind, s->sD));
  RYK_CUDA(cudaMemcpyAsync(out, step_out(s, b), sizeof(double) * s->max_out, kind, s->sD));
  RYK_CUDA(cudaEventRecord(s->ev[r].dec, s->sD));
  return 0;
}

// wait for step `ticket` of s and copy its samples out of the host ring
static int collect_out(Session* s, long long ticket, double* out, int out_capacity, int* n_out) {
  const int r = (int)(ticket % kRing);
  RYK_CUDA(cudaEventSynchronize(s->ev[r].dec));
  const int produced = *s->h_n[r];
  RYK_CHECK(produced <= out_capacity, "output buffer too small for the produced blocks");
  memcpy(out, s->h_out[r], sizeof(double) * produced);
  *n_out = produced;
  s->collected++;
  return 0;
}

}  // namespace ryk

using namespace ryk;
struct ryk_engine { Engine impl; };

extern "C" {

static int session_build(Engine* e, Session* s, const ryk_session_config* cfg);

int ryk_session_create_voice(ryk_engine* h, const ryk_session_config* cfg, int voice_id, int* session_id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(cfg && session_id, "null argument");
  Voice* v = engine_voice(e, voice_id);
  RYK_CHECK(v != nullptr, "no such voice");
  RYK_CHECK(v->stage1 && v->stage2, "load both models before creating a session");
  if (voice_id >= 1) {
    RYK_CHECK(voice_models_loaded(v), "load every layer of both of the voice's models before creating a session on it");
    if (voice_default_stage1_stats(v, v->stage1->in_ch)) return -1;
  }
  Session* s = new Session();
  s->voice = v; s->voice_id = voice_id;
  if (session_build(e, s, cfg)) {
    // free whatever the build made (buffers, analysis / CREPE plans, graphs, U-Net plans); ryk_last_error keeps the cause
    const int s1_owner = s->s1_owner, s2_owner[2] = {s->s2_owner[0], s->s2_owner[1]};
    session_free(s);
    if (s1_owner) unet_release_owner(v->stage1, s1_owner);
    for (int owner : s2_owner) if (owner) unet_release_owner(v->stage2, owner);
    return -1;
  }
  v->users++;
  e->sessions.push_back(s);
  *session_id = (int)e->sessions.size() - 1;
  return 0;
}

int ryk_session_create(ryk_engine* h, const ryk_session_config* cfg, int* session_id) { return ryk_session_create_voice(h, cfg, 0, session_id); }

int ryk_session_voice(ryk_engine* h, int id) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  return s->voice_id;
}

// Everything a session allocates and captures; on failure the caller frees the partly built session.
static int session_build(Engine* e, Session* s, const ryk_session_config* cfg) {
  s->cfg = *cfg;
  s->hop = (int)(cfg->fs * cfg->frame_period_ms / 1000.0);
  s->rate = (int)lround(1000.0 / cfg->frame_period_ms);
  s->n_wave = (int)lrint(cfg->buffer_time * cfg->fs);
  s->n_feat = (int)lrint(cfg->buffer_time * s->rate);
  s->e_wave = (int)lrint(cfg->encode_extra_time * cfg->fs);
  s->e_enc_frames = (int)lrint(cfg->encode_extra_time * s->rate);
  s->e_conv = (int)lrint(cfg->convert_extra_time * s->rate);
  s->e_dec = (int)lrint(cfg->decode_extra_time * s->rate);
  s->Lw = s->n_wave + 2 * s->e_wave;
  s->Tw = s->n_feat + 2 * s->e_conv;
  s->Td = s->n_feat + 2 * s->e_dec;
  s->Tp = s->Tw + (128 - s->Tw % 128);
  s->nb = cfg->fft_length / 2 + 1;
  s->C = cfg->order + 1;
  RYK_CHECK(s->n_wave == s->n_feat * s->hop && s->e_wave == s->e_enc_frames * s->hop, "buffer_time / encode_extra_time must be whole frames");
  RYK_CHECK(s->Lw / s->hop - 2 * s->e_enc_frames == s->n_feat, "encode window does not trim to one chunk of frames");
  RYK_CHECK(s->nb == 513 && s->voice->stage1->in_ch == s->C, "session configuration does not match the loaded models");
  // the synthesizer's spectra are cheaptrick_fft_size(fs) / 2 + 1 bins wide and read rows of the fft_length / 2 + 1 bin decode window
  RYK_CHECK(cheaptrick_fft_size(cfg->fs, 71.0) / 2 + 1 == s->nb,
            "fs does not match fft_length: the synthesizer at this fs needs a different spectrum width (run the session at the model's "
            "rate and set a device rate with ryk_session_set_input_rate / ryk_session_set_output_rate)");
  s->n_in = s->n_wave;
  if (sptk_prepare(e, cfg->order, cfg->alpha, cfg->fft_length, &s->sptk)) return -1;
  // The analysis, stage-1 and synthesis stages are chains of small, latency-bound kernels; stage 2 is bulk work that fills
  // every SM.  Higher stream priority for the former lets their CTAs take freed SM slots first, so their latency does not
  // inflate behind stage-2 waves.
  int prio_lo = 0, prio_hi = 0;
  RYK_CUDA(cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi));      // lo = least (numerically largest), hi = greatest
  RYK_CUDA(cudaStreamCreateWithPriority(&s->sE, cudaStreamNonBlocking, prio_hi));
  for (int i = 0; i < 2; ++i) RYK_CUDA(cudaStreamCreateWithPriority(&s->sA[i], cudaStreamNonBlocking, prio_hi));
  RYK_CUDA(cudaStreamCreateWithPriority(&s->sA_side, cudaStreamNonBlocking, prio_hi));
  RYK_CUDA(cudaStreamCreateWithPriority(&s->sC, cudaStreamNonBlocking, prio_hi));
  for (int i = 0; i < 2; ++i) RYK_CUDA(cudaStreamCreateWithPriority(&s->sC2s[i], cudaStreamNonBlocking, prio_lo));
  RYK_CUDA(cudaStreamCreateWithPriority(&s->sD, cudaStreamNonBlocking, prio_hi));
  for (StepEvents& ev : s->ev)
    for (cudaEvent_t* p : ev.all()) RYK_CUDA(cudaEventCreateWithFlags(p, cudaEventDisableTiming));
  { const char* v = getenv("RYK_STAGE_TIMES"); s->stage_times = v && atoi(v) != 0; }
  if (s->stage_times) for (int a = 0; a < 5; ++a) for (int w = 0; w < 2; ++w) for (int i = 0; i < kRing; ++i) RYK_CUDA(cudaEventCreate(&s->tev[a][w][i]));
  // zero-fill on the ENGINE stream: the template fill below (k_fill_rows on e->stream, a non-blocking stream) must be ordered after
  // it -- a legacy-default-stream cudaMemset is not, and could land after the fill (seen once as a 4e-3 RMSE mismatch)
  auto A = [&](void** p, size_t bytes) -> int { RYK_CUDA(cudaMalloc(p, bytes ? bytes : 16)); RYK_CUDA(cudaMemsetAsync(*p, 0, bytes ? bytes : 16, e->stream)); s->allocs.push_back(*p); return 0; };
  auto P = [&](void** p, size_t bytes) -> int { RYK_CUDA(cudaMallocHost(p, bytes ? bytes : 16)); memset(*p, 0, bytes ? bytes : 16); s->pinned.push_back(*p); return 0; };
  const int n_enc = s->Lw / s->hop;
  for (int i = 0; i < 2; ++i) {
    if (A((void**)&s->wave_win[i], sizeof(float) * s->Lw)) return -1;
    if (A((void**)&s->cw_f0[i], sizeof(float) * s->Tw)) return -1;
    if (A((void**)&s->cw_ap[i], sizeof(float) * (size_t)s->Tw * s->nb)) return -1;
    if (A((void**)&s->cw_mc[i], sizeof(float) * (size_t)s->Tw * s->C)) return -1;
    if (A((void**)&s->cw_voiced[i], (size_t)s->Tw)) return -1;
    if (A((void**)&s->cw_wave[i], sizeof(float) * (size_t)s->Tw * s->hop)) return -1;
    if (A((void**)&s->dw_f0[i], sizeof(float) * s->Td)) return -1;
    if (A((void**)&s->dw_ap[i], sizeof(float) * (size_t)s->Td * s->nb)) return -1;
    if (A((void**)&s->dw_sp[i], sizeof(float) * (size_t)s->Td * s->nb)) return -1;
    // silent template mel-cepstrum in the not-yet-filled part of the convert window
    k_fill_rows<float><<<64, 256, 0, e->stream>>>(s->cw_mc[i], s->Tw, s->C, kSilentMc0, 0.f);
    if (A((void**)&s->enc_f0[i], sizeof(float) * n_enc)) return -1;
    if (A((void**)&s->enc_sp[i], sizeof(float) * (size_t)n_enc * s->nb)) return -1;
    if (A((void**)&s->enc_ap[i], sizeof(float) * (size_t)n_enc * s->nb)) return -1;
    if (A((void**)&s->enc_mc[i], sizeof(float) * (size_t)n_enc * s->C)) return -1;
    if (A((void**)&s->enc_voiced[i], (size_t)n_enc)) return -1;
    if (A((void**)&s->d_mask[i], (size_t)s->Tw)) return -1;
    if (A((void**)&s->d_index[i], sizeof(int) * s->Tw)) return -1;
    if (A((void**)&s->d_count[i], sizeof(int) * 2)) return -1;
  }
  for (int i = 0; i < kHandoff; ++i) {
    if (A((void**)&s->cv_mc_out[i], sizeof(float) * (size_t)s->Tw * s->C)) return -1;
    if (A((void**)&s->cv_f0_out[i], sizeof(float) * s->Tw)) return -1;
    if (A((void**)&s->cv_ap_out[i], sizeof(float) * (size_t)s->Tw * s->nb)) return -1;
    if (A((void**)&s->cv_sp_out[i], sizeof(float) * (size_t)s->Tw * s->nb)) return -1;
    if (A((void**)&s->cv_voiced_out[i], (size_t)s->Tw)) return -1;
    if (A((void**)&s->cv_sp_mid[i], sizeof(float) * (size_t)s->Tw * s->nb)) return -1;
  }
  if (A((void**)&s->d_mse, sizeof(double) * s->Tw)) return -1;
  for (int i = 0; i < 2; ++i) if (A((void**)&s->d_colmin[i], sizeof(float) * kColminFloats)) return -1;
  if (A((void**)&s->dec_f0_f64, sizeof(double) * s->Td)) return -1;
  if (A((void**)&s->d_chunk_fixed, sizeof(float) * s->n_wave)) return -1;
  // the session starts on its voice's f0 map
  if (A((void**)&s->d_f0_map, sizeof(F0Map))) return -1;
  if (A((void**)&s->d_f0_stats, sizeof(F0Stats))) return -1;
  if (P((void**)&s->h_f0_map, sizeof(F0Map) * kRing)) return -1;
  s->f0_map = s->h_f0_map[0] = voice_f0_map(s->voice);
  RYK_CUDA(cudaMemcpyAsync(s->d_f0_map, s->h_f0_map, sizeof(F0Map), cudaMemcpyHostToDevice, e->stream));
  s->max_blocks = (s->Td * s->hop) / cfg->vocoder_buffer_size + 4;
  s->max_out = s->max_blocks * cfg->vocoder_buffer_size;
  const size_t out_samples = (size_t)s->max_out;
  for (int i = 0; i < 2; ++i) {
    if (A((void**)&s->d_out_fixed[i], sizeof(double) * out_samples)) return -1;
    if (A((void**)&s->d_n_fixed[i], sizeof(int))) return -1;
  }
  for (int i = 0; i < kRing; ++i) {
    if (A((void**)&s->d_chunk[i], sizeof(float) * s->n_wave)) return -1;
    if (A((void**)&s->d_out[i], sizeof(double) * out_samples)) return -1;
    if (A((void**)&s->d_n_out[i], sizeof(int))) return -1;
    if (P((void**)&s->h_in[i], sizeof(float) * s->n_wave)) return -1;
    if (P((void**)&s->h_out[i], sizeof(double) * out_samples)) return -1;
    if (P((void**)&s->h_n[i], sizeof(int))) return -1;
  }
  // f0 method 2: each step's encode window is analysed on its own, like one crepe.predict call per fetched window (DESIGN.md C3)
  for (int i = 0; i < 2; ++i) {
    const int rc = e->f0_method == 2 ? crepe_plan_create(e, s->Lw, cfg->fs, cfg->frame_period_ms, &s->crepe[i])
                                     : dio_plan_create(e, s->Lw, cfg->fs, cfg->frame_period_ms, cfg->f0_floor, cfg->f0_ceil, &s->dio[i], e->f0_method);
    if (rc) return -1;
  }
  if (synth_create(e, cfg->fs, cfg->frame_period_ms, cheaptrick_fft_size(cfg->fs, 71.0), cfg->vocoder_buffer_size, 4096, &s->synth)) return -1;
  // build the U-Net plans this session can need up front (allocation + tensor maps), not on the first chunk
  UNetPlan* p = nullptr;
  s->s1_owner = ++e->plan_owners;
  for (int b = 0; b < 2; ++b) s->s2_owner[b] = ++e->plan_owners;
  for (int Tp = 128; Tp <= s->Tp; Tp += 128) if (unet_get_plan(e, s->voice->stage1, 1, 1, Tp, e->precision, &p, s->s1_owner)) return -1;
  // (the stage-2 plans are created on first use: a session that joins a group never needs its own)
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  RYK_CUDA(cudaDeviceSynchronize());
  for (int j = 0; j < kHandoffGraphs; ++j) if (stage1_build_switch(e, s, j)) return -1;
  return 0;
}

int ryk_session_destroy(ryk_engine* h, int id) {
  Engine* e = &h->impl;
  Session* s = get_session(e, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(s->group == nullptr, "session belongs to a group: destroy the group first");
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  const int s1_owner = s->s1_owner, s2_owner[2] = {s->s2_owner[0], s->s2_owner[1]};
  Voice* v = s->voice;
  session_free(s);                         // synchronises the session's streams
  unet_release_owner(v->stage1, s1_owner);
  for (int owner : s2_owner) unet_release_owner(v->stage2, owner);
  v->users--;
  e->sessions[id] = nullptr;
  return 0;
}

// Queue one chunk (host samples) without waiting for its output; *ticket identifies it for ryk_session_collect.
int ryk_session_submit(ryk_engine* h, int id, const float* wave, int n, long long* ticket) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = get_session(e, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(n == s->n_in, "chunk length must be round(rate * buffer_time) at the session's input rate");
  RYK_CHECK(s->group == nullptr, "session belongs to a group: use ryk_group_submit");
  RYK_CHECK(s->step - s->collected < kRing - 2, "too many chunks in flight: collect before submitting more");
  const long long k = s->step;
  const int r = (int)(k % kRing);
  if (stage_in(s, r, wave)) return -1;
  if (session_enqueue(e, s, s->d_chunk[r])) return -1;
  if (stage_out(s, r, s->h_out[r], s->h_n[r], cudaMemcpyDeviceToHost)) return -1;
  if (ticket) *ticket = k;
  return 0;
}

// Wait for the chunk `ticket` (tickets must be collected in order) and copy its samples out.
int ryk_session_collect(ryk_engine* h, int id, long long ticket, double* out, int out_capacity, int* n_out) {
  Engine* e = &h->impl;
  Session* s = get_session(e, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(ticket == s->collected && ticket < s->step, "tickets are collected in submission order");
  return collect_out(s, ticket, out, out_capacity, n_out);
}

// Non-blocking completion query (cudaEventQuery of the step's last decode-stream event): *done = 1 when ryk_session_collect would
// not wait.  This is what queue_output_wave.get_nowait() needs (run.py:176-182).
int ryk_session_poll(ryk_engine* h, int id, long long ticket, int* done) {
  Engine* e = &h->impl;
  Session* s = get_session(e, id);
  RYK_CHECK(s != nullptr && done != nullptr, "no such session");
  RYK_CHECK(ticket >= 0 && ticket < s->step && ticket + kRing > s->step, "ticket is not among the last 8 steps");
  cudaError_t q = cudaEventQuery(s->ev[ticket % kRing].dec);
  if (q != cudaSuccess && q != cudaErrorNotReady) RYK_CUDA(q);
  *done = q == cudaSuccess ? 1 : 0;
  return 0;
}

int ryk_session_push(ryk_engine* h, int id, const float* wave, int n, double* out, int out_capacity, int* n_out) {
  long long ticket = 0;
  if (ryk_session_submit(h, id, wave, n, &ticket)) return -1;
  return ryk_session_collect(h, id, ticket, out, out_capacity, n_out);
}

// Device-resident step, asynchronous: returns as soon as the work is queued (output valid after ryk_engine_synchronize
// or any later stream-ordered work of this session).
int ryk_session_push_device(ryk_engine* h, int id, const float* wave_dev, int n, double* out_dev, int out_capacity, int* n_out_dev) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = get_session(e, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(n == s->n_in, "chunk length must be round(rate * buffer_time) at the session's input rate");
  RYK_CHECK(s->group == nullptr, "session belongs to a group: use ryk_group_push_device");
  RYK_CHECK(out_capacity >= s->max_out, "out_capacity must hold the most samples a step returns (ryk_session_io_geometry max_out)");
  const int r = (int)(s->step % kRing);
  if (session_enqueue(e, s, wave_dev)) return -1;
  if (stage_out(s, r, out_dev, n_out_dev, cudaMemcpyDeviceToDevice)) return -1;
  s->collected = s->step;         // device-resident steps are not collected through the host API
  return 0;
}

// ---- device rates: the session takes chunks at in.rate and returns samples at out.rate, converting on its own streams ----
// A zeroed allocation owned by the session (device, or pinned host); a buffer already at *p is released first.
static int session_realloc(Session* s, void** p, size_t bytes, bool host) {
  std::vector<void*>& owned = host ? s->pinned : s->allocs;
  if (*p) {
    for (size_t i = 0; i < owned.size(); ++i) if (owned[i] == *p) { owned.erase(owned.begin() + i); break; }
    if (host) cudaFreeHost(*p); else cudaFree(*p);
    *p = nullptr;
  }
  if (host) { RYK_CUDA(cudaMallocHost(p, bytes)); memset(*p, 0, bytes); }
  else { RYK_CUDA(cudaMalloc(p, bytes)); RYK_CUDA(cudaMemset(*p, 0, bytes)); }
  owned.push_back(*p);
  return 0;
}

// Geometry (DESIGN.md §4, DECIDE R1), with half = (n_taps - 1) / 2 and up / down = the resampler's output rate / input rate:
//   input:  delay_in = half / down model samples, the smallest delay for which every sample of a step's model-rate chunk has its whole
//           filter support in the chunks received; the history window holds the chunk and the ceil((delay_in * down + half) / up)
//           samples before it.
//   output: a step emits the outputs whose support ends inside the synthesizer samples so far; the kept history covers the left
//           support of the first output not yet emitted, and max_out bounds one step's count.
static int session_set_rate(Engine* e, int id, bool input, int rate, int up, int down, const double* taps, int n_taps) {
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = get_session(e, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(s->step == 0 && s->group == nullptr, "device rates can only be set on a fresh session (no chunk pushed, not in a group)");
  Session::RateSide& side = input ? s->in : s->out;
  RYK_CHECK(side.rate == 0, "this side's device rate is already set");
  RYK_CHECK(rate > 0, "device rate must be positive");
  const int fs = s->cfg.fs;
  if (rate == fs) return 0;                         // the session's own rate: no resampler on this side
  RYK_CHECK(taps && n_taps > 0 && (n_taps & 1) && up > 0 && down > 0 && std::gcd(up, down) == 1,
            "bad resampler arguments (coprime up / down, an odd number of taps)");
  const long long r_from = input ? rate : fs, r_to = input ? fs : rate;
  RYK_CHECK(r_to * down == r_from * up, "up / down must be the resampler's output rate / input rate, reduced");
  const int half = (n_taps - 1) / 2;
  if (input) {
    const int n_in = (int)lrint(s->cfg.buffer_time * rate);
    RYK_CHECK((long long)n_in * up == (long long)s->n_wave * down,
              "the chunk at this device rate is not a whole number of samples: round(rate * buffer_time) * up != round(fs * buffer_time) * down");
    const int delay = half / down;
    side.hist = n_in + (delay * down + half + up - 1) / up;
    for (int i = 0; i < 2; ++i) if (session_realloc(s, (void**)&s->in_win[i], sizeof(float) * side.hist, false)) return -1;
    if (session_realloc(s, (void**)&s->d_chunk_model, sizeof(float) * s->n_wave, false)) return -1;
    if (session_realloc(s, (void**)&s->d_chunk_fixed, sizeof(float) * n_in, false)) return -1;
    for (int r = 0; r < kRing; ++r) {
      if (session_realloc(s, (void**)&s->d_chunk[r], sizeof(float) * n_in, false)) return -1;
      if (session_realloc(s, (void**)&s->h_in[r], sizeof(float) * n_in, true)) return -1;
    }
  } else {
    const long long blocks = (long long)s->max_blocks * s->cfg.vocoder_buffer_size;
    const int max_out = (int)((blocks * up + down - 1) / down);
    side.hist = (2 * half + down + up - 1) / up + 1;
    for (int i = 0; i < 2; ++i) {
      if (session_realloc(s, (void**)&s->out_hist[i], sizeof(double) * side.hist, false)) return -1;
      if (session_realloc(s, (void**)&s->d_rout_fixed[i], sizeof(double) * max_out, false)) return -1;
      if (session_realloc(s, (void**)&s->d_rn_fixed[i], sizeof(int), false)) return -1;
    }
    for (int r = 0; r < kRing; ++r) if (session_realloc(s, (void**)&s->h_out[r], sizeof(double) * max_out, true)) return -1;
  }
  if (session_realloc(s, (void**)&side.d_h, sizeof(double) * n_taps, false)) return -1;
  if (session_realloc(s, (void**)&side.d_st, sizeof(ResampleState) * 2, false)) return -1;
  RYK_CUDA(cudaMemcpy(side.d_h, taps, sizeof(double) * n_taps, cudaMemcpyHostToDevice));
  RYK_CUDA(cudaDeviceSynchronize());               // the zero-fills ran on the legacy default stream; the session's streams do not wait for it
  side.rate = rate; side.up = up; side.down = down; side.n_taps = n_taps;
  if (input) {
    s->n_in = (int)lrint(s->cfg.buffer_time * rate);
    s->delay_in = half / down;
  } else {
    s->max_out = (int)(((long long)s->max_blocks * s->cfg.vocoder_buffer_size * up + down - 1) / down);
  }
  return 0;
}

int ryk_session_set_input_rate(ryk_engine* h, int id, int rate, int up, int down, const double* taps, int n_taps) {
  return session_set_rate(&h->impl, id, true, rate, up, down, taps, n_taps);
}

int ryk_session_set_output_rate(ryk_engine* h, int id, int rate, int up, int down, const double* taps, int n_taps) {
  return session_set_rate(&h->impl, id, false, rate, up, down, taps, n_taps);
}

int ryk_session_io_geometry(ryk_engine* h, int id, int* n_in, int* max_out, int* delay_in, int* in_rate, int* out_rate) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  if (n_in) *n_in = s->n_in;
  if (max_out) *max_out = s->max_out;
  if (delay_in) *delay_in = s->delay_in;
  if (in_rate) *in_rate = s->in.rate ? s->in.rate : s->cfg.fs;
  if (out_rate) *out_rate = s->out.rate ? s->out.rate : s->cfg.fs;
  return 0;
}

// ---- the session's f0 map and the statistics of its speaker (DESIGN.md §4a) ----
// These calls change host state only; f0_map_sync carries it to the device at the next submitted step, alone or in a group.
int ryk_session_get_f0_map(ryk_engine* h, int id, ryk_f0_map* map) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(map != nullptr, "null argument");
  map->in_mean = s->f0_map.mu_in; map->in_std = s->f0_map.sd_in; map->target_mean = s->f0_map.mu_tgt; map->target_std = s->f0_map.sd_tgt;
  return 0;
}

int ryk_session_set_f0_map(ryk_engine* h, int id, const ryk_f0_map* map) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(map != nullptr, "null argument");
  RYK_CHECK(isfinite(map->in_mean) && isfinite(map->in_std) && isfinite(map->target_mean) && isfinite(map->target_std),
            "the f0 map must be finite");
  RYK_CHECK(map->in_std > 0 && map->target_std > 0, "the standard deviations of the f0 map must be positive");
  s->f0_map.mu_in = map->in_mean; s->f0_map.sd_in = map->in_std; s->f0_map.mu_tgt = map->target_mean; s->f0_map.sd_tgt = map->target_std;
  s->f0_map.has_stats = 1;
  s->f0_dirty = true;
  return 0;
}

int ryk_session_f0_measure(ryk_engine* h, int id, int enable) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(s->step == 0, "f0 measurement can only be switched on a fresh session (no chunk pushed): the head of stage 1 is captured at the first steps");
  RYK_CHECK(enable || !s->f0_map.follow, "the session follows its measurement: turn follow mode off first");
  s->f0_measure = enable != 0;
  return 0;
}

int ryk_session_f0_follow(ryk_engine* h, int id, int follow, int min_voiced_frames, double sd_floor) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  if (follow) {
    RYK_CHECK(s->f0_measure, "follow mode needs f0 measurement (ryk_session_f0_measure)");
    RYK_CHECK(s->f0_map.has_stats, "follow mode needs an f0 map: the voice has no f0 statistics and none were set on the session");
    RYK_CHECK(min_voiced_frames >= 1, "min_voiced_frames must be at least 1");
    RYK_CHECK(isfinite(sd_floor) && sd_floor > 0, "sd_floor must be finite and positive");
    s->f0_map.min_voiced = min_voiced_frames; s->f0_map.sd_floor = sd_floor;
  }
  s->f0_map.follow = follow != 0;
  s->f0_dirty = true;
  return 0;
}

int ryk_session_f0_measure_reset(ryk_engine* h, int id) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(s->f0_measure, "f0 measurement is not enabled for this session");
  s->f0_reset = true;
  s->f0_dirty = true;            // follow mode: back to the host's input side until min_voiced_frames are counted again
  return 0;
}

int ryk_session_f0_measured(ryk_engine* h, int id, long long* n_voiced, double* mean, double* std_) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = get_session(e, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(s->f0_measure, "f0 measurement is not enabled for this session");
  F0Stats st = {};
  if (!s->f0_reset) {             // (a reset not yet submitted already reads as empty)
    RYK_CUDA(cudaMemcpyAsync(&st, s->d_f0_stats, sizeof(st), cudaMemcpyDeviceToHost, s->sC));
    RYK_CUDA(cudaStreamSynchronize(s->sC));      // behind the head of stage 1 of every submitted step
  }
  if (n_voiced) *n_voiced = st.n;
  if (mean) *mean = st.mean;
  if (std_) *std_ = st.n >= 2 ? sqrt(st.m2 / (double)st.n) : 0.0;
  return 0;
}

// ---- groups: several sessions of one GPU sharing one batched stage-2 forward per step (BASELINE config 5) ----
static Group* get_group(Engine* e, int id) { return (id >= 0 && id < (int)e->groups.size()) ? e->groups[id] : nullptr; }

// Why a member's stream state survives a membership change.  A change runs only when none of the session's or the group's host-API
// steps is uncollected, and it synchronises the device before it frees or rebuilds anything, so no step of the old layout is in flight.
// The guards of the steps after it still hold across the switch of a member's stage 2 between sC2s[0] (grouped) and sC2s[b] (alone):
//   * every cross-stage guard is an event of the member's own ring, indexed by its own step count (which a change keeps), so the
//     waits of step k on the events of steps k-1, k-2 and k-3 find them wherever those steps ran;
//   * d_colmin[0] is only ever written on sC2s[0] and d_colmin[1] only on sC2s[1] (a member uses sC2s[0] with d_colmin[0], a single
//     session sC2s[b] with d_colmin[b]), so each stays ordered by its stream;
//   * the stage-2 plans a step uses are new after a change (the group's rebuilt plan, or the leaving member's own plans built by the
//     change), and the group's waits on ev_fwd / pro / conv of steps before the change find completed events.
// The host staging ring (h_in / h_out / h_n, ev[r].dec) is indexed by the group's step while grouped and by the session's step alone;
// with nothing in flight at a change, no slot of one indexing is still in use when the other takes over.

// The conditions on a group's member list (create, add and remove all end in one); nullptr when it may form a group.
static const char* group_refusal(Engine* e, const std::vector<Session*>& members) {
  if (members.empty() || (int)members.size() > kMaxGroupBatch) return "a group holds 1..64 sessions";
  const Session* s0 = members[0];
  for (const Session* s : members)
    if (s->Tw != s0->Tw) return "group members must be distinct sessions with the same window length";
  // one chunk length serves every member in ryk_group_submit / ryk_group_push_device
  for (const Session* s : members)
    if (s->n_in != s0->n_in || s->in.rate != s0->in.rate || s->out.rate != s0->out.rate)
      return "group members must have the same device input and output rates";
  std::vector<const Voice*> voices;
  for (const Session* s : members)
    if (std::find(voices.begin(), voices.end(), s->voice) == voices.end()) voices.push_back(s->voice);
  if (voices.size() > 1 && e->precision != 1) return "a group of several voices needs precision 1 (FP16 tensor cores)";
  if ((int)voices.size() > kMaxGroupVoices) return "a group holds at most 8 distinct voices";
  const UNet* n0 = voices[0]->stage2;
  for (const Voice* v : voices)
    if (v->stage2->in_ch != n0->in_ch || v->stage2->out_ch != n0->out_ch || v->stage2->base != n0->base)
      return "the members' stage-2 models must have the same (in, out, base) channels";
  return nullptr;
}

// A session's host-API steps are all collected (device-resident steps count as collected).
static bool session_idle(const Session* s) { return s->collected == s->step; }

// The one way a group's batched stage 2 is built: around `members` (slot i = members[i]), for ryk_group_create, _add and _remove.
// Builds the voice table, a plan at the new batch size and keep hull under a new owner id and its per-item weights first; only when
// all of that succeeded does it release the old plan (on the net of the old first voice), move the voices' `users` counts, and reset
// the graphs that hold slot offsets into the old plan (the group's forward, every member's stage-2 prologue / epilogue).  A session
// that was not a member before also drops its own stage-2 plans and graphs: a session that ran alone captured s2_layers on them.  On
// failure the group and every session are left as they were.  Waits for the device: the old graphs may still be running.
static int group_rebuild(Engine* e, Group* G, const std::vector<Session*>& members) {
  const char* refusal = group_refusal(e, members);
  if (refusal) { set_error(refusal); return -1; }
  RYK_CUDA(cudaDeviceSynchronize());
  // Members of different voices share the forward: each batch item reads its voice's weights (unet_plan_set_voices).
  std::vector<Voice*> voices;
  std::vector<int> voice_of;
  for (Session* m : members) {
    const auto it = std::find(voices.begin(), voices.end(), m->voice);
    voice_of.push_back((int)(it - voices.begin()));
    if (it == voices.end()) voices.push_back(m->voice);
  }
  std::vector<const UNet*> nets;
  for (const Voice* v : voices) nets.push_back(v->stage2);
  // the batched forward computes the decoder rows of the hull of the members' kept frames (their e_conv may differ); the members
  // share Tw, so their padded tails start at the same row
  std::vector<int> kb, kl;
  for (Session* m : members) { kb.push_back(m->e_conv); kl.push_back(m->n_feat); }
  int keep_begin = 0, keep_len = 0;
  keep_hull((int)members.size(), kb.data(), kl.data(), &keep_begin, &keep_len);
  const int owner = ++e->plan_owners;
  UNetPlan* p2 = nullptr;
  if (unet_get_plan(e, voices[0]->stage2, (int)members.size(), members[0]->Tp, 512, e->precision, &p2, owner, keep_begin, keep_len, false,
                    members[0]->Tw) ||
      unet_plan_set_voices(p2, nets, voice_of)) {
    unet_release_owner(voices[0]->stage2, owner);
    return -1;
  }
  if (G->p2) unet_release_owner(G->voices[0]->stage2, G->owner);
  for (Voice* v : G->voices) v->users--;
  for (Voice* v : voices) v->users++;
  G->voices = voices; G->owner = owner; G->p2 = p2;
  G->fwd_graph.reset();
  for (size_t i = 0; i < members.size(); ++i) {
    Session* m = members[i];
    if (m->group != G) {
      for (int b = 0; b < 2; ++b) unet_release_owner(m->voice->stage2, m->s2_owner[b]);
      for (ParityGraphs& pg : m->graphs) pg.s2_layers.reset();
    }
    m->group = G; m->slot = (int)i;
    for (HandoffGraphs& hg : m->hgraphs) { hg.s2_pro.reset(); hg.s2_epi.reset(); }
  }
  G->members = members;
  return 0;
}

int ryk_group_create(ryk_engine* h, const int* session_ids, int n_sessions, int* group_id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(session_ids && group_id && n_sessions >= 1 && n_sessions <= kMaxGroupBatch, "a group holds 1..64 sessions");
  std::vector<Session*> members;
  for (int i = 0; i < n_sessions; ++i) {
    Session* s = get_session(e, session_ids[i]);
    RYK_CHECK(s && !s->group && std::find(members.begin(), members.end(), s) == members.end(),
              "group members must be distinct sessions with the same window length, none of them in a group");
    RYK_CHECK(session_idle(s), "collect every submitted chunk of a session before it joins a group");
    members.push_back(s);
  }
  Group* G = new Group();
  if (group_rebuild(e, G, members)) { delete G; return -1; }
  { int lo = 0, hi = 0; RYK_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi)); RYK_CUDA(cudaStreamCreateWithPriority(&G->sG, cudaStreamNonBlocking, lo)); }
  for (int i = 0; i < kRing; ++i) RYK_CUDA(cudaEventCreateWithFlags(&G->ev_fwd[i], cudaEventDisableTiming));
  RYK_CUDA(cudaDeviceSynchronize());
  e->groups.push_back(G);
  *group_id = (int)e->groups.size() - 1;
  return 0;
}

int ryk_group_add(ryk_engine* h, int group_id, int session_id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Group* G = get_group(e, group_id);
  RYK_CHECK(G != nullptr, "no such group");
  Session* s = get_session(e, session_id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(s->group == nullptr, "the session is already in a group");
  RYK_CHECK(G->collected == G->step, "collect every submitted chunk of the group before changing its members");
  RYK_CHECK(session_idle(s), "collect every submitted chunk of a session before it joins a group");
  std::vector<Session*> members = G->members;
  members.push_back(s);
  return group_rebuild(e, G, members);
}

int ryk_group_remove(ryk_engine* h, int group_id, int session_id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Group* G = get_group(e, group_id);
  RYK_CHECK(G != nullptr, "no such group");
  Session* s = get_session(e, session_id);
  RYK_CHECK(s != nullptr && s->group == G, "the session is not a member of this group");
  RYK_CHECK(G->members.size() > 1, "the session is the group's last member: destroy the group instead");
  RYK_CHECK(G->collected == G->step, "collect every submitted chunk of the group before changing its members");
  std::vector<Session*> members = G->members;
  members.erase(members.begin() + s->slot);
  RYK_CUDA(cudaDeviceSynchronize());
  // the session's own stage-2 plans, as session_build makes its stage-1 plans: its next step (alone) allocates nothing
  for (int b = 0; b < 2; ++b) {
    UNetPlan* p = nullptr;
    if (s2_plan(e, s, b, &p)) {
      for (int c = 0; c < 2; ++c) unet_release_owner(s->voice->stage2, s->s2_owner[c]);
      return -1;
    }
  }
  if (group_rebuild(e, G, members)) {
    for (int b = 0; b < 2; ++b) unet_release_owner(s->voice->stage2, s->s2_owner[b]);
    return -1;
  }
  s->group = nullptr; s->slot = 0;
  for (ParityGraphs& pg : s->graphs) pg.s2_layers.reset();
  for (HandoffGraphs& hg : s->hgraphs) { hg.s2_pro.reset(); hg.s2_epi.reset(); }
  return 0;
}

int ryk_group_members(ryk_engine* h, int group_id, int* session_ids, int capacity) {
  Engine* e = &h->impl;
  Group* G = get_group(e, group_id);
  RYK_CHECK(G != nullptr, "no such group");
  const int n = (int)G->members.size();
  for (int i = 0; i < n && i < capacity && session_ids; ++i) {
    const auto it = std::find(e->sessions.begin(), e->sessions.end(), G->members[i]);
    session_ids[i] = (int)(it - e->sessions.begin());
  }
  return n;
}

int ryk_group_destroy(ryk_engine* h, int group_id) {
  Engine* e = &h->impl;
  Group* G = get_group(e, group_id);
  RYK_CHECK(G != nullptr, "no such group");
  RYK_CUDA(cudaDeviceSynchronize());
  const int owner = G->owner;
  const std::vector<Voice*> voices = G->voices;
  group_free(G);                     // the member sessions survive (ungrouped) and are destroyed separately
  unet_release_owner(voices[0]->stage2, owner);
  for (Voice* v : voices) v->users--;
  e->groups[group_id] = nullptr;
  return 0;
}

int ryk_group_size(ryk_engine* h, int group_id) {
  Group* G = get_group(&h->impl, group_id);
  return G ? (int)G->members.size() : -1;
}

// Queue one chunk per member (host samples; waves[i] belongs to the member in slot i, see ryk_group_members).
int ryk_group_submit(ryk_engine* h, int group_id, const float* const* waves, int n, long long* ticket) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Group* G = get_group(e, group_id);
  RYK_CHECK(G != nullptr, "no such group");
  RYK_CHECK(G->step - G->collected < kRing - 2, "too many chunks in flight: collect before submitting more");
  const long long k = G->step;
  const int r = (int)(k % kRing);
  std::vector<const float*> d_chunks(G->members.size());
  for (size_t i = 0; i < G->members.size(); ++i) {
    Session* s = G->members[i];
    RYK_CHECK(n == s->n_in, "chunk length must be round(rate * buffer_time) at the session's input rate");
    if (stage_in(s, r, waves[i])) return -1;
    d_chunks[i] = s->d_chunk[r];
  }
  if (group_enqueue(e, G, d_chunks.data())) return -1;
  for (Session* s : G->members)
    if (stage_out(s, r, s->h_out[r], s->h_n[r], cudaMemcpyDeviceToHost)) return -1;
  if (ticket) *ticket = k;
  return 0;
}

// Wait for step `ticket` of every member; outs[i] receives member i's samples, n_outs[i] their count.
int ryk_group_collect(ryk_engine* h, int group_id, long long ticket, double* const* outs, int out_capacity, int* n_outs) {
  Engine* e = &h->impl;
  Group* G = get_group(e, group_id);
  RYK_CHECK(G != nullptr, "no such group");
  RYK_CHECK(ticket == G->collected && ticket < G->step, "tickets are collected in submission order");
  for (size_t i = 0; i < G->members.size(); ++i)
    if (collect_out(G->members[i], ticket, outs[i], out_capacity, &n_outs[i])) return -1;
  G->collected++;
  return 0;
}

// Device-resident group step, asynchronous (see ryk_session_push_device).
int ryk_group_push_device(ryk_engine* h, int group_id, const float* const* waves_dev, int n, double* const* outs_dev, int out_capacity,
                          int* const* n_outs_dev) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Group* G = get_group(e, group_id);
  RYK_CHECK(G != nullptr, "no such group");
  for (Session* s : G->members) {
    RYK_CHECK(n == s->n_in, "chunk length must be round(rate * buffer_time) at the session's input rate");
    RYK_CHECK(out_capacity >= s->max_out, "out_capacity must hold the most samples a step returns (ryk_session_io_geometry max_out)");
  }
  const int r = (int)(G->step % kRing);
  if (group_enqueue(e, G, waves_dev)) return -1;
  for (size_t i = 0; i < G->members.size(); ++i) {
    Session* s = G->members[i];
    if (stage_out(s, r, outs_dev[i], n_outs_dev[i], cudaMemcpyDeviceToDevice)) return -1;
    s->collected = s->step;
  }
  G->collected = G->step;
  return 0;
}

// Diagnostics (RYK_STAGE_TIMES=1 at session creation): device timeline of the last min(steps, 8) steps.  start/end[i*5 + a] =
// ms since the oldest listed step began, for stage a in {wave slides (+ input resampler), WORLD analysis, stage 1 (feature slides +
// silence gate, U-Net, mc2sp), stage 2 (prologue..epilogue), synthesis}; returns the number of steps listed (oldest first).
int ryk_session_stage_times(ryk_engine* h, int id, float* start, float* end) {
  Engine* e = &h->impl;
  Session* s = get_session(e, id);
  RYK_CHECK(s != nullptr && s->stage_times && s->step >= 1, "stage timing is not enabled for this session (RYK_STAGE_TIMES=1) or no step ran");
  RYK_CUDA(cudaDeviceSynchronize());
  const int n = s->step < kRing ? (int)s->step : kRing;
  const int r0 = (int)((s->step - n) % kRing);
  for (int i = 0; i < n; ++i) {
    const int r = (int)((s->step - n + i) % kRing);
    for (int a = 0; a < 5; ++a) {
      RYK_CUDA(cudaEventElapsedTime(&start[i * 5 + a], s->tev[0][0][r0], s->tev[a][0][r]));
      RYK_CUDA(cudaEventElapsedTime(&end[i * 5 + a], s->tev[0][0][r0], s->tev[a][1][r]));
    }
  }
  return n;
}


// ---- output re-blocker + silence gate -----------------------------------------------------------------
static Reblock* get_reblock(Engine* e, int id) { return (id >= 0 && id < (int)e->reblocks.size()) ? e->reblocks[id] : nullptr; }

int ryk_reblock_create(ryk_engine* h, int out_audio_chunk, int max_in, int n_fft, int hop, double threshold_db, int* reblock_id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(out_audio_chunk > n_fft / 2 && max_in > 0, "out_audio_chunk must exceed n_fft / 2 (reflect-centred STFT)");
  RYK_CHECK(n_fft >= 64 && n_fft <= 4096 && (n_fft & (n_fft - 1)) == 0 && hop > 0, "unsupported STFT geometry");
  Reblock* R = new Reblock();
  for (int i = 0; i < kRing; ++i) R->ev[i] = nullptr;
  R->chunk = out_audio_chunk; R->max_in = max_in; R->n_fft = n_fft; R->hop = hop; R->threshold_db = threshold_db;
  R->cap = 2 * out_audio_chunk + 2 * max_in;
  auto A = [&](void** p, size_t bytes) -> int { RYK_CUDA(cudaMalloc(p, bytes)); RYK_CUDA(cudaMemset(*p, 0, bytes)); R->allocs.push_back(*p); return 0; };
  auto H = [&](void** p, size_t bytes) -> int { RYK_CUDA(cudaMallocHost(p, bytes)); memset(*p, 0, bytes); R->pinned.push_back(*p); return 0; };
  int rc = 0;
  rc |= A((void**)&R->d_state, sizeof(ReblockState));
  for (int i = 0; i < 2; ++i) rc |= A((void**)&R->d_frag[i], sizeof(double) * R->cap);
  rc |= A((void**)&R->d_scratch, sizeof(double) * output_gate_scratch_doubles(out_audio_chunk, n_fft, hop));
  rc |= A((void**)&R->d_stage_in, sizeof(double) * max_in);
  rc |= A((void**)&R->d_stage_n, sizeof(int));
  for (int i = 0; i < kRing && !rc; ++i) {
    rc |= A((void**)&R->d_chunk[i], sizeof(double) * out_audio_chunk);
    rc |= A((void**)&R->d_nvalid[i], sizeof(int));
    rc |= A((void**)&R->d_status[i], sizeof(int));
    rc |= A((void**)&R->d_power[i], sizeof(double));
    rc |= H((void**)&R->h_chunk[i], sizeof(double) * out_audio_chunk);
    rc |= H((void**)&R->h_status[i], sizeof(int));
    rc |= H((void**)&R->h_power[i], sizeof(double));
    rc |= H((void**)&R->h_overflow[i], sizeof(int));
    if (!rc && cudaEventCreateWithFlags(&R->ev[i], cudaEventDisableTiming) != cudaSuccess) rc = -1;
  }
  if (rc) { reblock_free(R); return -1; }
  RYK_CUDA(cudaDeviceSynchronize());             // the zero-fills ran on the legacy default stream; pushes use other (non-blocking) streams
  e->reblocks.push_back(R);
  *reblock_id = (int)e->reblocks.size() - 1;
  return 0;
}

int ryk_reblock_destroy(ryk_engine* h, int id) {
  Engine* e = &h->impl;
  Reblock* R = get_reblock(e, id);
  RYK_CHECK(R != nullptr, "no such re-blocker");
  RYK_CUDA(cudaDeviceSynchronize());
  reblock_free(R);
  e->reblocks[id] = nullptr;
  return 0;
}

// Append *n_dev samples (device memory) and emit at most one chunk + its gate decision into ring slot ticket % 8.
// session_id >= 0: the work is queued on that session's decode stream right behind its latest step; with wave_dev == NULL the
// step's own output (blocks + count) is consumed in place.  session_id < 0: engine stream, wave_dev / n_dev required.
int ryk_reblock_push_device(ryk_engine* h, int id, int session_id, const double* wave_dev, const int* n_dev, long long* ticket) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Reblock* R = get_reblock(e, id);
  RYK_CHECK(R != nullptr, "no such re-blocker");
  cudaStream_t st = e->stream;
  if (session_id >= 0) {
    Session* s = get_session(e, session_id);
    RYK_CHECK(s != nullptr, "no such session");
    RYK_CHECK(s->step > 0, "the session has not processed a chunk yet");
    st = s->sD;
    if (!wave_dev) {
      const int b = (int)((s->step - 1) & 1);
      RYK_CHECK(s->max_out <= R->max_in, "re-blocker max_in is smaller than the most samples a session step returns");
      wave_dev = step_out(s, b); n_dev = step_n_out(s, b);
    }
  }
  RYK_CHECK(wave_dev != nullptr && n_dev != nullptr, "wave_dev / n_dev are required without an attached session");
  const long long k = R->pushed;
  const int r = (int)(k % kRing);
  k_reblock<<<1, 1024, 0, st>>>(R->d_state, R->d_frag[0], R->d_frag[1], R->cap, wave_dev, n_dev, R->max_in, R->chunk, R->d_chunk[r], R->d_nvalid[r]);
  RYK_CUDA(cudaGetLastError());
  if (output_gate_async(e, R->d_chunk[r], R->d_nvalid[r], R->chunk, R->n_fft, R->hop, R->threshold_db, R->d_scratch, R->d_power[r], R->d_status[r], st)) return -1;
  RYK_CUDA(cudaMemcpyAsync(R->h_status[r], R->d_status[r], sizeof(int), cudaMemcpyDeviceToHost, st));
  RYK_CUDA(cudaMemcpyAsync(R->h_power[r], R->d_power[r], sizeof(double), cudaMemcpyDeviceToHost, st));
  RYK_CUDA(cudaMemcpyAsync(R->h_chunk[r], R->d_chunk[r], sizeof(double) * R->chunk, cudaMemcpyDeviceToHost, st));
  RYK_CUDA(cudaMemcpyAsync(R->h_overflow[r], &R->d_state->overflow, sizeof(int), cudaMemcpyDeviceToHost, st));
  RYK_CUDA(cudaEventRecord(R->ev[r], st));
  R->pushed++;
  if (ticket) *ticket = k;
  return 0;
}

// Wait for push `ticket` (one of the last 8): *status 0 = no chunk this step, 1 = chunk written to chunk_out, 2 = chunk was
// silent (the reference forwards None); *power_db = mean STFT power of the chunk (0 when status is 0).
int ryk_reblock_collect(ryk_engine* h, int id, long long ticket, double* chunk_out, int* status, double* power_db) {
  Engine* e = &h->impl;
  Reblock* R = get_reblock(e, id);
  RYK_CHECK(R != nullptr, "no such re-blocker");
  RYK_CHECK(ticket >= 0 && ticket < R->pushed && ticket + kRing > R->pushed, "ticket is not among the last 8 pushes");
  const int r = (int)(ticket % kRing);
  RYK_CUDA(cudaEventSynchronize(R->ev[r]));
  // the reference's wave_fragment grows without bound when a step yields more than one out_audio_chunk (decode_worker.py:47-52);
  // the device fragment is bounded, so that configuration is an error here instead of silently dropped samples
  RYK_CHECK(*R->h_overflow[r] == 0, "re-blocker fragment overflow: a step produced more samples than out_audio_chunk can drain");
  const int stt = *R->h_status[r];
  if (status) *status = stt;
  if (power_db) *power_db = *R->h_power[r];
  if (chunk_out && stt != 0) memcpy(chunk_out, R->h_chunk[r], sizeof(double) * R->chunk);
  return 0;
}

// Non-blocking: *done = 1 when ryk_reblock_collect(ticket) would not wait.
int ryk_reblock_poll(ryk_engine* h, int id, long long ticket, int* done) {
  Engine* e = &h->impl;
  Reblock* R = get_reblock(e, id);
  RYK_CHECK(R != nullptr && done != nullptr, "no such re-blocker");
  RYK_CHECK(ticket >= 0 && ticket < R->pushed && ticket + kRing > R->pushed, "ticket is not among the last 8 pushes");
  cudaError_t q = cudaEventQuery(R->ev[ticket % kRing]);
  if (q != cudaSuccess && q != cudaErrorNotReady) RYK_CUDA(q);
  *done = q == cudaSuccess ? 1 : 0;
  return 0;
}

// Device pointers of ring slot ticket % 8 (valid until 8 further pushes; ordered after the push on its stream).
int ryk_reblock_result_device(ryk_engine* h, int id, long long ticket, const double** chunk_dev, const int** status_dev, const double** power_dev) {
  Engine* e = &h->impl;
  Reblock* R = get_reblock(e, id);
  RYK_CHECK(R != nullptr, "no such re-blocker");
  RYK_CHECK(ticket >= 0 && ticket < R->pushed && ticket + kRing > R->pushed, "ticket is not among the last 8 pushes");
  const int r = (int)(ticket % kRing);
  if (chunk_dev) *chunk_dev = R->d_chunk[r];
  if (status_dev) *status_dev = R->d_status[r];
  if (power_dev) *power_dev = R->d_power[r];
  return 0;
}

// Host buffers: H2D + push + collect.
int ryk_reblock_push(ryk_engine* h, int id, const double* wave, int n, double* chunk_out, int* status, double* power_db) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Reblock* R = get_reblock(e, id);
  RYK_CHECK(R != nullptr, "no such re-blocker");
  RYK_CHECK(n >= 0 && n <= R->max_in, "more samples than the re-blocker's max_in");
  if (n > 0) RYK_CUDA(cudaMemcpyAsync(R->d_stage_in, wave, sizeof(double) * n, cudaMemcpyHostToDevice, e->stream));
  RYK_CUDA(cudaMemcpyAsync(R->d_stage_n, &n, sizeof(int), cudaMemcpyHostToDevice, e->stream));
  RYK_CUDA(cudaStreamSynchronize(e->stream));           // n lives on the caller's stack
  long long ticket = 0;
  if (ryk_reblock_push_device(h, id, -1, R->d_stage_in, R->d_stage_n, &ticket)) return -1;
  return ryk_reblock_collect(h, id, ticket, chunk_out, status, power_db);
}

}  // extern "C"
