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
// Session state is grouped by the counter that selects it: ParitySet par[step & 1], HandoffSlot ho[step % 3] (three hand-off slots, so
// that stage 1 of a chunk does not wait for stage 2 of the chunk two steps before), StepEvents ev[step % kRing], and HostSlot
// io[ticket % kRing], numbered by the caller's ticket.  Events order producer/consumer and guard reuse.
// The effective-frame count that selects the stage-1 plan (T_eff + 128 - T_eff % 128) is read on the device by a
// conditional graph node, so the host never waits inside a step.
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <array>
#include <chrono>
#include <numeric>
#include <vector>

#include "../../include/ryk.h"
#include "agc.h"
#include "echo.h"
#include "engine.h"
#include "features.h"
#include "limiter.h"
#include "snapshot.h"
#include "synth.h"
#include "unet.h"

namespace ryk {

constexpr int kRing = 8;          // event / host-slot ring (pipeline depth is bounded by the buffer guards below)
constexpr int kHandoff = 3;       // slots of the stage-1 -> stage-2 -> decode hand-off buffers, h = step % kHandoff
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
// The session's inputs: the microphone, and with echo cancellation the far end.  Each has an InputSignal in Session and an InputState in
// each ParitySet; one input path (input_alloc, input_to_model) serves both.
enum { kMic = 0, kFar = 1, kInputs = 2 };
struct InputSignal {               // the step's samples, read by the captured gate graph
  float* d_fixed = nullptr;        // as given (n_in samples)
  float* d_model = nullptr;        // device input rate: their resampling (n_wave model-rate samples)
};
// The stream state of one input that step k reads from par[b] and writes for the next step into par[b ^ 1].
struct InputState {
  float* win = nullptr;            // device input rate: history window (in.hist device-rate samples)
  ResampleState* rs = nullptr;     // device input rate: the streaming resampler's position
  DenoiseState* dn = nullptr;      // the frame stage of noise suppression / echo cancellation (the microphone's also holds the filter's)
};
// What the parity b = k & 1 of the session's own step k selects.  Step k reads the sliding windows of par[b] and writes those of
// par[b ^ 1]; the rest of par[b] is step k's own.  Buffers are null until allocated, so a partly built session can be freed.
struct ParitySet {
  // sliding windows
  float* wave_win = nullptr;
  float *cw_f0 = nullptr, *cw_ap = nullptr, *cw_mc = nullptr, *cw_wave = nullptr; uint8_t* cw_voiced = nullptr;
  float *dw_f0 = nullptr, *dw_ap = nullptr, *dw_sp = nullptr;
  InputState input[kInputs];                     // the microphone's and the far end's input windows and stream state
  double* out_hist = nullptr;                    // device rates: kept synthesizer samples (out.hist)
  ResampleState* out_st = nullptr;               // device rates: the output resampler's position
  LimHist lim;                                   // output limiter: the history of y and g0 and the stream position
  AgcState* agc = nullptr;                       // automatic gain control: the stream position, level, gains and block history
  // inter-stage buffers
  float *enc_f0 = nullptr, *enc_sp = nullptr, *enc_ap = nullptr, *enc_mc = nullptr; uint8_t* enc_voiced = nullptr;
  uint8_t* d_mask = nullptr; int* d_index = nullptr; int* d_count = nullptr;     // silence gate
  double* d_out_fixed = nullptr; int* d_n_fixed = nullptr;      // blocks written by the (captured) decode graph
  double* d_rout_fixed = nullptr; int* d_rn_fixed = nullptr;    // their device-rate resampling
  double* d_lim_out = nullptr;                   // output limiter: the samples the step returns (as many as the two above)
  cudaStream_t sA = nullptr;                     // WORLD analysis: two chunks' analyses may be in flight
  DioPlan* dio = nullptr;                        // f0 methods 0 and 1 (owned)
  CrepePlan* crepe = nullptr;                    // f0 method 2: one CREPE forward in place of DIO/Harvest (owned)
  ParityGraphs graphs;
};
// The hand-off set of slot h = k % kHandoff: written by stage 1 (sp_out by the stage-2 epilogue), read by stage 2 and the decode slide.
struct HandoffSlot {
  float *mc_out = nullptr, *f0_out = nullptr, *ap_out = nullptr, *sp_mid = nullptr, *sp_out = nullptr; uint8_t* voiced_out = nullptr;
  double* formant = nullptr;       // the step's formant ratio: written by the stage-1 epilogue, read by the stage-2 epilogue
};
// What the session's own step k keeps in slot r = k % kRing.  Null until created, so a partly built session can be freed.
struct StepEvents {
  cudaEvent_t gate = nullptr;      // wave slides of step k done (stream E)
  cudaEvent_t enc = nullptr;       // analysis of step k done
  cudaEvent_t cslide = nullptr;    // head of stage 1 of step k done: par[b].enc_* and par[b ^ 1].cw_wave consumed
  cudaEvent_t s1 = nullptr;        // stage 1 of step k done
  cudaEvent_t pro = nullptr;       // stage-2 prologue of step k done (group members only)
  cudaEvent_t conv = nullptr;      // stage 2 of step k done
  cudaEvent_t dslide = nullptr;    // the converted features of step k sit in the decode window
  std::array<cudaEvent_t*, 7> all() { return {&gate, &enc, &cslide, &s1, &pro, &conv, &dslide}; }
  cudaEvent_t tev[5][2] = {};      // RYK_STAGE_TIMES=1: [stage E1,E2,S1,S2,D][begin/end]
};
// A block the host sets between steps and the captured graphs read: the setters change `next`, host_block_sync copies it (DESIGN.md §4a).
template <typename T> struct HostBlock {
  T next = {};                     // what the next submitted step uses
  bool dirty = false;              // next changed since the last submitted step
  T* ring = nullptr;               // pinned staging: slot k % kRing for step k (the session's BufferSet)
};
// The host-API staging of the caller's ticket t in slot t % kRing: the session's own step alone, the group's step while grouped.  A
// membership change needs every host-API step collected, so no slot of one numbering is in use when the other takes over.
struct HostSlot {
  float* h_in = nullptr; double* h_out = nullptr; int* h_n = nullptr;     // pinned
  cudaEvent_t dec = nullptr;       // output staged (after the copies the entry point appends to stream D)
};
// Stage 2 of a session alone runs the chunks of parity b on lane b, with two activation plans: the latency-bound bottleneck layers
// (c4-d2: 30 % of a forward's time, a few CTAs each) of one chunk overlap the GPU-filling layers of its neighbour.  A group member runs
// its prologue and epilogue on lane 0 (s2_lane).
struct Stage2Lane {
  cudaStream_t stream = nullptr;
  float* d_colmin = nullptr;       // stage-2 prologue scratch, written only on this lane's stream
  int owner = 0;                   // plan-cache owner id of the lane's stage-2 plan
  StageGraph s2_layers;            // alone: stage-2 layers 1..14
};
struct Group;
struct Session {
  int s1_owner = 0;                // plan-cache owner id of the stage-1 plans (activation buffers are private to the session)
  Group* group = nullptr; int slot = 0;        // member of a batched stage-2 group (config 5), else nullptr
  Voice* voice = nullptr; int voice_id = 0;    // the voice the session converts into (ryk_session_set_voice changes it between steps)
  int precision = 1; bool s1_fused = true;     // the engine's precision and stage-1 mode at creation: every plan and graph keeps them
  ryk_session_config cfg;
  SptkMats sptk;                   // the engine's sp2mc / mc2sp matrices of cfg's (order, alpha, fft_length), captured in the graphs
  int hop, rate, n_wave, n_feat, e_wave, e_enc_frames, e_conv, e_dec;
  int Lw, Tw, Td, nb, C;
  int Tp;                          // stage-2 padded length: Tw rounded up to the next multiple of 128 (always > Tw)
  long long step = 0;              // chunks submitted
  long long collected = 0;         // chunks collected through the host API
  cudaStream_t sE = nullptr, sC = nullptr, sD = nullptr;     // gate | stage 1 | decode
  cudaStream_t sA_side = nullptr;            // D4C branch of the analysis graphs while they are captured; never used at step time
  ParitySet par[2];
  HandoffSlot ho[kHandoff];
  StepEvents ev[kRing]; bool stage_times = false;
  HostSlot io[kRing];
  Stage2Lane lane[2];
  std::array<cudaStream_t, 7> streams() const { return {sE, par[0].sA, par[1].sA, sC, lane[0].stream, lane[1].stream, sD}; }
  double* d_mse = nullptr;             // silence-gate scratch (stream C)
  double* dec_f0_f64 = nullptr;
  int max_blocks;
  InputSignal input[kInputs];          // the microphone (always) and the far end (echo cancellation)
  HandoffGraphs hgraphs[kHandoffGraphs];
  Synth* synth = nullptr;
  // Device rates (ryk_session_set_input_rate / _output_rate): chunks arrive at in.rate and outputs leave at out.rate; analysis, the
  // U-Nets and synthesis stay at cfg.fs.  rate 0 = that side runs at fs (no resampler).
  struct RateSide {
    int rate = 0, up = 1, down = 1, n_taps = 0;
    int hist = 0;                                 // input: history window (chunk + left support); output: kept synthesizer samples
    double* d_h = nullptr;
  } in, out;
  int n_in = 0;                    // samples per pushed chunk (n_wave without an input resampler)
  int delay_in = 0;                // leading zeros of the model-rate input (model samples)
  int max_out = 0;                 // most output samples one step can return
  // The session's f0 map (ryk_session_set_f0_map / _f0_follow), its formant ratio (ryk_session_set_formant) and the statistics of its
  // speaker (ryk_session_f0_measure).  The captured stage-1 graphs read *d_f0_map, a host block synced on stream C in front of a step's
  // stage 1 (follow mode: its input side is the fallback).  The formant ratio reaches stage 2 through ho[h].formant, never from
  // *d_f0_map (DESIGN.md §4a).
  HostBlock<F0Map> f0_map;
  bool f0_measure = false;         // the head of stage 1 ends with k_f0_measure
  bool f0_reset = false;           // the statistics restart at the next submitted step
  F0Map* d_f0_map = nullptr; F0Stats* d_f0_stats = nullptr;
  // Input noise suppression (ryk_session_denoise, DESIGN.md §4f): the filter runs in the wave-slide graph on the model-rate chunk.  Its
  // parameter block dn.params is a host block synced on stream E in front of the graph; the learning state is device-owned.
  bool denoise = false;
  DenoiseWork dn;
  HostBlock<DenoiseParams> dn_params;
  float* d_chunk_dn = nullptr;     // the step's filtered chunk (n_wave model-rate samples)
  // Echo cancellation (ryk_session_echo_cancel, DESIGN.md §4g): the canceller runs in the frame stage it shares with the noise
  // suppression, on the far end (input[kFar]) the host hands in for each step.  Its parameter block aec.params is a host block synced
  // on stream E in front of the graph; the filter block is device-owned and updated in place.
  bool echo = false;
  EchoWork aec;
  HostBlock<EchoParams> aec_params;
  std::vector<float> far_next;     // the far end of the next submitted step (ryk_session_echo_reference; zeros when none was given)
  bool far_set = false;
  float* h_far = nullptr;          // pinned staging of the far end: slot k % kRing (n_in samples) for step k
  // Output limiter (ryk_session_limiter, DESIGN.md §4i): runs last in the synthesis graph, at the output rate.  Its settings block
  // lim.params is a host block synced on stream D in front of the decode slides; the history is double-buffered by parity.
  bool limiter = false;
  double lim_lookahead_ms = 0.0, lim_hold_ms = 0.0;   // L and R follow the output rate (ryk_session_set_output_rate reallocates)
  double lim_ceiling_db = 0.0;     // what the next submitted step uses, with lim_params.next.gain
  LimWork lim;
  HostBlock<LimParams> lim_params;
  // Automatic gain control (ryk_session_agc, DESIGN.md §4j): runs in the wave-slide graph after the frame stage, at the model rate.  Its
  // settings block agc.params is a host block synced on stream E in front of the graph; the state is double-buffered by parity.
  bool agc = false;
  double agc_db[3] = {};           // target, max gain and gate in dB of the next submitted step
  AgcWork agcw;
  HostBlock<AgcParams> agc_params;
  float* d_chunk_agc = nullptr;    // the step's gain-controlled chunk (n_wave model-rate samples)
  BufferSet mem;                   // every device and pinned buffer above
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

// The session when it has not run a chunk yet (what its graphs capture at the first steps can still change), else nullptr with the
// error set: "no such session", or `refusal`.
static Session* fresh_session(Engine* e, int id, const char* refusal) {
  Session* s = get_session(e, id);
  if (!s) set_error("no such session");
  else if (s->step != 0) set_error(refusal);
  return s && s->step == 0 ? s : nullptr;
}

// (Re)allocates input i at chunk length n_in, with a history window and resampler state pair when `resampled` (device input rate, window
// of in.hist samples).  The far end also gets its host staging, the next step's samples and kRing pinned slots; the microphone is
// staged through HostSlot::h_in.
static int input_alloc(Session* s, int i, int n_in, bool resampled) {
  BufferSet& m = s->mem;
  InputSignal& x = s->input[i];
  if (m.device(&x.d_fixed, n_in)) return -1;
  if (resampled) {
    for (ParitySet& p : s->par) if (m.device(&p.input[i].win, s->in.hist) || m.device(&p.input[i].rs, 1)) return -1;
    if (m.device(&x.d_model, s->n_wave)) return -1;
  }
  if (i == kFar) {
    if (m.pinned(&s->h_far, (size_t)kRing * n_in)) return -1;
    s->far_next.assign(n_in, 0.f);
    s->far_set = false;
  }
  return 0;
}

// Drop the stage-2 plans of a session's own lanes and the graphs captured on them (a no-op for plans a group already released).
static void lanes_release(Session* s) {
  for (Stage2Lane& L : s->lane) {
    L.s2_layers.reset();
    unet_release_owner(s->voice->stage2, L.owner);
  }
}

// Frees a session, built or partly built, and releases its U-Net plans (call before the voice is freed).
static void session_free(Session* s) {
  if (!s) return;
  for (cudaStream_t st : s->streams()) if (st) { cudaStreamSynchronize(st); cudaStreamDestroy(st); }
  if (s->sA_side) cudaStreamDestroy(s->sA_side);
  for (StepEvents& ev : s->ev) {
    for (cudaEvent_t* p : ev.all()) if (*p) cudaEventDestroy(*p);
    for (auto& pair : ev.tev) for (cudaEvent_t t : pair) if (t) cudaEventDestroy(t);
  }
  for (HostSlot& io : s->io) if (io.dec) cudaEventDestroy(io.dec);
  for (ParitySet& p : s->par) { dio_plan_free(p.dio); crepe_plan_free(p.crepe); }
  synth_destroy(s->synth);
  unet_release_owner(s->voice->stage1, s->s1_owner);
  lanes_release(s);
  delete s;                                       // drops the stage graphs and frees the buffers
}

static void group_free(Group* G) {
  if (!G) return;
  if (G->sG) { cudaStreamSynchronize(G->sG); cudaStreamDestroy(G->sG); }
  for (int i = 0; i < kRing; ++i) if (G->ev_fwd[i]) cudaEventDestroy(G->ev_fwd[i]);
  for (Session* m : G->members) {
    m->group = nullptr;
    for (HandoffGraphs& hg : m->hgraphs) { hg.s2_pro.reset(); hg.s2_epi.reset(); }     // (they point into the group's plan)
  }
  delete G;
}

void session_destroy_all(Engine* e) {
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

static int stage1_body(Engine* e, Session* s, Voice* v, int owner, int b, int h, int tp1);

// Build into g the stage-1 graph of the chunks of step % 6 = j with a device-side switch over the padded-length buckets (CUDA
// conditional nodes, 12.8+), on the stage-1 plans of voice v under plan owner `owner`.
static int stage1_build_switch(Engine* e, Session* s, Voice* v, int owner, int j, StageGraph& g) {
  const int b = j & 1, h = j % kHandoff;
  const int n_buckets = s->Tp / 128 + 1;                 // <= 16: session_build refuses longer windows
  cudaGraph_t graph = nullptr;
  RYK_CUDA(cudaGraphCreate(&graph, 0));
  cudaGraphConditionalHandle handle;
  RYK_CUDA(cudaGraphConditionalHandleCreate(&handle, graph, 0, cudaGraphCondAssignDefault));
  // node 1: the setter (its body table is filled in once the bodies are captured)
  cudaGraphNode_t set_node = nullptr;
  const int* cnt = s->par[b].d_count;
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
    int rc = stage1_body(e, s, v, owner, b, h, i * 128);
    cudaGraph_t out = nullptr;
    cudaError_t err = cudaStreamEndCapture(s->sC, &out);
    if (rc) return rc;
    RYK_CUDA(err);
    kernels.n[i] = graph_kernels(body);
    if (kernels.n[i] < 0) return -1;
  }
  RYK_CUDA(cudaGraphKernelNodeSetParams(set_node, &kp));
  if (stage_graph_init(g, graph)) return -1;
  RYK_CUDA(cudaGraphUpload(g.exec, s->sC));     // the first step of each copy does not pay for the upload
  return 0;
}

// The head of stage 1 of a chunk of parity b: slide the feature window by the analysis outputs and run the silence gate on the
// chunk's wave window (mask / index / count of par[b], which only stage 1 reads).  It is all of stage 1 that the next chunks of this
// parity wait for: once it ran, their analysis may overwrite par[b].enc_* and their wave slide par[b ^ 1].cw_wave.
static int stage1_head(Engine* e, Session* s, int b) {
  const ParitySet &p = s->par[b], &q = s->par[b ^ 1];
  const int pe = s->e_enc_frames;
  const ryk_session_config& c = s->cfg;
  SlideBatch sb; sb.n = 0;
  slide_add<float>(sb, p.cw_f0, p.enc_f0 + pe, q.cw_f0, s->Tw, s->n_feat, 1);
  slide_add<float>(sb, p.cw_ap, p.enc_ap + (size_t)pe * s->nb, q.cw_ap, s->Tw, s->n_feat, s->nb);
  slide_add<float>(sb, p.cw_mc, p.enc_mc + (size_t)pe * s->C, q.cw_mc, s->Tw, s->n_feat, s->C);
  slide_add<uint8_t>(sb, p.cw_voiced, p.enc_voiced + pe, q.cw_voiced, s->Tw, s->n_feat, 1);
  if (slide_batch(sb, s->sC)) return -1;
  if (gate_mask_run(e, q.cw_wave, s->Tw * s->hop, c.fft_length, s->hop, c.threshold_db, s->Tw, s->d_mse, p.d_mask, p.d_index, p.d_count,
                    s->sC)) return -1;
  // the chunk's own frames: over a stream they tile the input, every 5 ms frame exactly once
  if (s->f0_measure && f0_measure_run(p.enc_f0 + pe, p.enc_voiced + pe, s->n_feat, s->d_f0_stats, s->d_f0_map, s->sC)) return -1;
  return 0;
}

// In front of the graphs of step k that read *dev, on the stream st that runs them in step order: when the block changed, stage it in
// pinned slot k % kRing and copy it into *dev, so step k is the first to see it.  The slot was last read by a copy of step k - kRing or
// earlier, which ended before the guard event of step k - kRing: the host waits for that event (at once unless a whole ring ahead).
template <typename T>
static int host_block_sync(HostBlock<T>& b, T* dev, long long k, cudaEvent_t guard, cudaStream_t st) {
  if (!b.dirty) return 0;
  if (k >= kRing) RYK_CUDA(cudaEventSynchronize(guard));
  T* slot = b.ring + k % kRing;
  *slot = b.next;
  RYK_CUDA(cudaMemcpyAsync(dev, slot, sizeof(T), cudaMemcpyHostToDevice, st));
  b.dirty = false;
  return 0;
}

// In front of the gate graph of step k on stream E, with echo cancellation: the step's far end (the samples given since the previous
// step, else zeros), copied on every step through pinned slot k % kRing under the guard host_block_sync uses on stream E.
static int far_sync(Session* s, long long k) {
  if (k >= kRing) RYK_CUDA(cudaEventSynchronize(s->ev[k % kRing].gate));
  float* slot = s->h_far + (size_t)(k % kRing) * s->n_in;
  if (s->far_set) memcpy(slot, s->far_next.data(), sizeof(float) * s->n_in);
  else memset(slot, 0, sizeof(float) * s->n_in);
  s->far_set = false;
  RYK_CUDA(cudaMemcpyAsync(s->input[kFar].d_fixed, slot, sizeof(float) * s->n_in, cudaMemcpyHostToDevice, s->sE));
  return 0;
}

// Input i at the model rate, enqueued on stream E in the gate graph of a step of parity b: at a device input rate its history window
// slides and its own copy of the streaming resampler runs, so the microphone and the far end stay aligned sample for sample.
static int input_to_model(Engine* e, Session* s, int b, int i, const float** model) {
  const InputSignal& x = s->input[i];
  const InputState &p = s->par[b].input[i], &q = s->par[b ^ 1].input[i];
  *model = x.d_fixed;
  if (!s->in.rate) return 0;
  if (slide<float>(p.win, x.d_fixed, q.win, s->in.hist, s->n_in, 1, s->sE)) return -1;
  if (resample_stream_in_run(e, q.win, s->in.hist, s->n_in, s->delay_in, s->in.up, s->in.down, s->in.d_h, s->in.n_taps, p.rs, q.rs,
                             x.d_model, s->n_wave, s->sE)) return -1;
  *model = x.d_model;
  return 0;
}

// The rest of stage 1 of a chunk of parity b and hand-off slot h: (gather ->) 1-D U-Net at padded length tp1 (0: no effective frame,
// voice_changer.py:32-35 skips the net) -> scatter into the silent template + f0 map, mc2sp.  Enqueued on stream C while it is captured
// as one body of the chunk's SWITCH graph; every body is captured when the session is created so that no chunk ever pays for a capture
// in the middle of a stream.
static int stage1_body(Engine* e, Session* s, Voice* v, int owner, int b, int h, int tp1) {
  const ParitySet &p = s->par[b], &q = s->par[b ^ 1];
  const HandoffSlot& o = s->ho[h];
  const ryk_session_config& c = s->cfg;
  const float* d_y = nullptr;
  if (tp1 > 0) {
    UNetPlan* p1 = nullptr;
    if (unet_get_plan(e, v->stage1, 1, 1, tp1, e->precision, &p1, owner)) return -1;
    if (stage1_prologue_run(v, q.cw_mc, p.d_index, p.d_count, s->C, (float*)p1->d_in, tp1, s->sC)) return -1;
    if (unet_forward(e, p1, s->sC)) return -1;
    d_y = (const float*)p1->d_out;
  }
  if (stage1_epilogue_run(v, d_y, p.d_index, p.d_mask, p.d_count, s->Tw, s->C, q.cw_f0, q.cw_ap, q.cw_voiced, s->nb, kSilentMc0,
                          o.mc_out, o.f0_out, o.ap_out, o.voiced_out, s->d_f0_map, s->sC, o.formant)) return -1;
  return mc2sp_run(e, s->sptk.d_H, o.mc_out, s->Tw, c.order, c.fft_length, 1e-16, o.sp_mid, nullptr, s->sC);
}

// Step k = s->step is enqueued in three parts so that a group can interleave its members:
//   front: streams E and C (analysis, gate, stage 1, mc2sp) and the stage-2 prologue
//   mid:   the stage-2 U-Net forward (single session: on its own lane; group: one batched forward on the group stream)
//   back:  stage-2 epilogue and stream D (synthesizer); results land in par[b].d_out_fixed / d_n_fixed; s->step advances.
// In each part b = k & 1: p = par[b] holds the step's own buffers and the sliding windows it reads, q = par[b ^ 1] the windows it
// writes; h = k % 3 is the hand-off slot, hgraphs[k % 6] the graphs that touch it, and ev[k % kRing] the step's events.

// The lane stage 2 of a chunk of parity b runs on: lane b for a session alone, lane 0 for a group member.
static Stage2Lane& s2_lane(Session* s, int b) { return s->lane[s->group ? 0 : b]; }
// The decode slide reads only the chunk's frames [e_conv, e_conv + n_feat) of the converted window, so stage 2 computes only the
// decoder rows those frames depend on; the prologue pads rows [Tw, Tp) with one row, so the encoder computes one copy of the rows
// that depend only on it.
static int s2_plan(Engine* e, const Session* s, Voice* v, int owner, UNetPlan** p2) {
  return unet_get_plan(e, v->stage2, 1, s->Tp, 512, e->precision, p2, owner, s->e_conv, s->n_feat, false, s->Tw);
}
static int s2_plan(Engine* e, const Session* s, const Stage2Lane& L, UNetPlan** p2) { return s2_plan(e, s, s->voice, L.owner, p2); }

// begin (which = 0) / end (1) of a stage in the RYK_STAGE_TIMES timeline
static int stage_time(Session* s, int stage, int which, int r, cudaStream_t st) {
  if (s->stage_times) RYK_CUDA(cudaEventRecord(s->ev[r].tev[stage][which], st));
  return 0;
}

// d_chunk_user: the caller's chunk in device memory, or nullptr when stage_in already copied it into input[kMic].d_fixed
static int session_front(Engine* e, Session* s, const float* d_chunk_user) {
  const long long k = s->step;
  const int b = (int)(k & 1), r = (int)(k % kRing);
  ParitySet &p = s->par[b], &q = s->par[b ^ 1];
  StepEvents& ev = s->ev[r];
  const ryk_session_config& c = s->cfg;
  const int pe = s->e_enc_frames;
  Stage2Lane& lane = s2_lane(s, b);
  cudaStream_t sC2 = lane.stream;

  // ================= stream E: wave slides =================
  if (d_chunk_user) RYK_CUDA(cudaMemcpyAsync(s->input[kMic].d_fixed, d_chunk_user, sizeof(float) * s->n_in, cudaMemcpyDeviceToDevice, s->sE));
  if (k >= 2) {
    RYK_CUDA(cudaStreamWaitEvent(s->sE, s->ev[(k - 2) % kRing].cslide, 0));  // q.cw_wave: last read by the silence gate in the head of stage 1 of k-2
    RYK_CUDA(cudaStreamWaitEvent(s->sE, s->ev[(k - 2) % kRing].enc, 0));     // q.wave_win: last read by the analysis of k-2
  }
  if (host_block_sync(s->dn_params, s->dn.params, k, ev.gate, s->sE)) return -1;
  if (host_block_sync(s->aec_params, s->aec.params, k, ev.gate, s->sE)) return -1;
  if (host_block_sync(s->agc_params, s->agcw.params, k, ev.gate, s->sE)) return -1;
  if (s->echo && far_sync(s, k)) return -1;
  if (stage_time(s, 0, 0, r, s->sE)) return -1;
  if (run_graph(e, p.graphs.gate, s->sE, [&]() -> int {
        const float *chunk = nullptr, *far = nullptr;
        if (input_to_model(e, s, b, kMic, &chunk)) return -1;
        if (s->echo && input_to_model(e, s, b, kFar, &far)) return -1;
        if (s->denoise || s->echo) {  // the frame stage in front of the wave slide: echo cancellation, then noise suppression
          const DenoiseWork& w = s->dn;
          const InputState &pm = p.input[kMic], &qm = q.input[kMic], &pf = p.input[kFar], &qf = q.input[kFar];
          if (denoise_forward(e, w.max_frames, pm.dn, qm.dn, chunk, s->n_wave, w.spec, s->sE)) return -1;
          if (s->echo) {
            if (denoise_forward(e, w.max_frames, pf.dn, qf.dn, far, s->n_wave, s->aec.far_spec, s->sE)) return -1;
            if (echo_scan(s->aec, pm.dn, s->n_wave, w.spec, s->sE)) return -1;
          }
          if (s->denoise && denoise_scan(w, pm.dn, qm.dn, s->n_wave, s->sE)) return -1;
          if (denoise_inverse(e, w, pm.dn, qm.dn, s->n_wave, s->d_chunk_dn, s->sE)) return -1;
          chunk = s->d_chunk_dn;
        }
        if (s->agc) {                 // the gain control after the frame stage: a varying gain there would look like a moving echo path
          if (agc_run(s->agcw, p.agc, q.agc, chunk, s->n_wave, s->d_chunk_agc, s->sE)) return -1;
          chunk = s->d_chunk_agc;
        }
        if (slide<float>(p.wave_win, chunk, q.wave_win, s->Lw, s->n_wave, 1, s->sE)) return -1;
        return slide<float>(p.cw_wave, q.wave_win + (size_t)pe * s->hop, q.cw_wave, (size_t)s->Tw * s->hop, (size_t)s->n_feat * s->hop, 1, s->sE);
      })) return -1;
  if (stage_time(s, 0, 1, r, s->sE)) return -1;
  RYK_CUDA(cudaEventRecord(ev.gate, s->sE));

  // ================= stream A of par[b]: WORLD analysis (the chunks of one parity share a plan and a stream) =================
  cudaStream_t sA = p.sA;
  RYK_CUDA(cudaStreamWaitEvent(sA, ev.gate, 0));
  if (k >= 2) RYK_CUDA(cudaStreamWaitEvent(sA, s->ev[(k - 2) % kRing].cslide, 0));   // p.enc_* consumed by stage 1 of k-2
  if (stage_time(s, 1, 0, r, sA)) return -1;
  if (run_graph(e, p.graphs.analysis, sA, [&]() -> int {
        const double* d_f0 = nullptr;
        if (p.crepe) {
          if (crepe_plan_run(e, p.crepe, q.wave_win, sA)) return -1;
          d_f0 = crepe_plan_f0(p.crepe);
        } else {
          if (dio_stonemask_run(e, p.dio, q.wave_win, sA)) return -1;
          d_f0 = dio_plan_f0(p.dio);
        }
        const int n_enc = s->Lw / s->hop;
        return spectral_analysis_run(e, q.wave_win, s->Lw, c.fs, c.frame_period_ms, d_f0, n_enc, c.fft_length, c.order, s->sptk.d_G,
                                     p.enc_sp, p.enc_ap, p.enc_mc, p.enc_f0, p.enc_voiced, sA, s->sA_side);
      })) return -1;
  if (stage_time(s, 1, 1, r, sA)) return -1;
  RYK_CUDA(cudaEventRecord(ev.enc, sA));

  // ================= stream C: stage 1 (head: feature slides + silence gate; then U-Net, f0 map, mc2sp) =================
  // the mask / index / count of par[b] are written by the head and read by the SWITCH graph, both on stream C: no guard between steps
  // needed (nor for the f0 map: the host's copy, the measuring kernel in the head and the epilogue in the SWITCH graph are all on
  // stream C; the copy goes before the head so that it cannot overwrite what this step's measurement writes in follow mode)
  if (s->f0_reset) RYK_CUDA(cudaMemsetAsync(s->d_f0_stats, 0, sizeof(F0Stats), s->sC));
  s->f0_reset = false;
  if (host_block_sync(s->f0_map, s->d_f0_map, k, ev.cslide, s->sC)) return -1;
  RYK_CUDA(cudaStreamWaitEvent(s->sC, ev.enc, 0));                             // (the analysis of step k waited for its wave slides)
  if (stage_time(s, 2, 0, r, s->sC)) return -1;
  if (run_graph(e, p.graphs.s1_head, s->sC, [&]() -> int { return stage1_head(e, s, b); })) return -1;
  // the next chunks of this parity wait only for the head, so stage 1's U-Net is off the gate -> analysis -> stage 1 recurrence
  RYK_CUDA(cudaEventRecord(ev.cslide, s->sC));
  // three hand-off slots: stage 1 rewrites what step k-3 handed on, so it runs beside stage 2 of k-2 (and k-1)
  if (k >= kHandoff) {
    RYK_CUDA(cudaStreamWaitEvent(s->sC, s->ev[(k - 3) % kRing].dslide, 0));   // ho[h].{f0,ap}_out consumed by decode k-3
    RYK_CUDA(cudaStreamWaitEvent(s->sC, s->ev[(k - 3) % kRing].conv, 0));     // ho[h].sp_mid consumed by stage 2 of k-3
  }
  if (stage_graph_launch(e, s->hgraphs[k % kHandoffGraphs].s1, s->sC)) return -1;   // counts the setter; k_set_bucket counts the body
  if (stage_time(s, 2, 1, r, s->sC)) return -1;
  RYK_CUDA(cudaEventRecord(ev.s1, s->sC));

  // ================= stage 2 lane: stage-2 prologue =================
  RYK_CUDA(cudaStreamWaitEvent(sC2, ev.s1, 0));
  if (k >= kHandoff) RYK_CUDA(cudaStreamWaitEvent(sC2, s->ev[(k - 3) % kRing].dslide, 0));  // ho[h].sp_out consumed by decode k-3
  if (stage_time(s, 3, 0, r, sC2)) return -1;
  if (s->group) {
    Group* G = s->group;
    if (G->step >= 1) RYK_CUDA(cudaStreamWaitEvent(sC2, G->ev_fwd[(G->step - 1) % kRing], 0));   // batched input read by forward k-1
    float* dst = (float*)G->p2->d_in + (size_t)s->slot * s->Tp * 512;
    if (run_handoff_graph(e, s, k, &HandoffGraphs::s2_pro, sC2, [&](int h) -> int {
          return sr_prologue_run(e, s->ho[h].sp_mid, s->Tw, s->Tp, s->nb, dst, sC2, lane.d_colmin);
        })) return -1;
    RYK_CUDA(cudaEventRecord(ev.pro, sC2));
  } else {
    UNetPlan* p2 = nullptr;
    if (s2_plan(e, s, lane, &p2)) return -1;
    if (run_handoff_graph(e, s, k, &HandoffGraphs::s2_pro, sC2, [&](int h) -> int {
          if (sr_prologue_run(e, s->ho[h].sp_mid, s->Tw, s->Tp, s->nb, (float*)p2->d_in, sC2, lane.d_colmin)) return -1;
          return unet_forward(e, p2, sC2, 0, 0);
        })) return -1;
  }
  return 0;
}

// single session: stage-2 layers 1..14 (the wgmma layers) on the session's own lane
static int session_mid_single(Engine* e, Session* s) {
  Stage2Lane& lane = s2_lane(s, (int)(s->step & 1));
  UNetPlan* p2 = nullptr;
  if (s2_plan(e, s, lane, &p2)) return -1;
  cudaEvent_t pe0 = nullptr, pe1 = nullptr;
  if (e->profile) { RYK_CUDA(cudaEventCreate(&pe0)); RYK_CUDA(cudaEventCreate(&pe1)); RYK_CUDA(cudaEventRecord(pe0, lane.stream)); }
  if (run_graph(e, lane.s2_layers, lane.stream, [&]() -> int { return unet_forward(e, p2, lane.stream, 1, 14); })) return -1;
  if (e->profile) { RYK_CUDA(cudaEventRecord(pe1, lane.stream)); e->prof_events.emplace_back(pe0, pe1); }
  return 0;
}

// the samples a step of parity b returns and their count: the synthesizer's blocks, or their device-rate resampling (synth_out), or
// with the output limiter its output for them
static double* synth_out(Session* s, int b) { return s->out.rate ? s->par[b].d_rout_fixed : s->par[b].d_out_fixed; }
static double* step_out(Session* s, int b) { return s->limiter ? s->par[b].d_lim_out : synth_out(s, b); }
static int* step_n_out(Session* s, int b) { return s->out.rate ? s->par[b].d_rn_fixed : s->par[b].d_n_fixed; }

static int session_back(Engine* e, Session* s) {
  const long long k = s->step;
  const int b = (int)(k & 1), r = (int)(k % kRing);
  ParitySet &p = s->par[b], &q = s->par[b ^ 1];
  StepEvents& ev = s->ev[r];
  const ryk_session_config& c = s->cfg;
  const int pc = s->e_conv;
  Stage2Lane& lane = s2_lane(s, b);
  cudaStream_t sC2 = lane.stream;
  if (s->group) {
    Group* G = s->group;
    RYK_CUDA(cudaStreamWaitEvent(sC2, G->ev_fwd[G->step % kRing], 0));
    const float* src = (const float*)G->p2->d_out + (size_t)s->slot * s->Tp * 512;
    if (run_handoff_graph(e, s, k, &HandoffGraphs::s2_epi, sC2, [&](int h) -> int {
          return sr_epilogue_run(e, src, s->Tw, s->nb, s->ho[h].sp_out, sC2, pc, pc + s->n_feat, 1.0, s->ho[h].formant);
        })) return -1;
  } else {
    UNetPlan* p2 = nullptr;
    if (s2_plan(e, s, lane, &p2)) return -1;
    if (run_handoff_graph(e, s, k, &HandoffGraphs::s2_epi, sC2, [&](int h) -> int {
          if (unet_forward(e, p2, sC2, 15, 15)) return -1;
          return sr_epilogue_run(e, (const float*)p2->d_out, s->Tw, s->nb, s->ho[h].sp_out, sC2, pc, pc + s->n_feat, 1.0, s->ho[h].formant);
        })) return -1;
  }
  if (stage_time(s, 3, 1, r, sC2)) return -1;
  RYK_CUDA(cudaEventRecord(ev.conv, sC2));

  // ================= stream D: realtime synthesizer =================
  RYK_CUDA(cudaStreamWaitEvent(s->sD, ev.conv, 0));
  if (stage_time(s, 4, 0, r, s->sD)) return -1;
  if (synth_host_advance(e, s->synth, s->Td, s->sD)) return -1;
  const int max_blocks = s->max_blocks;
  // the limiter's settings: its pinned slot was last read by a copy of step k - kRing, ahead of that step's decode slides
  if (host_block_sync(s->lim_params, s->lim.params, k, ev.dslide, s->sD)) return -1;
  if (run_handoff_graph(e, s, k, &HandoffGraphs::dec_slide, s->sD, [&](int h) -> int {
        const HandoffSlot& o = s->ho[h];
        SlideBatch sb; sb.n = 0;
        slide_add<float>(sb, p.dw_f0, o.f0_out + pc, q.dw_f0, s->Td, s->n_feat, 1);
        slide_add<float>(sb, p.dw_ap, o.ap_out + (size_t)pc * s->nb, q.dw_ap, s->Td, s->n_feat, s->nb);
        slide_add<float>(sb, p.dw_sp, o.sp_out + (size_t)pc * s->nb, q.dw_sp, s->Td, s->n_feat, s->nb);
        if (slide_batch(sb, s->sD)) return -1;
        k_f32_to_f64<<<(s->Td + 127) / 128, 128, 0, s->sD>>>(q.dw_f0, s->dec_f0_f64, s->Td);
        RYK_CUDA(cudaGetLastError());
        return 0;
      })) return -1;
  // the converted features of this hand-off slot are free again as soon as they sit in the decode window
  RYK_CUDA(cudaEventRecord(ev.dslide, s->sD));
  if (run_graph(e, p.graphs.synth, s->sD, [&]() -> int {
        if (synth_add_kernel(e, s->synth, s->dec_f0_f64, s->Td, q.dw_sp, q.dw_ap, s->sD)) return -1;
        if (synth_drain_async(e, s->synth, p.d_out_fixed, max_blocks, s->sD)) return -1;
        k_scrub<<<8, 256, 0, s->sD>>>(p.d_out_fixed, s->synth->dev.state, c.vocoder_buffer_size, max_blocks * c.vocoder_buffer_size, p.d_n_fixed);
        RYK_CUDA(cudaGetLastError());
        // fs -> device rate: the outputs whose filter support the synthesizer has produced; the rest waits for the next step
        if (s->out.rate &&
            resample_stream_out_run(e, p.out_hist, q.out_hist, s->out.hist, p.d_out_fixed, p.d_n_fixed, s->out.up, s->out.down,
                                    s->out.d_h, s->out.n_taps, p.out_st, q.out_st, p.d_rout_fixed, s->max_out, p.d_rn_fixed, s->sD))
          return -1;
        if (!s->limiter) return 0;
        // the limiter last, at the output rate: it changes no upstream state
        return limiter_run(s->lim, p.lim, q.lim, synth_out(s, b), step_n_out(s, b), p.d_lim_out, s->sD);
      })) return -1;
  if (stage_time(s, 4, 1, r, s->sD)) return -1;
  // the step's HostSlot::dec is recorded by stage_out after the copies it appends to stream D
  s->step++;
  return 0;
}

static int session_enqueue(Engine* e, Session* s, const float* d_chunk_user) {
  int rc = session_front(e, s, d_chunk_user);
  if (!rc) rc = session_mid_single(e, s);
  if (!rc) rc = session_back(e, s);
  return rc;
}

// One step of every member + the batched stage-2 forward between their front and back halves.  d_chunks: one device chunk per
// member, or nullptr when stage_in staged every member's chunk.
static int group_enqueue(Engine* e, Group* G, const float* const* d_chunks) {
  const int r = (int)(G->step % kRing);
  for (size_t i = 0; i < G->members.size(); ++i)
    if (session_front(e, G->members[i], d_chunks ? d_chunks[i] : nullptr)) return -1;
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

// ---- host-API staging shared by sessions and groups ----
// The host slot of the caller's ticket: the session's own step alone, the group's step for a member.
static HostSlot& host_slot(Session* s, long long ticket) { return s->io[ticket % kRing]; }

// host chunk -> pinned slot -> input[kMic].d_fixed on stream E, in front of the step's wave slides
static int stage_in(Session* s, HostSlot& io, const float* wave) {
  memcpy(io.h_in, wave, sizeof(float) * s->n_in);
  RYK_CUDA(cudaMemcpyAsync(s->input[kMic].d_fixed, io.h_in, sizeof(float) * s->n_in, cudaMemcpyHostToDevice, s->sE));
  return 0;
}

// after a step of s was enqueued: copy its samples and sample count to out / n_out (kind: to the host slot or to device buffers) behind
// the decode stream and record io.dec.  The output buffers are those of the parity of the session's own step, which differs from the
// group's for a member that joined at a group step of the other parity.
static int stage_out(Session* s, HostSlot& io, double* out, int* n_out, cudaMemcpyKind kind) {
  const int b = (int)((s->step - 1) & 1);
  RYK_CUDA(cudaMemcpyAsync(n_out, step_n_out(s, b), sizeof(int), kind, s->sD));
  RYK_CUDA(cudaMemcpyAsync(out, step_out(s, b), sizeof(double) * s->max_out, kind, s->sD));
  RYK_CUDA(cudaEventRecord(io.dec, s->sD));
  return 0;
}

// wait for the step staged in io and copy its samples out of the host slot
static int collect_out(Session* s, HostSlot& io, double* out, int out_capacity, int* n_out) {
  RYK_CUDA(cudaEventSynchronize(io.dec));
  const int produced = *io.h_n;
  RYK_CHECK(produced <= out_capacity, "output buffer too small for the produced blocks");
  memcpy(out, io.h_out, sizeof(double) * produced);
  *n_out = produced;
  s->collected++;
  return 0;
}

// the checks the submit and push entry points of sessions and groups share
static int check_chunk(const Session* s, int n) { RYK_CHECK(n == s->n_in, "chunk length must be round(rate * buffer_time) at the session's input rate"); return 0; }
static int check_in_flight(long long in_flight) { RYK_CHECK(in_flight < kRing - 2, "too many chunks in flight: collect before submitting more"); return 0; }
static int check_out_capacity(const Session* s, int out_capacity) {
  RYK_CHECK(out_capacity >= s->max_out, "out_capacity must hold the most samples a step returns (ryk_session_io_geometry max_out)");
  return 0;
}

int session_last_output(Engine* e, int id, const double** out, const int** n_out, int* max_out, cudaStream_t* sD) {
  Session* s = get_session(e, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(s->step > 0, "the session has not processed a chunk yet");
  const int b = (int)((s->step - 1) & 1);
  *out = step_out(s, b); *n_out = step_n_out(s, b); *max_out = s->max_out; *sD = s->sD;
  return 0;
}

}  // namespace ryk

using namespace ryk;
struct ryk_engine { Engine impl; };

extern "C" {

static int session_build(Engine* e, Session* s, const ryk_session_config* cfg, int f0_method);

// The one way a session is made (ryk_session_create_voice, ryk_session_restore): f0_method is the engine's, or the one a snapshot records.
static int session_create(Engine* e, const ryk_session_config* cfg, int voice_id, int f0_method, int* session_id) {
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
  if (session_build(e, s, cfg, f0_method)) { session_free(s); return -1; }     // frees whatever the build made; ryk_last_error keeps the cause
  v->users++;
  e->sessions.push_back(s);
  *session_id = (int)e->sessions.size() - 1;
  return 0;
}

int ryk_session_create_voice(ryk_engine* h, const ryk_session_config* cfg, int voice_id, int* session_id) {
  return session_create(&h->impl, cfg, voice_id, h->impl.f0_method, session_id);
}

int ryk_session_create(ryk_engine* h, const ryk_session_config* cfg, int* session_id) { return ryk_session_create_voice(h, cfg, 0, session_id); }

int ryk_session_voice(ryk_engine* h, int id) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  return s->voice_id;
}

// Everything a session allocates and captures; on failure the caller frees the partly built session.
static int session_build(Engine* e, Session* s, const ryk_session_config* cfg, int f0_method) {
  s->cfg = *cfg;
  // the stream's times become frame counts at 1000 / frame_period frames per second; any other period rounds that rate, and the
  // frame counts drift from the samples they stand for (6 ms: 167 or 166 frames a second for the true 166.67)
  const double frames_per_second = 1000.0 / cfg->frame_period_ms;
  RYK_CHECK(cfg->frame_period_ms > 0 && frames_per_second == floor(frames_per_second),
            "the frame period must divide 1000 ms into a whole number of frames per second, such as 1, 2, 4, 5, 8 or 10 ms");
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
  // the stage-1 SWITCH has a body per padded-length bucket 0 .. Tp / 128 (BucketKernels holds 16): Tw <= 1919
  RYK_CHECK(s->Tp / 128 + 1 <= 16, "window too long for the stage-1 graph table");
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
  for (ParitySet& p : s->par) RYK_CUDA(cudaStreamCreateWithPriority(&p.sA, cudaStreamNonBlocking, prio_hi));
  RYK_CUDA(cudaStreamCreateWithPriority(&s->sA_side, cudaStreamNonBlocking, prio_hi));
  RYK_CUDA(cudaStreamCreateWithPriority(&s->sC, cudaStreamNonBlocking, prio_hi));
  for (Stage2Lane& L : s->lane) RYK_CUDA(cudaStreamCreateWithPriority(&L.stream, cudaStreamNonBlocking, prio_lo));
  RYK_CUDA(cudaStreamCreateWithPriority(&s->sD, cudaStreamNonBlocking, prio_hi));
  { const char* v = getenv("RYK_STAGE_TIMES"); s->stage_times = v && atoi(v) != 0; }
  // the template fill below (k_fill_rows on e->stream) runs after the zero-fills (on e->stream too): a legacy-default-stream memset
  // is not ordered before it (seen once as a 4e-3 RMSE mismatch)
  BufferSet& m = s->mem;
  m.stream = e->stream;
  for (StepEvents& ev : s->ev) {
    for (cudaEvent_t* p : ev.all()) RYK_CUDA(cudaEventCreateWithFlags(p, cudaEventDisableTiming));
    if (s->stage_times) for (auto& pair : ev.tev) for (cudaEvent_t& t : pair) RYK_CUDA(cudaEventCreate(&t));
  }
  for (HostSlot& io : s->io) RYK_CUDA(cudaEventCreateWithFlags(&io.dec, cudaEventDisableTiming));
  s->max_blocks = (s->Td * s->hop) / cfg->vocoder_buffer_size + 4;
  s->max_out = s->max_blocks * cfg->vocoder_buffer_size;
  const size_t n_enc = s->Lw / s->hop, Tw = s->Tw, Td = s->Td, nb = s->nb, C = s->C;
  for (ParitySet& p : s->par) {
    if (m.device(&p.wave_win, s->Lw) || m.device(&p.cw_f0, Tw) || m.device(&p.cw_ap, Tw * nb) || m.device(&p.cw_mc, Tw * C) ||
        m.device(&p.cw_voiced, Tw) || m.device(&p.cw_wave, Tw * s->hop) || m.device(&p.dw_f0, Td) || m.device(&p.dw_ap, Td * nb) ||
        m.device(&p.dw_sp, Td * nb)) return -1;
    // silent template mel-cepstrum in the not-yet-filled part of the convert window
    k_fill_rows<float><<<64, 256, 0, e->stream>>>(p.cw_mc, s->Tw, s->C, kSilentMc0, 0.f);
    if (m.device(&p.enc_f0, n_enc) || m.device(&p.enc_sp, n_enc * nb) || m.device(&p.enc_ap, n_enc * nb) || m.device(&p.enc_mc, n_enc * C) ||
        m.device(&p.enc_voiced, n_enc) || m.device(&p.d_mask, Tw) || m.device(&p.d_index, Tw) || m.device(&p.d_count, 2) ||
        m.device(&p.d_out_fixed, s->max_out) || m.device(&p.d_n_fixed, 1)) return -1;
  }
  for (HandoffSlot& o : s->ho)
    if (m.device(&o.mc_out, Tw * C) || m.device(&o.f0_out, Tw) || m.device(&o.ap_out, Tw * nb) || m.device(&o.sp_out, Tw * nb) ||
        m.device(&o.voiced_out, Tw) || m.device(&o.sp_mid, Tw * nb) || m.device(&o.formant, 1)) return -1;
  for (Stage2Lane& L : s->lane) if (m.device(&L.d_colmin, kColminFloats)) return -1;
  if (m.device(&s->d_mse, Tw) || m.device(&s->dec_f0_f64, Td) || input_alloc(s, kMic, s->n_in, false)) return -1;
  // the session starts on its voice's f0 map and an unwarped envelope
  if (m.device(&s->d_f0_map, 1) || m.device(&s->d_f0_stats, 1) || m.pinned(&s->f0_map.ring, kRing)) return -1;
  s->f0_map.next = voice_f0_map(s->voice);
  s->f0_map.next.formant = 1.0;
  s->f0_map.dirty = true;
  for (HostSlot& io : s->io) if (m.pinned(&io.h_in, s->n_wave) || m.pinned(&io.h_out, s->max_out) || m.pinned(&io.h_n, 1)) return -1;
  // f0 method 2: each step's encode window is analysed on its own, like one crepe.predict call per fetched window (DESIGN.md C3)
  for (ParitySet& p : s->par) {
    const int rc = f0_method == 2 ? crepe_plan_create(e, s->Lw, cfg->fs, cfg->frame_period_ms, &p.crepe)
                                  : dio_plan_create(e, s->Lw, cfg->fs, cfg->frame_period_ms, cfg->f0_floor, cfg->f0_ceil, &p.dio, f0_method);
    if (rc) return -1;
  }
  if (synth_create(e, cfg->fs, cfg->frame_period_ms, cheaptrick_fft_size(cfg->fs, 71.0), cfg->vocoder_buffer_size, 4096, &s->synth)) return -1;
  // build the U-Net plans this session can need up front (allocation + tensor maps), not on the first chunk
  UNetPlan* p = nullptr;
  s->s1_owner = ++e->plan_owners;
  for (Stage2Lane& L : s->lane) L.owner = ++e->plan_owners;
  for (int Tp = 128; Tp <= s->Tp; Tp += 128) if (unet_get_plan(e, s->voice->stage1, 1, 1, Tp, e->precision, &p, s->s1_owner)) return -1;
  // (the stage-2 plans are created on first use: a session that joins a group never needs its own)
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  RYK_CUDA(cudaDeviceSynchronize());
  s->precision = e->precision; s->s1_fused = e->s1_fused;
  for (int j = 0; j < kHandoffGraphs; ++j) if (stage1_build_switch(e, s, s->voice, s->s1_owner, j, s->hgraphs[j].s1)) return -1;
  return 0;
}

int ryk_session_destroy(ryk_engine* h, int id) {
  Engine* e = &h->impl;
  Session* s = get_session(e, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(s->group == nullptr, "session belongs to a group: destroy the group first");
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  s->voice->users--;
  session_free(s);                         // synchronises the session's streams
  e->sessions[id] = nullptr;
  return 0;
}

// Queue one chunk (host samples) without waiting for its output; *ticket identifies it for ryk_session_collect.
int ryk_session_submit(ryk_engine* h, int id, const float* wave, int n, long long* ticket) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = get_session(e, id);
  RYK_CHECK(s != nullptr, "no such session");
  if (int rc = check_chunk(s, n)) return rc;
  RYK_CHECK(s->group == nullptr, "session belongs to a group: use ryk_group_submit");
  if (int rc = check_in_flight(s->step - s->collected)) return rc;
  const long long k = s->step;
  HostSlot& io = host_slot(s, k);
  if (stage_in(s, io, wave)) return -1;
  if (session_enqueue(e, s, nullptr)) return -1;
  if (stage_out(s, io, io.h_out, io.h_n, cudaMemcpyDeviceToHost)) return -1;
  if (ticket) *ticket = k;
  return 0;
}

// Wait for the chunk `ticket` (tickets must be collected in order) and copy its samples out.
int ryk_session_collect(ryk_engine* h, int id, long long ticket, double* out, int out_capacity, int* n_out) {
  Engine* e = &h->impl;
  Session* s = get_session(e, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(ticket == s->collected && ticket < s->step, "tickets are collected in submission order");
  return collect_out(s, host_slot(s, ticket), out, out_capacity, n_out);
}

// Non-blocking completion query (cudaEventQuery of the step's last decode-stream event): *done = 1 when ryk_session_collect would
// not wait.  This is what queue_output_wave.get_nowait() needs (run.py:176-182).
int ryk_session_poll(ryk_engine* h, int id, long long ticket, int* done) {
  Engine* e = &h->impl;
  Session* s = get_session(e, id);
  RYK_CHECK(s != nullptr && done != nullptr, "no such session");
  RYK_CHECK(ticket >= 0 && ticket < s->step && ticket + kRing > s->step, "ticket is not among the last 8 steps");
  cudaError_t q = cudaEventQuery(host_slot(s, ticket).dec);
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
  RYK_CHECK(wave_dev != nullptr, "null argument");
  if (int rc = check_chunk(s, n)) return rc;
  RYK_CHECK(s->group == nullptr, "session belongs to a group: use ryk_group_push_device");
  if (int rc = check_out_capacity(s, out_capacity)) return rc;
  HostSlot& io = host_slot(s, s->step);
  if (session_enqueue(e, s, wave_dev)) return -1;
  if (stage_out(s, io, out_dev, n_out_dev, cudaMemcpyDeviceToDevice)) return -1;
  s->collected = s->step;         // device-resident steps are not collected through the host API
  return 0;
}

// (Re)allocates the output limiter at the session's output rate and max_out (DECIDE L1): its shape, scratch, meter and settings block,
// and each parity's history, position and output.  The settings block starts as zeros, so the next submitted step copies the settings.
static int limiter_alloc(Session* s) {
  BufferSet& m = s->mem;
  LimWork& w = s->lim;
  limiter_shape(s->out.rate ? s->out.rate : s->cfg.fs, s->lim_lookahead_ms, s->lim_hold_ms, &w.L, &w.R);
  w.max_n = s->max_out;
  size_t n_g0, n_t32, n_t1k, n_m;
  limiter_scratch_sizes(w, &n_g0, &n_t32, &n_t1k, &n_m);
  if (m.device(&w.params, 1) || m.device(&w.meter, 1) || m.device(&w.g0, n_g0) || m.device(&w.t32, n_t32) || m.device(&w.t1k, n_t1k) ||
      m.device(&w.m, n_m))
    return -1;
  for (ParitySet& p : s->par)
    if (m.device(&p.lim.g0, (size_t)w.R + 2 * w.L - 1) || m.device(&p.lim.y, w.L) || m.device(&p.lim.st, 1) ||
        m.device(&p.d_lim_out, s->max_out))
      return -1;
  s->lim_params.dirty = true;
  return 0;
}

// ---- device rates: the session takes chunks at in.rate and returns samples at out.rate, converting on its own streams ----
// Geometry (DESIGN.md §4, DECIDE R1), with half = (n_taps - 1) / 2 and up / down = the resampler's output rate / input rate:
//   input:  delay_in = half / down model samples, the smallest delay for which every sample of a step's model-rate chunk has its whole
//           filter support in the chunks received; the history window holds the chunk and the ceil((delay_in * down + half) / up)
//           samples before it.
//   output: a step emits the outputs whose support ends inside the synthesizer samples so far; the kept history covers the left
//           support of the first output not yet emitted, and max_out bounds one step's count.
static int session_set_rate(Engine* e, int id, bool input, int rate, int up, int down, const double* taps, int n_taps) {
  RYK_CUDA(cudaSetDevice(e->device));
  const char* refusal = "device rates can only be set on a fresh session (no chunk pushed, not in a group)";
  Session* s = fresh_session(e, id, refusal);
  if (!s) return -2;
  RYK_CHECK(s->group == nullptr, refusal);
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
  BufferSet& m = s->mem;
  if (input) {
    const int n_in = (int)lrint(s->cfg.buffer_time * rate);
    RYK_CHECK((long long)n_in * up == (long long)s->n_wave * down,
              "the chunk at this device rate is not a whole number of samples: round(rate * buffer_time) * up != round(fs * buffer_time) * down");
    const int delay = half / down;
    side.hist = n_in + (delay * down + half + up - 1) / up;
    for (int i = 0; i < kInputs; ++i) if (s->input[i].d_fixed && input_alloc(s, i, n_in, true)) return -1;
    for (HostSlot& io : s->io) if (m.pinned(&io.h_in, n_in)) return -1;
  } else {
    const long long blocks = (long long)s->max_blocks * s->cfg.vocoder_buffer_size;
    const int max_out = (int)((blocks * up + down - 1) / down);
    side.hist = (2 * half + down + up - 1) / up + 1;
    for (ParitySet& p : s->par)
      if (m.device(&p.out_hist, side.hist) || m.device(&p.out_st, 1) || m.device(&p.d_rout_fixed, max_out) || m.device(&p.d_rn_fixed, 1))
        return -1;
    for (HostSlot& io : s->io) if (m.pinned(&io.h_out, max_out)) return -1;
  }
  if (m.device(&side.d_h, n_taps)) return -1;
  RYK_CUDA(cudaMemcpyAsync(side.d_h, taps, sizeof(double) * n_taps, cudaMemcpyHostToDevice, e->stream));
  RYK_CUDA(cudaStreamSynchronize(e->stream));      // the zero-fills and the taps: the session's streams do not wait for the engine stream
  side.rate = rate; side.up = up; side.down = down; side.n_taps = n_taps;
  if (input) {
    s->n_in = (int)lrint(s->cfg.buffer_time * rate);
    s->delay_in = half / down;
  } else {
    s->max_out = (int)(((long long)s->max_blocks * s->cfg.vocoder_buffer_size * up + down - 1) / down);
    if (s->limiter) {                               // the limiter's L, R and buffers at the new rate and max_out
      if (limiter_alloc(s)) return -1;
      RYK_CUDA(cudaStreamSynchronize(e->stream));
    }
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
  if (delay_in) *delay_in = s->delay_in + (s->denoise || s->echo ? kDnDelay : 0);
  if (in_rate) *in_rate = s->in.rate ? s->in.rate : s->cfg.fs;
  if (out_rate) *out_rate = s->out.rate ? s->out.rate : s->cfg.fs;
  return 0;
}

// ---- the session's f0 map and the statistics of its speaker (DESIGN.md §4a) ----
// These calls change host state only; host_block_sync carries it to the device at the next submitted step, alone or in a group.
int ryk_session_get_f0_map(ryk_engine* h, int id, ryk_f0_map* map) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(map != nullptr, "null argument");
  const F0Map& f = s->f0_map.next;
  map->in_mean = f.mu_in; map->in_std = f.sd_in; map->target_mean = f.mu_tgt; map->target_std = f.sd_tgt;
  return 0;
}

int ryk_session_set_f0_map(ryk_engine* h, int id, const ryk_f0_map* map) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(map != nullptr, "null argument");
  RYK_CHECK(isfinite(map->in_mean) && isfinite(map->in_std) && isfinite(map->target_mean) && isfinite(map->target_std),
            "the f0 map must be finite");
  RYK_CHECK(map->in_std > 0 && map->target_std > 0, "the standard deviations of the f0 map must be positive");
  F0Map& f = s->f0_map.next;
  f.mu_in = map->in_mean; f.sd_in = map->in_std; f.mu_tgt = map->target_mean; f.sd_tgt = map->target_std;
  f.has_stats = 1;
  s->f0_map.dirty = true;
  return 0;
}

int ryk_session_f0_measure(ryk_engine* h, int id, int enable) {
  Session* s = fresh_session(&h->impl, id, "f0 measurement can only be switched on a fresh session (no chunk pushed): the head of stage 1 is captured at the first steps");
  if (!s) return -2;
  RYK_CHECK(enable || !s->f0_map.next.follow, "the session follows its measurement: turn follow mode off first");
  s->f0_measure = enable != 0;
  return 0;
}

int ryk_session_f0_follow(ryk_engine* h, int id, int follow, int min_voiced_frames, double sd_floor) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  if (follow) {
    RYK_CHECK(s->f0_measure, "follow mode needs f0 measurement (ryk_session_f0_measure)");
    RYK_CHECK(s->f0_map.next.has_stats, "follow mode needs an f0 map: the voice has no f0 statistics and none were set on the session");
    RYK_CHECK(min_voiced_frames >= 1, "min_voiced_frames must be at least 1");
    RYK_CHECK(isfinite(sd_floor) && sd_floor > 0, "sd_floor must be finite and positive");
    s->f0_map.next.min_voiced = min_voiced_frames; s->f0_map.next.sd_floor = sd_floor;
  }
  s->f0_map.next.follow = follow != 0;
  s->f0_map.dirty = true;
  return 0;
}

int ryk_session_f0_measure_reset(ryk_engine* h, int id) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(s->f0_measure, "f0 measurement is not enabled for this session");
  s->f0_reset = true;
  s->f0_map.dirty = true;            // follow mode: back to the host's input side until min_voiced_frames are counted again
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

// The formant ratio travels in the f0 map block to stage 1 of the next submitted step, whose epilogue copies it into the step's hand-off
// slot for the stage-2 epilogue.
int ryk_session_set_formant(ryk_engine* h, int id, double ratio) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(isfinite(ratio) && ratio >= 0.5 && ratio <= 2.0, "the formant ratio must be finite and within [0.5, 2]");
  s->f0_map.next.formant = ratio;
  s->f0_map.dirty = true;
  return 0;
}

int ryk_session_get_formant(ryk_engine* h, int id, double* ratio) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(ratio != nullptr, "null argument");
  *ratio = s->f0_map.next.formant;
  return 0;
}

// ---- input noise suppression (DESIGN.md §4f) ----
// The setters change host state only; host_block_sync carries it to the device in front of the wave slides of the next submitted step.
static Session* denoise_session(Engine* e, int id) {
  Session* s = get_session(e, id);
  if (!s) set_error("no such session");
  else if (!s->denoise) set_error("noise suppression is not enabled for this session (ryk_session_denoise)");
  return s && s->denoise ? s : nullptr;
}

// The frame stage noise suppression and echo cancellation share (N1, E1): the microphone's transforms, overlap-add and stream state,
// allocated by whichever of the two is enabled first.  Step 0 reads par[0]: G_{-1} = 1.
static int frame_stage_alloc(Engine* e, Session* s) {
  if (s->dn.spec) return 0;
  BufferSet& m = s->mem;
  DenoiseWork& w = s->dn;
  w.max_frames = denoise_max_frames(s->n_wave);
  if (m.device(&w.spec, (size_t)kDnBins * w.max_frames) || m.device(&w.frames, (size_t)kDnN * w.max_frames) || m.device(&w.done, 1) ||
      m.device(&s->d_chunk_dn, s->n_wave))
    return -1;
  for (ParitySet& p : s->par) if (m.device(&p.input[kMic].dn, 1)) return -1;
  void* hp = nullptr;
  if (engine_pinned(e, sizeof(DenoiseState), &hp)) return -1;
  denoise_state_init((DenoiseState*)hp);
  RYK_CUDA(cudaMemcpyAsync(s->par[0].input[kMic].dn, hp, sizeof(DenoiseState), cudaMemcpyHostToDevice, e->stream));
  RYK_CUDA(cudaStreamSynchronize(e->stream));      // the staging is the engine's, and the session's streams do not wait for its stream
  return 0;
}

int ryk_session_denoise(ryk_engine* h, int id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = fresh_session(e, id, "noise suppression can only be enabled on a fresh session (no chunk pushed): the wave slides are captured at the first steps");
  if (!s) return -2;
  if (s->denoise) return 0;
  if (frame_stage_alloc(e, s)) return -1;
  BufferSet& m = s->mem;
  DenoiseWork& w = s->dn;
  if (m.device(&w.params, 1) || m.device(&w.learn, 1) || m.pinned(&s->dn_params.ring, kRing)) return -1;
  // the parameter block starts at 20 dB without a profile
  s->dn_params.next = {};
  s->dn_params.next.gain_floor = pow(10.0, -20.0 / 20.0);
  s->dn_params.dirty = true;
  RYK_CUDA(cudaStreamSynchronize(e->stream));      // the zero-fills: the session's streams do not wait for the engine stream
  s->denoise = true;
  return 0;
}

int ryk_session_set_denoise(ryk_engine* h, int id, double reduction_db) {
  Session* s = denoise_session(&h->impl, id);
  if (!s) return -2;
  if (int rc = denoise_check(reduction_db, nullptr)) return rc;
  s->dn_params.next.gain_floor = pow(10.0, -reduction_db / 20.0);
  s->dn_params.dirty = true;
  return 0;
}

int ryk_session_denoise_learn(ryk_engine* h, int id, long long n_frames) {
  Session* s = denoise_session(&h->impl, id);
  if (!s) return -2;
  RYK_CHECK(n_frames >= 1, "n_frames must be at least 1");
  DenoiseParams& P = s->dn_params.next;
  P.learn_serial++;
  P.learn_frames = n_frames;
  s->dn_params.dirty = true;
  return 0;
}

int ryk_session_set_noise_profile(ryk_engine* h, int id, const double* phi) {
  Session* s = denoise_session(&h->impl, id);
  if (!s) return -2;
  RYK_CHECK(phi != nullptr, "null argument");
  if (int rc = denoise_check(0.0, phi)) return rc;
  DenoiseParams& P = s->dn_params.next;
  memcpy(P.phi, phi, sizeof(double) * kDnBins);
  P.profile_serial++;
  P.learn_serial++;                                // cancels a learning in progress
  P.learn_frames = 0;
  s->dn_params.dirty = true;
  return 0;
}

int ryk_session_noise_profile(ryk_engine* h, int id, double* phi, long long* frames_left) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = denoise_session(e, id);
  if (!s) return -2;
  void* hp = nullptr;
  if (engine_pinned(e, sizeof(DenoiseLearn), &hp)) return -1;
  DenoiseLearn* L = (DenoiseLearn*)hp;
  RYK_CUDA(cudaMemcpyAsync(L, s->dn.learn, sizeof(DenoiseLearn), cudaMemcpyDeviceToHost, s->sE));
  RYK_CUDA(cudaStreamSynchronize(s->sE));          // behind the wave slides of every submitted step
  // requests not yet applied (not submitted yet: every submitted step's gain scan has run) are what the next step applies
  const DenoiseParams& P = s->dn_params.next;
  const bool new_profile = P.profile_serial != L->profile_serial, new_learn = P.learn_serial != L->learn_serial;
  if (phi) memcpy(phi, new_profile ? P.phi : L->phi, sizeof(double) * kDnBins);
  if (frames_left) *frames_left = new_learn ? P.learn_frames : L->remaining;
  return 0;
}

// ---- echo cancellation (DESIGN.md §4g) ----
// The setters change host state only; host_block_sync and far_sync carry it to the device in front of the wave slides of the next
// submitted step.
static Session* echo_session(Engine* e, int id) {
  Session* s = get_session(e, id);
  if (!s) set_error("no such session");
  else if (!s->echo) set_error("echo cancellation is not enabled for this session (ryk_session_echo_cancel)");
  return s && s->echo ? s : nullptr;
}

int ryk_session_echo_cancel(ryk_engine* h, int id, int taps, int delay_frames) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = fresh_session(e, id, "echo cancellation can only be enabled on a fresh session (no chunk pushed): the wave slides are captured at the first steps");
  if (!s) return -2;
  RYK_CHECK(!s->echo, "echo cancellation is already enabled for this session");
  if (int rc = echo_check(taps, delay_frames, 0.0)) return rc;
  if (frame_stage_alloc(e, s)) return -1;
  BufferSet& m = s->mem;
  EchoWork& a = s->aec;
  a.taps = taps; a.delay = delay_frames;
  if (m.device(&a.params, 1) || m.device(&a.filter, 1) || m.device(&a.ring, (size_t)kDnBins * (taps + delay_frames)) ||
      m.device(&a.far_spec, (size_t)kDnBins * s->dn.max_frames) || m.pinned(&s->aec_params.ring, kRing))
    return -1;
  for (ParitySet& p : s->par) if (m.device(&p.input[kFar].dn, 1)) return -1;     // zero: in_end 0, an empty history
  if (input_alloc(s, kFar, s->n_in, s->in.rate != 0)) return -1;
  // the filters start at zero; the residual suppression at 0 dB (gain 1)
  s->aec_params.next = {};
  s->aec_params.next.gain_floor = 1.0;
  s->aec_params.dirty = true;
  RYK_CUDA(cudaStreamSynchronize(e->stream));      // the zero-fills: the session's streams do not wait for the engine stream
  s->echo = true;
  return 0;
}

int ryk_session_echo_reference(ryk_engine* h, int id, const float* far, int n) {
  Session* s = echo_session(&h->impl, id);
  if (!s) return -2;
  RYK_CHECK(far != nullptr, "null argument");
  RYK_CHECK(n == s->n_in, "the far end of a step must be one chunk at the session's input rate (ryk_session_io_geometry n_in)");
  memcpy(s->far_next.data(), far, sizeof(float) * n);
  s->far_set = true;
  return 0;
}

int ryk_session_set_echo_suppression(ryk_engine* h, int id, double db) {
  Session* s = echo_session(&h->impl, id);
  if (!s) return -2;
  if (int rc = echo_check(1, 0, db)) return rc;
  s->aec_params.next.gain_floor = pow(10.0, -db / 20.0);
  s->aec_params.dirty = true;
  return 0;
}

int ryk_session_echo_stats(ryk_engine* h, int id, long long* frames, double* erle_db) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = echo_session(e, id);
  if (!s) return -2;
  void* hp = nullptr;
  if (engine_pinned(e, sizeof(EchoStats), &hp)) return -1;
  RYK_CUDA(cudaMemcpyAsync(hp, &s->aec.filter->stats, sizeof(EchoStats), cudaMemcpyDeviceToHost, s->sE));
  RYK_CUDA(cudaStreamSynchronize(s->sE));          // behind the wave slides of every submitted step
  const EchoStats* f = (const EchoStats*)hp;
  double sd = 0.0, sz = 0.0;
  for (int k = 0; k < kDnBins; ++k) { sd += f->sum_d[k]; sz += f->sum_z[k]; }
  if (frames) *frames = f->frames;
  if (erle_db) *erle_db = sd > 0.0 ? 10.0 * log10(sd / sz) : 0.0;
  return 0;
}

// ---- output limiter (DESIGN.md §4i) ----
// The setter changes host state only; host_block_sync carries it to the device in front of the decode slides of the next submitted step.
static Session* limiter_session(Engine* e, int id) {
  Session* s = get_session(e, id);
  if (!s) set_error("no such session");
  else if (!s->limiter) set_error("the output limiter is not enabled for this session (ryk_session_limiter)");
  return s && s->limiter ? s : nullptr;
}

int ryk_session_limiter(ryk_engine* h, int id, double lookahead_ms, double hold_ms) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = fresh_session(e, id, "the output limiter can only be enabled on a fresh session (no chunk pushed): the synthesis graphs are captured at the first steps");
  if (!s) return -2;
  RYK_CHECK(!s->limiter, "the output limiter is already enabled for this session");
  if (int rc = limiter_check_shape(lookahead_ms, hold_ms)) return rc;
  s->lim_lookahead_ms = lookahead_ms;
  s->lim_hold_ms = hold_ms;
  if (s->mem.pinned(&s->lim_params.ring, kRing) || limiter_alloc(s)) return -1;
  // the ceiling starts at -1 dB of the samples as returned (gain 1)
  s->lim_ceiling_db = -1.0;
  s->lim_params.next = limiter_params(-1.0, 1.0);
  RYK_CUDA(cudaStreamSynchronize(e->stream));      // the zero-fills: the session's streams do not wait for the engine stream
  s->limiter = true;
  return 0;
}

int ryk_session_set_limiter(ryk_engine* h, int id, double ceiling_db, double gain) {
  Session* s = limiter_session(&h->impl, id);
  if (!s) return -2;
  if (int rc = limiter_check_settings(ceiling_db, gain)) return rc;
  s->lim_ceiling_db = ceiling_db;
  s->lim_params.next = limiter_params(ceiling_db, gain);
  s->lim_params.dirty = true;
  return 0;
}

int ryk_session_get_limiter(ryk_engine* h, int id, double* ceiling_db, double* gain, int* lookahead, int* hold) {
  Session* s = limiter_session(&h->impl, id);
  if (!s) return -2;
  if (ceiling_db) *ceiling_db = s->lim_ceiling_db;
  if (gain) *gain = s->lim_params.next.gain;
  if (lookahead) *lookahead = s->lim.L;
  if (hold) *hold = s->lim.R;
  return 0;
}

int ryk_session_limiter_stats(ryk_engine* h, int id, double* reduction_db, long long* limited) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = limiter_session(e, id);
  if (!s) return -2;
  void* hp = nullptr;
  if (engine_pinned(e, sizeof(LimMeter), &hp)) return -1;
  RYK_CUDA(cudaMemcpyAsync(hp, s->lim.meter, sizeof(LimMeter), cudaMemcpyDeviceToHost, s->sD));
  RYK_CUDA(cudaStreamSynchronize(s->sD));          // behind the synthesis of every submitted step
  const LimMeter* mt = (const LimMeter*)hp;
  double g = 1.0;
  memcpy(&g, &mt->min_bits, sizeof(double));
  if (reduction_db) *reduction_db = mt->limited ? -20.0 * log10(g) : 0.0;
  if (limited) *limited = (long long)mt->limited;
  return 0;
}

// ---- automatic gain control (DESIGN.md §4j) ----
// The setter changes host state only; host_block_sync carries it to the device in front of the wave slides of the next submitted step.
static Session* agc_session(Engine* e, int id) {
  Session* s = get_session(e, id);
  if (!s) set_error("no such session");
  else if (!s->agc) set_error("the automatic gain control is not enabled for this session (ryk_session_agc)");
  return s && s->agc ? s : nullptr;
}

static void agc_set_next(Session* s, double target_db, double max_gain_db, double gate_db) {
  s->agc_db[0] = target_db; s->agc_db[1] = max_gain_db; s->agc_db[2] = gate_db;
  s->agc_params.next = agc_params(s->cfg.fs, target_db, max_gain_db, gate_db);
  s->agc_params.dirty = true;
}

// The AGC runs on the model-rate chunk, whose length n_wave no device rate changes: nothing here depends on ryk_session_set_input_rate.
int ryk_session_agc(ryk_engine* h, int id, double target_db, double max_gain_db, double gate_db) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = fresh_session(e, id, "the automatic gain control can only be enabled on a fresh session (no chunk pushed): the wave slides are captured at the first steps");
  if (!s) return -2;
  RYK_CHECK(!s->agc, "the automatic gain control is already enabled for this session");
  if (int rc = agc_check(target_db, max_gain_db, gate_db)) return rc;
  BufferSet& m = s->mem;
  AgcWork& w = s->agcw;
  if (m.device(&w.params, 1) || m.device(&w.meter, 1) || m.device(&s->d_chunk_agc, s->n_wave) || m.pinned(&s->agc_params.ring, kRing))
    return -1;
  for (ParitySet& p : s->par) if (m.device(&p.agc, 1)) return -1;
  // step 0 reads par[0]: position 0, gains 1, no level yet
  void* hp = nullptr;
  if (engine_pinned(e, sizeof(AgcState) + sizeof(AgcMeter), &hp)) return -1;
  AgcState* st = (AgcState*)hp;
  AgcMeter* mt = (AgcMeter*)(st + 1);
  agc_state_init(st);
  agc_meter_init(mt);
  RYK_CUDA(cudaMemcpyAsync(s->par[0].agc, st, sizeof(AgcState), cudaMemcpyHostToDevice, e->stream));
  RYK_CUDA(cudaMemcpyAsync(w.meter, mt, sizeof(AgcMeter), cudaMemcpyHostToDevice, e->stream));
  RYK_CUDA(cudaStreamSynchronize(e->stream));      // the staging is the engine's, and the session's streams do not wait for its stream
  agc_set_next(s, target_db, max_gain_db, gate_db);
  s->agc = true;
  return 0;
}

int ryk_session_set_agc(ryk_engine* h, int id, double target_db, double max_gain_db, double gate_db) {
  Session* s = agc_session(&h->impl, id);
  if (!s) return -2;
  if (int rc = agc_check(target_db, max_gain_db, gate_db)) return rc;
  agc_set_next(s, target_db, max_gain_db, gate_db);
  return 0;
}

int ryk_session_get_agc(ryk_engine* h, int id, double* target_db, double* max_gain_db, double* gate_db, double* linear) {
  Session* s = agc_session(&h->impl, id);
  if (!s) return -2;
  if (target_db) *target_db = s->agc_db[0];
  if (max_gain_db) *max_gain_db = s->agc_db[1];
  if (gate_db) *gate_db = s->agc_db[2];
  if (linear) {
    const AgcParams& P = s->agc_params.next;
    const double v[7] = {P.target, P.gate, P.gmax, P.ginv, P.a, P.s_up, P.s_dn};
    memcpy(linear, v, sizeof(v));
  }
  return 0;
}

int ryk_session_agc_stats(ryk_engine* h, int id, double* level_db, double* gain_db, int* active) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = agc_session(e, id);
  if (!s) return -2;
  void* hp = nullptr;
  if (engine_pinned(e, sizeof(AgcMeter), &hp)) return -1;
  RYK_CUDA(cudaMemcpyAsync(hp, s->agcw.meter, sizeof(AgcMeter), cudaMemcpyDeviceToHost, s->sE));
  RYK_CUDA(cudaStreamSynchronize(s->sE));          // behind the wave slides of every submitted step
  const AgcMeter* mt = (const AgcMeter*)hp;
  if (level_db) *level_db = mt->started ? 10.0 * log10(mt->level) : -HUGE_VAL;
  if (gain_db) *gain_db = 20.0 * log10(mt->gain);
  if (active) *active = mt->active;
  return 0;
}

// ---- groups: several sessions of one GPU sharing one batched stage-2 forward per step (BASELINE config 5) ----
static Group* get_group(Engine* e, int id) { return (id >= 0 && id < (int)e->groups.size()) ? e->groups[id] : nullptr; }

// Why a member's stream state survives a membership change.  A change runs only when none of the session's or the group's host-API
// steps is uncollected, and it synchronises the device before it frees or rebuilds anything, so no step of the old layout is in flight.
// The guards between steps are events of the member's own StepEvents ring, which a change keeps, and each lane's scratch stays ordered
// by the lane's stream.  The stage-2 plans a step uses are new after a change (the group's rebuilt plan, or the leaving member's own
// plans built by the change), and the group's waits on ev_fwd / pro / conv of steps before the change find completed events.

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
    if (m->group != G) lanes_release(m);
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
  for (const Stage2Lane& L : s->lane) {
    UNetPlan* p = nullptr;
    if (s2_plan(e, s, L, &p)) {
      lanes_release(s);
      return -1;
    }
  }
  if (group_rebuild(e, G, members)) {
    lanes_release(s);
    return -1;
  }
  s->group = nullptr; s->slot = 0;
  for (Stage2Lane& L : s->lane) L.s2_layers.reset();
  for (HandoffGraphs& hg : s->hgraphs) { hg.s2_pro.reset(); hg.s2_epi.reset(); }
  return 0;
}

// ---- voice switch (DESIGN.md §4a): the session converts into another voice from its next submitted step on ----
// What depends on the voice is rebuilt: the stage-1 plans and the six stage-1 SWITCH graphs that hold the voice's statistics, and the
// stage-2 plans (the lanes' own, or the group's batched plan through group_rebuild).  Everything that holds stream state carries over.
// Built first under fresh owner ids, then swapped in: a failure releases what was built and leaves the session on its old voice.  The
// call waits for the device, so no step of the old plans is in flight when they are released and no event guard is needed.
int ryk_session_set_voice(ryk_engine* h, int id, int voice_id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = get_session(e, id);
  RYK_CHECK(s != nullptr, "no such session");
  Voice* v = engine_voice(e, voice_id);
  RYK_CHECK(v != nullptr, "no such voice");
  if (v == s->voice) return 0;
  RYK_CHECK(voice_models_loaded(v), "load every layer of both of the voice's models before switching a session to it");
  RYK_CHECK(v->stage1->in_ch == s->C, "the voice's stage-1 model does not take the session's mel-cepstrum order");
  RYK_CHECK(session_idle(s) && (!s->group || s->group->collected == s->group->step),
            "collect every submitted chunk of the session and of its group before switching its voice");
  RYK_CHECK(e->precision == s->precision && e->s1_fused == s->s1_fused,
            "the engine's precision or stage-1 mode changed since the session was created: a session keeps the numerics it was created with");
  RYK_CHECK(!s->f0_map.next.follow || v->has_f0_stats, "follow mode needs an f0 map: the voice has no f0 statistics (turn follow mode off first)");
  Group* G = s->group;
  Voice* const old = s->voice;
  if (G) {
    s->voice = v;                                  // the member list as the switch would leave it
    const char* refusal = group_refusal(e, G->members);
    s->voice = old;
    if (refusal) { set_error(refusal); return -1; }
  }
  if (voice_id >= 1 && voice_default_stage1_stats(v, s->C)) return -1;
  RYK_CUDA(cudaDeviceSynchronize());
  const int s1_owner = ++e->plan_owners;
  int lane_owner[2];
  for (int& o : lane_owner) o = ++e->plan_owners;
  StageGraph s1[kHandoffGraphs];
  auto build = [&]() -> int {
    UNetPlan* p = nullptr;
    for (int Tp = 128; Tp <= s->Tp; Tp += 128) if (unet_get_plan(e, v->stage1, 1, 1, Tp, e->precision, &p, s1_owner)) return -1;
    if (!G) for (int o : lane_owner) if (s2_plan(e, s, v, o, &p)) return -1;     // a member runs the group's plan
    for (int j = 0; j < kHandoffGraphs; ++j) if (stage1_build_switch(e, s, v, s1_owner, j, s1[j])) return -1;
    if (G) {
      s->voice = v;
      const int rc = group_rebuild(e, G, G->members);     // commits the group's new plan only on success
      s->voice = old;
      if (rc) return rc;
    }
    return 0;
  };
  if (int rc = build()) {
    for (StageGraph& g : s1) g.reset();
    unet_release_owner(v->stage1, s1_owner);
    for (int o : lane_owner) unet_release_owner(v->stage2, o);
    return rc;
  }
  // swap: nothing below fails
  unet_release_owner(old->stage1, s->s1_owner);
  lanes_release(s);                                // the old lane plans and s2_layers (a group member has none)
  old->users--; v->users++;
  s->voice = v; s->voice_id = voice_id; s->s1_owner = s1_owner;
  for (int i = 0; i < 2; ++i) s->lane[i].owner = lane_owner[i];
  for (int j = 0; j < kHandoffGraphs; ++j) {
    HandoffGraphs& hg = s->hgraphs[j];
    std::swap(hg.s1.exec, s1[j].exec); std::swap(hg.s1.launches, s1[j].launches);     // s1[j] drops the old graph
    hg.s2_pro.reset(); hg.s2_epi.reset();
  }
  // the new voice's f0 map, as a session created on it starts; the speaker statistics, follow mode and formant ratio stay
  const F0Map vm = voice_f0_map(v);
  F0Map& f = s->f0_map.next;
  f.mu_in = vm.mu_in; f.sd_in = vm.sd_in; f.mu_tgt = vm.mu_tgt; f.sd_tgt = vm.sd_tgt;
  f.has_stats = vm.has_stats;
  s->f0_map.dirty = true;
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
  if (int rc = check_in_flight(G->step - G->collected)) return rc;
  for (Session* s : G->members) if (int rc = check_chunk(s, n)) return rc;
  const long long k = G->step;
  for (size_t i = 0; i < G->members.size(); ++i)
    if (stage_in(G->members[i], host_slot(G->members[i], k), waves[i])) return -1;
  if (group_enqueue(e, G, nullptr)) return -1;
  for (Session* s : G->members) {
    HostSlot& io = host_slot(s, k);
    if (stage_out(s, io, io.h_out, io.h_n, cudaMemcpyDeviceToHost)) return -1;
  }
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
    if (collect_out(G->members[i], host_slot(G->members[i], ticket), outs[i], out_capacity, &n_outs[i])) return -1;
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
  RYK_CHECK(waves_dev != nullptr, "null argument");
  for (size_t i = 0; i < G->members.size(); ++i) {
    RYK_CHECK(waves_dev[i] != nullptr, "null argument");
    if (int rc = check_chunk(G->members[i], n)) return rc;
    if (int rc = check_out_capacity(G->members[i], out_capacity)) return rc;
  }
  const long long k = G->step;
  if (group_enqueue(e, G, waves_dev)) return -1;
  for (size_t i = 0; i < G->members.size(); ++i) {
    Session* s = G->members[i];
    if (stage_out(s, host_slot(s, k), outs_dev[i], n_outs_dev[i], cudaMemcpyDeviceToDevice)) return -1;
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
  const cudaEvent_t t0 = s->ev[(s->step - n) % kRing].tev[0][0];
  for (int i = 0; i < n; ++i) {
    const StepEvents& ev = s->ev[(s->step - n + i) % kRing];
    for (int a = 0; a < 5; ++a) {
      RYK_CUDA(cudaEventElapsedTime(&start[i * 5 + a], t0, ev.tev[a][0]));
      RYK_CUDA(cudaEventElapsedTime(&end[i * 5 + a], t0, ev.tev[a][1]));
    }
  }
  return n;
}

// ---- moving a session: snapshot and restore (DESIGN.md §4k) ----
// A session blob holds, in order: CONF (ryk_snapshot_session), TAPI / TAPO (the device rates' taps, when set), HOST (SnapHost), FARN
// (the far end of the next step, with echo cancellation), then one section per device region of session_regions, in its order.

// The host side of the stream state: every host block's next value and dirty flag, the f0 reset and far-end flags, the limiter's and
// AGC's dB settings and the synthesizer's host counters.
struct SnapHost {
  long long step;
  F0Map f0_next; DenoiseParams dn_next; EchoParams aec_next; LimParams lim_next; AgcParams agc_next;
  double lim_ceiling_db, agc_db[3];
  long long host_cum_frames, host_noise_generated;
  int f0_dirty, dn_dirty, aec_dirty, lim_dirty, agc_dirty, f0_reset, far_set, host_noise_slot;
};
static_assert(sizeof(SnapHost) == 2320, "snapshot layout: bump kSnapVersion (snapshot.h)");

// One device region of the stream state and the tag of its section.
struct SnapRegion { uint32_t tag; void* dev; size_t bytes; };

// The device regions that carry stream state, in blob order.  Both parities of every double-buffered region go in: step k reads
// par[k & 1], and carrying par[k & 1 ^ 1] as well keeps the blob independent of which fields a step rewrites in full.  Everything else a
// session owns is scratch or derived and goes in no section: the analysis outputs, silence-gate mask, hand-off slots, step outputs,
// stage-2 lane scratch and per-step spectra (written by a step before it reads them), plans, graphs and events (rebuilt by the
// restoring session), the resampler taps and constant tables (configuration).
static std::vector<SnapRegion> session_regions(const Session* s) {
  std::vector<SnapRegion> r;
  auto add = [&](const char (&t)[5], const void* p, size_t bytes) { r.push_back({snap_tag(t), (void*)p, bytes}); };
  const size_t Lw = s->Lw, Tw = s->Tw, Td = s->Td, nb = s->nb, C = s->C, hop = s->hop;
  for (const ParitySet& p : s->par) {
    add("WAVE", p.wave_win, sizeof(float) * Lw);
    add("CWF0", p.cw_f0, sizeof(float) * Tw);
    add("CWAP", p.cw_ap, sizeof(float) * Tw * nb);
    add("CWMC", p.cw_mc, sizeof(float) * Tw * C);
    add("CWVO", p.cw_voiced, Tw);
    add("CWWV", p.cw_wave, sizeof(float) * Tw * hop);
    add("DWF0", p.dw_f0, sizeof(float) * Td);
    add("DWAP", p.dw_ap, sizeof(float) * Td * nb);
    add("DWSP", p.dw_sp, sizeof(float) * Td * nb);
    for (int i = 0; i < kInputs; ++i) {
      const InputState& x = p.input[i];
      if (x.win) {
        add(i == kMic ? "MWIN" : "FWIN", x.win, sizeof(float) * s->in.hist);
        add(i == kMic ? "MRES" : "FRES", x.rs, sizeof(ResampleState));
      }
      if (x.dn) add(i == kMic ? "MFRM" : "FFRM", x.dn, sizeof(DenoiseState));
    }
    if (p.out_hist) {
      add("OHIS", p.out_hist, sizeof(double) * s->out.hist);
      add("ORES", p.out_st, sizeof(ResampleState));
    }
    if (s->limiter) {
      add("LG0H", p.lim.g0, sizeof(double) * (s->lim.R + 2 * s->lim.L - 1));
      add("LYH ", p.lim.y, sizeof(double) * s->lim.L);
      add("LPOS", p.lim.st, sizeof(LimState));
    }
    if (s->agc) add("AGCS", p.agc, sizeof(AgcState));
  }
  add("F0MP", s->d_f0_map, sizeof(F0Map));
  add("F0ST", s->d_f0_stats, sizeof(F0Stats));
  if (s->denoise) {
    add("DNPA", s->dn.params, sizeof(DenoiseParams));
    add("DNLE", s->dn.learn, sizeof(DenoiseLearn));
  }
  if (s->echo) {
    add("AECP", s->aec.params, sizeof(EchoParams));
    add("AECF", s->aec.filter, sizeof(EchoFilter));
    add("AECR", s->aec.ring, sizeof(double2) * kDnBins * (s->aec.taps + s->aec.delay));
  }
  if (s->limiter) {
    add("LIMP", s->lim.params, sizeof(LimParams));
    add("LIMM", s->lim.meter, sizeof(LimMeter));
  }
  if (s->agc) {
    add("AGCP", s->agcw.params, sizeof(AgcParams));
    add("AGCM", s->agcw.meter, sizeof(AgcMeter));
  }
  const SynthDev& D = s->synth->dev;
  const size_t sb = D.fft_size / 2 + 1;
  add("SYST", D.state, sizeof(SynthState));
  add("SYF0", D.f0, sizeof(double) * D.cap_frames);
  add("SYSP", D.sp, sizeof(float) * D.cap_frames * sb);
  add("SYAP", D.ap, sizeof(float) * D.cap_frames * sb);
  add("SYPI", D.p_index, sizeof(long long) * D.cap_pulses);
  add("SYPT", D.p_time, sizeof(double) * D.cap_pulses);
  add("SYPV", D.p_vuv, sizeof(int) * D.cap_pulses);
  add("SYNZ", D.noise, sizeof(uint32_t) * D.cap_noise);
  add("SYC0", D.carry[0], sizeof(double) * D.carry_len);
  add("SYC1", D.carry[1], sizeof(double) * D.carry_len);
  return r;
}

static void unet_channels(const UNet* n, int* c) { c[0] = n->in_ch; c[1] = n->out_ch; c[2] = n->base; }

// What a session's blob records besides its device regions.
struct SessionBlob {
  ryk_snapshot_session conf;
  std::vector<double> taps_in, taps_out;
  SnapHost host;
  std::vector<SnapRegion> regions;
  int far_n = 0;                   // far-end samples of the next step (echo cancellation)
  std::vector<size_t> payloads() const {
    std::vector<size_t> p = {sizeof(conf)};
    if (conf.in_rate) p.push_back(sizeof(double) * taps_in.size());
    if (conf.out_rate) p.push_back(sizeof(double) * taps_out.size());
    p.push_back(sizeof(host));
    if (conf.echo) p.push_back(sizeof(float) * far_n);
    for (const SnapRegion& x : regions) p.push_back(x.bytes);
    return p;
  }
};

// The session when a snapshot may be taken, else nullptr with the refusal set.
static Session* quiescent_session(Engine* e, int id) {
  Session* s = get_session(e, id);
  if (!s) { set_error("no such session"); return nullptr; }
  if (!session_idle(s)) { set_error("the session has steps in flight: collect every submitted chunk before a snapshot"); return nullptr; }
  if (s->group && s->group->collected != s->group->step) {
    set_error("the session's group has steps in flight: collect every submitted group chunk before a snapshot");
    return nullptr;
  }
  return s;
}

// The configuration and host state of s (the taps are read from the device: the caller has synchronised the session's streams).
static int session_blob(Session* s, int f0_method, int precision, int s1_fused, SessionBlob* b) {
  ryk_snapshot_session& c = b->conf;
  memset(&c, 0, sizeof(c));
  c.cfg = s->cfg;
  c.voice_id = s->voice_id;
  c.precision = precision; c.stage1_fused = s1_fused; c.f0_method = f0_method;
  unet_channels(s->voice->stage1, c.stage1_channels);
  unet_channels(s->voice->stage2, c.stage2_channels);
  c.in_rate = s->in.rate; c.in_up = s->in.up; c.in_down = s->in.down; c.in_taps = s->in.n_taps;
  c.out_rate = s->out.rate; c.out_up = s->out.up; c.out_down = s->out.down; c.out_taps = s->out.n_taps;
  c.denoise = s->denoise; c.echo = s->echo; c.echo_taps = s->aec.taps; c.echo_delay_frames = s->aec.delay;
  c.limiter = s->limiter; c.agc = s->agc; c.f0_measure = s->f0_measure;
  c.limiter_lookahead_ms = s->lim_lookahead_ms; c.limiter_hold_ms = s->lim_hold_ms;
  c.step = s->step;
  b->taps_in.assign(c.in_taps, 0.0);
  b->taps_out.assign(c.out_taps, 0.0);
  if (c.in_rate) RYK_CUDA(cudaMemcpy(b->taps_in.data(), s->in.d_h, sizeof(double) * c.in_taps, cudaMemcpyDeviceToHost));
  if (c.out_rate) RYK_CUDA(cudaMemcpy(b->taps_out.data(), s->out.d_h, sizeof(double) * c.out_taps, cudaMemcpyDeviceToHost));
  SnapHost& h = b->host;
  memset(&h, 0, sizeof(h));
  h.step = s->step;
  h.f0_next = s->f0_map.next; h.f0_dirty = s->f0_map.dirty; h.f0_reset = s->f0_reset;
  h.dn_next = s->dn_params.next; h.dn_dirty = s->dn_params.dirty;
  h.aec_next = s->aec_params.next; h.aec_dirty = s->aec_params.dirty; h.far_set = s->far_set;
  h.lim_next = s->lim_params.next; h.lim_dirty = s->lim_params.dirty; h.lim_ceiling_db = s->lim_ceiling_db;
  h.agc_next = s->agc_params.next; h.agc_dirty = s->agc_params.dirty;
  for (int i = 0; i < 3; ++i) h.agc_db[i] = s->agc_db[i];
  h.host_cum_frames = s->synth->host_cum_frames; h.host_noise_generated = s->synth->host_noise_generated;
  h.host_noise_slot = s->synth->host_noise_slot;
  b->far_n = s->echo ? s->n_in : 0;
  b->regions = session_regions(s);
  return 0;
}

static int session_f0_method(const Session* s) { return s->par[0].crepe ? 2 : dio_plan_harvest(s->par[0].dio) ? 1 : 0; }

using Clock = std::chrono::steady_clock;
static double ms_since(Clock::time_point t) { return std::chrono::duration<double, std::milli>(Clock::now() - t).count(); }

int ryk_session_snapshot_size(ryk_engine* h, int id, size_t* bytes) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(bytes != nullptr, "null argument");
  Session* s = quiescent_session(e, id);
  if (!s) return -2;
  for (cudaStream_t st : s->streams()) RYK_CUDA(cudaStreamSynchronize(st));
  SessionBlob b;
  if (session_blob(s, session_f0_method(s), s->precision, s->s1_fused, &b)) return -1;
  *bytes = snap_size(b.payloads());
  return 0;
}

int ryk_session_snapshot(ryk_engine* h, int id, void* buf, size_t bytes) {
  Engine* e = &h->impl;
  const Clock::time_point t0 = Clock::now();
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(buf != nullptr, "null argument");
  Session* s = quiescent_session(e, id);
  if (!s) return -2;
  for (cudaStream_t st : s->streams()) RYK_CUDA(cudaStreamSynchronize(st));
  SessionBlob b;
  if (session_blob(s, session_f0_method(s), s->precision, s->s1_fused, &b)) return -1;
  const size_t total = snap_size(b.payloads());
  RYK_CHECK(bytes == total, "the buffer must be exactly ryk_session_snapshot_size bytes");
  size_t dev_bytes = 0;
  for (const SnapRegion& x : b.regions) dev_bytes += x.bytes;
  void* hp = nullptr;
  if (engine_pinned(e, dev_bytes, &hp)) return -1;
  const Clock::time_point t1 = Clock::now();
  size_t off = 0;
  for (const SnapRegion& x : b.regions) {
    RYK_CUDA(cudaMemcpyAsync((uint8_t*)hp + off, x.dev, x.bytes, cudaMemcpyDeviceToHost, s->sE));
    off += x.bytes;
  }
  RYK_CUDA(cudaStreamSynchronize(s->sE));
  const double device_ms = ms_since(t1);
  uint8_t* cur = snap_begin(buf, kSnapSession);
  memcpy(snap_section(&cur, snap_tag("CONF"), sizeof(b.conf)), &b.conf, sizeof(b.conf));
  if (b.conf.in_rate) memcpy(snap_section(&cur, snap_tag("TAPI"), sizeof(double) * b.taps_in.size()), b.taps_in.data(), sizeof(double) * b.taps_in.size());
  if (b.conf.out_rate) memcpy(snap_section(&cur, snap_tag("TAPO"), sizeof(double) * b.taps_out.size()), b.taps_out.data(), sizeof(double) * b.taps_out.size());
  memcpy(snap_section(&cur, snap_tag("HOST"), sizeof(b.host)), &b.host, sizeof(b.host));
  if (b.conf.echo) memcpy(snap_section(&cur, snap_tag("FARN"), sizeof(float) * b.far_n), s->far_next.data(), sizeof(float) * b.far_n);
  off = 0;
  for (const SnapRegion& x : b.regions) {
    memcpy(snap_section(&cur, x.tag, x.bytes), (const uint8_t*)hp + off, x.bytes);
    off += x.bytes;
  }
  snap_finish(buf, total);
  e->snap_device_ms = device_ms;
  e->snap_host_ms = ms_since(t0) - device_ms;
  return 0;
}

// The checks of a session blob that need no allocation: its configuration and sections, against engine e and voice voice_id.
static int restore_check(Engine* e, int voice_id, const void* buf, size_t bytes, ryk_snapshot_session* c, std::vector<SnapSection>* sec) {
  uint32_t kind = 0, version = 0;
  if (const char* refusal = snap_parse(buf, bytes, &kind, &version, sec)) { set_error(refusal); return -2; }
  RYK_CHECK(kind == kSnapSession, "not a session snapshot");
  RYK_CHECK(!sec->empty() && (*sec)[0].tag == snap_tag("CONF") && (*sec)[0].bytes == sizeof(*c), "malformed session snapshot: no configuration");
  memcpy(c, (*sec)[0].data, sizeof(*c));
  RYK_CHECK(c->precision == e->precision && c->stage1_fused == (int)e->s1_fused,
            "the engine's precision or stage-1 mode differ from those the snapshot records: a session keeps the numerics it was created with");
  Voice* v = engine_voice(e, voice_id);
  RYK_CHECK(v != nullptr, "no such voice");
  RYK_CHECK(v->stage1 && v->stage2, "load both models before restoring a session");
  int c1[3], c2[3];
  unet_channels(v->stage1, c1);
  unet_channels(v->stage2, c2);
  RYK_CHECK(memcmp(c1, c->stage1_channels, sizeof(c1)) == 0 && memcmp(c2, c->stage2_channels, sizeof(c2)) == 0,
            "the voice's stage-1 or stage-2 (in, out, base) channels differ from those the snapshot records");
  RYK_CHECK(c->f0_method >= 0 && c->f0_method <= 2, "malformed session snapshot: unknown f0 method");
  if (c->f0_method == 2) {
    const char* refusal = crepe_plan_refusal(c->cfg.fs);
    if (refusal) { set_error(refusal); return -2; }
  }
  // CONF, then TAPI / TAPO as the configuration says, HOST and FARN
  size_t i = 1;
  auto expect = [&](const char (&t)[5], size_t n) { return i < sec->size() && (*sec)[i].tag == snap_tag(t) && (*sec)[i++].bytes == n; };
  RYK_CHECK(!c->in_rate || expect("TAPI", sizeof(double) * c->in_taps), "malformed session snapshot: input resampler taps");
  RYK_CHECK(!c->out_rate || expect("TAPO", sizeof(double) * c->out_taps), "malformed session snapshot: output resampler taps");
  RYK_CHECK(expect("HOST", sizeof(SnapHost)), "malformed session snapshot: host state");
  if (c->echo) RYK_CHECK(i < sec->size() && (*sec)[i++].tag == snap_tag("FARN"), "malformed session snapshot: far end");
  return 0;
}

// Enables on session id what the blob records, through the public calls; the settings given here are replaced by the recorded ones.
static int restore_enable(ryk_engine* h, int id, const ryk_snapshot_session& c, const std::vector<SnapSection>& sec) {
  size_t i = 1;
  if (c.in_rate && ryk_session_set_input_rate(h, id, c.in_rate, c.in_up, c.in_down, (const double*)sec[i++].data, c.in_taps)) return -1;
  if (c.out_rate && ryk_session_set_output_rate(h, id, c.out_rate, c.out_up, c.out_down, (const double*)sec[i++].data, c.out_taps)) return -1;
  if (c.denoise && ryk_session_denoise(h, id)) return -1;
  if (c.echo && ryk_session_echo_cancel(h, id, c.echo_taps, c.echo_delay_frames)) return -1;
  if (c.limiter && ryk_session_limiter(h, id, c.limiter_lookahead_ms, c.limiter_hold_ms)) return -1;
  if (c.agc && ryk_session_agc(h, id, -26.0, 20.0, -50.0)) return -1;
  if (c.f0_measure && ryk_session_f0_measure(h, id, 1)) return -1;
  return 0;
}

// Copies the blob's state into the new session s: its device regions through the engine's pinned staging, then its host state.
static int restore_state(Engine* e, Session* s, const ryk_snapshot_session& c, const std::vector<SnapSection>& sec, double* device_ms) {
  size_t i = 1 + (c.in_rate ? 1 : 0) + (c.out_rate ? 1 : 0);
  SnapHost hs;
  memcpy(&hs, sec[i++].data, sizeof(hs));
  const SnapSection* far = c.echo ? &sec[i++] : nullptr;
  RYK_CHECK(!far || far->bytes == sizeof(float) * s->n_in, "malformed session snapshot: far end");
  const std::vector<SnapRegion> regions = session_regions(s);
  RYK_CHECK(sec.size() - i == regions.size(), "the snapshot's state sections do not match the session its configuration makes");
  size_t dev_bytes = 0;
  for (size_t r = 0; r < regions.size(); ++r) {
    RYK_CHECK(sec[i + r].tag == regions[r].tag && sec[i + r].bytes == regions[r].bytes,
              "the snapshot's state sections do not match the session its configuration makes");
    dev_bytes += regions[r].bytes;
  }
  void* hp = nullptr;
  if (engine_pinned(e, dev_bytes, &hp)) return -1;
  size_t off = 0;
  for (size_t r = 0; r < regions.size(); ++r) { memcpy((uint8_t*)hp + off, sec[i + r].data, regions[r].bytes); off += regions[r].bytes; }
  // on the engine stream, behind the zero-fills of the new buffers; the session's streams do not wait for it, so wait here
  const Clock::time_point t1 = Clock::now();
  off = 0;
  for (const SnapRegion& x : regions) {
    RYK_CUDA(cudaMemcpyAsync(x.dev, (const uint8_t*)hp + off, x.bytes, cudaMemcpyHostToDevice, e->stream));
    off += x.bytes;
  }
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  *device_ms = ms_since(t1);
  s->step = s->collected = hs.step;
  s->f0_map.next = hs.f0_next; s->f0_map.dirty = hs.f0_dirty; s->f0_reset = hs.f0_reset;
  s->dn_params.next = hs.dn_next; s->dn_params.dirty = hs.dn_dirty;
  s->aec_params.next = hs.aec_next; s->aec_params.dirty = hs.aec_dirty;
  if (far) memcpy(s->far_next.data(), far->data, far->bytes);
  s->far_set = hs.far_set;
  s->lim_params.next = hs.lim_next; s->lim_params.dirty = hs.lim_dirty; s->lim_ceiling_db = hs.lim_ceiling_db;
  s->agc_params.next = hs.agc_next; s->agc_params.dirty = hs.agc_dirty;
  for (int k = 0; k < 3; ++k) s->agc_db[k] = hs.agc_db[k];
  s->synth->host_cum_frames = hs.host_cum_frames; s->synth->host_noise_generated = hs.host_noise_generated;
  s->synth->host_noise_slot = hs.host_noise_slot;
  return 0;
}

int ryk_session_restore(ryk_engine* h, int voice_id, const void* buf, size_t bytes, int* session_id) {
  Engine* e = &h->impl;
  const Clock::time_point t0 = Clock::now();
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(session_id != nullptr, "null argument");
  ryk_snapshot_session c;
  std::vector<SnapSection> sec;
  if (int rc = restore_check(e, voice_id, buf, bytes, &c, &sec)) return rc;
  int id = -1;
  if (int rc = session_create(e, &c.cfg, voice_id, c.f0_method, &id)) return rc;
  double device_ms = 0.0;
  if (int rc = restore_enable(h, id, c, sec) ? -1 : restore_state(e, e->sessions[id], c, sec, &device_ms)) {
    const std::string cause = ryk_last_error();
    ryk_session_destroy(h, id);
    set_error(cause);
    return rc;
  }
  *session_id = id;
  e->snap_device_ms = device_ms;
  e->snap_host_ms = ms_since(t0) - device_ms;
  return 0;
}

int ryk_snapshot_last_times(ryk_engine* h, double* host_ms, double* device_ms) {
  if (host_ms) *host_ms = h->impl.snap_host_ms;
  if (device_ms) *device_ms = h->impl.snap_device_ms;
  return 0;
}

}  // extern "C"
