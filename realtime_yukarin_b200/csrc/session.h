// session.h -- the state of streaming sessions and groups, shared by the session*.cu files (private to libryk).
#pragma once
#include <array>
#include <vector>

#include "../../include/ryk.h"
#include "agc.h"
#include "echo.h"
#include "engine.h"
#include "features.h"
#include "limiter.h"
#include "pitch.h"

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
  T& edit() { dirty = true; return next; }     // what a setter changes
};
// The host-API staging of the caller's ticket t in slot t % kRing: the session's own step alone, the group's step while grouped.  A
// membership change needs every host-API step collected, so no slot of one numbering is in use when the other takes over.
struct HostSlot {
  float* h_in = nullptr; double* h_out = nullptr; int* h_n = nullptr;     // pinned
  cudaEvent_t dec = nullptr;       // output staged (after the copies the entry point appends to stream D)
};
// Stage 2 of a session alone runs the chunks of parity b on lane b, so the bottleneck layers of one chunk overlap the GPU-filling
// layers of its neighbour.  A group member runs its prologue and epilogue on lane 0 (s2_lane).
struct Stage2Lane {
  cudaStream_t stream = nullptr;
  float* d_colmin = nullptr;       // stage-2 prologue scratch, written only on this lane's stream
  int owner = 0;                   // plan-cache owner id of the lane's stage-2 plan
  StageGraph s2_layers;            // alone: stage-2 layers 1..14
};

// The optional stages of a session, one member each (DESIGN.md §4a, §4f-§4j, §4m): `on`, the host block whose device copy is the `params` of
// the work struct the kernels read, the settings as the user gave them, and the stage's buffers.  Per-parity state stays in ParitySet.
struct F0Control {                 // the f0 map, formant ratio and speaker statistics
  static constexpr const char* refusal = "f0 measurement is not enabled for this session";
  bool on = false;                 // measuring (k_f0_measure)
  bool reset = false;              // the statistics restart at the next submitted step
  HostBlock<F0Map> block;
  F0Map* d_map = nullptr; F0Stats* d_stats = nullptr;
};
struct FrameStage {                // shared by noise suppression (w.params, w.learn) and echo cancellation
  DenoiseWork w;
  float* d_chunk = nullptr;        // the step's filtered chunk
};
struct DenoiseStage {
  static constexpr const char* refusal = "noise suppression is not enabled for this session (ryk_session_denoise)";
  bool on = false;
  HostBlock<DenoiseParams> block;
};
struct EchoStage {
  static constexpr const char* refusal = "echo cancellation is not enabled for this session (ryk_session_echo_cancel)";
  bool on = false;
  HostBlock<EchoParams> block;
  EchoWork w;
  std::vector<float> far_next;     // the far end of the next submitted step (zeros when none was given)
  bool far_set = false;
  float* h_far = nullptr;          // pinned staging of the far end: slot k % kRing (n_in samples) for step k
};
struct LimiterStage {
  static constexpr const char* refusal = "the output limiter is not enabled for this session (ryk_session_limiter)";
  bool on = false;
  HostBlock<LimParams> block;
  LimWork w;
  double lookahead_ms = 0.0, hold_ms = 0.0, ceiling_db = 0.0;   // L and R follow the output rate
};
struct AgcStage {
  static constexpr const char* refusal = "the automatic gain control is not enabled for this session (ryk_session_agc)";
  bool on = false;
  HostBlock<AgcParams> block;
  AgcWork w;
  double db[3] = {};               // target, max gain and gate
  float* d_chunk = nullptr;        // the step's gain-controlled chunk
};
struct PitchStage {
  static constexpr const char* refusal = "pitch correction is not enabled for this session (ryk_session_pitch_correct)";
  bool on = false;
  HostBlock<PitchParams> block;
  PitchWork w;
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
  F0Control f0;
  FrameStage frame;
  DenoiseStage dn;
  EchoStage aec;
  LimiterStage lim;
  AgcStage agc;
  PitchStage pitch;
  BufferSet mem;                   // every device and pinned buffer above
};

// Several sessions on one GPU sharing ONE batched stage-2 forward per step (BASELINE config 5; session_group.cu).  Everything else stays
// per stream: those stages carry per-stream state and data-dependent lengths, and they are a small share of the SM time.
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

inline Session* get_session(Engine* e, int id) { return (id >= 0 && id < (int)e->sessions.size()) ? e->sessions[id] : nullptr; }
// The session when it has not run a chunk yet (what its graphs capture at the first steps can still change), else nullptr with the
// error set: "no such session", or `refusal`.
Session* fresh_session(Engine* e, int id, const char* refusal);
// A session's host-API steps are all collected (device-resident steps count as collected).
inline bool session_idle(const Session* s) { return s->collected == s->step; }
// The one way a session is made (ryk_session_create_voice, ryk_session_restore): f0_method is the engine's, or the one a snapshot records.
int session_create(Engine* e, const ryk_session_config* cfg, int voice_id, int f0_method, int* session_id);
int input_alloc(Session* s, int i, int n_in, bool resampled);
int limiter_alloc(Session* s, const LimParams& first);
int s2_plan(Engine* e, const Session* s, Voice* v, int owner, UNetPlan** p2);
void lanes_release(Session* s);
int stage1_build_switch(Engine* e, Session* s, Voice* v, int owner, int j, StageGraph& g);
void group_free(Group* G);

// Allocates block b's device copy *dev and its kRing pinned slots, and makes `first` what the next submitted step copies.
template <typename T>
int host_block_alloc(BufferSet& m, HostBlock<T>& b, T** dev, const T& first) {
  if (m.device(dev, 1) || m.pinned(&b.ring, kRing)) return -1;
  b.next = first;
  b.dirty = true;
  return 0;
}

// The host slot of the caller's ticket: the session's own step alone, the group's step for a member.
inline HostSlot& host_slot(Session* s, long long ticket) { return s->io[ticket % kRing]; }
int stage_in(Session* s, HostSlot& io, const float* wave);
int stage_out(Session* s, HostSlot& io, double* out, int* n_out, cudaMemcpyKind kind);
int collect_out(Session* s, HostSlot& io, double* out, int out_capacity, int* n_out);
// the checks the submit and push entry points of sessions and groups share
inline int check_chunk(const Session* s, int n) { RYK_CHECK(n == s->n_in, "chunk length must be round(rate * buffer_time) at the session's input rate"); return 0; }
inline int check_in_flight(long long in_flight) { RYK_CHECK(in_flight < kRing - 2, "too many chunks in flight: collect before submitting more"); return 0; }
inline int check_out_capacity(const Session* s, int out_capacity) {
  RYK_CHECK(out_capacity >= s->max_out, "out_capacity must hold the most samples a step returns (ryk_session_io_geometry max_out)");
  return 0;
}
int group_enqueue(Engine* e, Group* G, const float* const* d_chunks);

}  // namespace ryk
