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
#include <numeric>
#include <vector>

#include "../../include/ryk.h"
#include "session.h"

namespace ryk {

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

Session* fresh_session(Engine* e, int id, const char* refusal) {
  Session* s = get_session(e, id);
  if (!s) set_error("no such session");
  else if (s->step != 0) set_error(refusal);
  return s && s->step == 0 ? s : nullptr;
}

// (Re)allocates input i at chunk length n_in, with a history window and resampler state pair when `resampled` (device input rate, window
// of in.hist samples).  The far end also gets its host staging, the next step's samples and kRing pinned slots; the microphone is
// staged through HostSlot::h_in.
int input_alloc(Session* s, int i, int n_in, bool resampled) {
  BufferSet& m = s->mem;
  InputSignal& x = s->input[i];
  if (m.device(&x.d_fixed, n_in)) return -1;
  if (resampled) {
    for (ParitySet& p : s->par) if (m.device(&p.input[i].win, s->in.hist) || m.device(&p.input[i].rs, 1)) return -1;
    if (m.device(&x.d_model, s->n_wave)) return -1;
  }
  if (i == kFar) {
    if (m.pinned(&s->aec.h_far, (size_t)kRing * n_in)) return -1;
    s->aec.far_next.assign(n_in, 0.f);
    s->aec.far_set = false;
  }
  return 0;
}

// Drop the stage-2 plans of a session's own lanes and the graphs captured on them (a no-op for plans a group already released).
void lanes_release(Session* s) {
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

void group_free(Group* G) {
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

// every stream of the engine's sessions and groups
static std::vector<cudaStream_t> session_streams(Engine* e) {
  std::vector<cudaStream_t> all;
  for (Session* s : e->sessions) if (s) for (cudaStream_t st : s->streams()) all.push_back(st);
  for (Group* G : e->groups) if (G) all.push_back(G->sG);
  return all;
}
// make every session stream wait for what is already queued on the engine's main stream
int session_streams_fork(Engine* e, cudaEvent_t ev) {
  for (cudaStream_t st : session_streams(e)) RYK_CUDA(cudaStreamWaitEvent(st, ev, 0));
  return 0;
}
// make the engine's main stream wait for everything queued on the session streams
int session_streams_join(Engine* e) {
  for (cudaStream_t st : session_streams(e)) {
    cudaEvent_t ev;
    RYK_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
    RYK_CUDA(cudaEventRecord(ev, st));
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
int stage1_build_switch(Engine* e, Session* s, Voice* v, int owner, int j, StageGraph& g) {
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
  if (s->f0.on && f0_measure_run(p.enc_f0 + pe, p.enc_voiced + pe, s->n_feat, s->f0.d_stats, s->f0.d_map, s->sC)) return -1;
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
  EchoStage& a = s->aec;
  float* slot = a.h_far + (size_t)(k % kRing) * s->n_in;
  if (a.far_set) memcpy(slot, a.far_next.data(), sizeof(float) * s->n_in);
  else memset(slot, 0, sizeof(float) * s->n_in);
  a.far_set = false;
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
                          o.mc_out, o.f0_out, o.ap_out, o.voiced_out, s->f0.d_map, s->sC, o.formant)) return -1;
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
int s2_plan(Engine* e, const Session* s, Voice* v, int owner, UNetPlan** p2) {
  return unet_get_plan(e, v->stage2, 1, s->Tp, 512, e->precision, p2, owner, s->e_conv, s->n_feat, false, s->Tw);
}

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
  if (host_block_sync(s->dn.block, s->frame.w.params, k, ev.gate, s->sE)) return -1;
  if (host_block_sync(s->aec.block, s->aec.w.params, k, ev.gate, s->sE)) return -1;
  if (host_block_sync(s->agc.block, s->agc.w.params, k, ev.gate, s->sE)) return -1;
  if (s->aec.on && far_sync(s, k)) return -1;
  if (stage_time(s, 0, 0, r, s->sE)) return -1;
  if (run_graph(e, p.graphs.gate, s->sE, [&]() -> int {
        const float *chunk = nullptr, *far = nullptr;
        if (input_to_model(e, s, b, kMic, &chunk)) return -1;
        if (s->aec.on && input_to_model(e, s, b, kFar, &far)) return -1;
        if (s->dn.on || s->aec.on) {  // the frame stage in front of the wave slide: echo cancellation, then noise suppression
          const DenoiseWork& w = s->frame.w;
          const InputState &pm = p.input[kMic], &qm = q.input[kMic], &pf = p.input[kFar], &qf = q.input[kFar];
          if (denoise_forward(e, w.max_frames, pm.dn, qm.dn, chunk, s->n_wave, w.spec, s->sE)) return -1;
          if (s->aec.on) {
            if (denoise_forward(e, w.max_frames, pf.dn, qf.dn, far, s->n_wave, s->aec.w.far_spec, s->sE)) return -1;
            if (echo_scan(s->aec.w, pm.dn, s->n_wave, w.spec, s->sE)) return -1;
          }
          if (s->dn.on && denoise_scan(w, pm.dn, qm.dn, s->n_wave, s->sE)) return -1;
          if (denoise_inverse(e, w, pm.dn, qm.dn, s->n_wave, s->frame.d_chunk, s->sE)) return -1;
          chunk = s->frame.d_chunk;
        }
        if (s->agc.on) {              // the gain control after the frame stage: a varying gain there would look like a moving echo path
          if (agc_run(s->agc.w, p.agc, q.agc, chunk, s->n_wave, s->agc.d_chunk, s->sE)) return -1;
          chunk = s->agc.d_chunk;
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
  if (s->f0.reset) RYK_CUDA(cudaMemsetAsync(s->f0.d_stats, 0, sizeof(F0Stats), s->sC));
  s->f0.reset = false;
  if (host_block_sync(s->f0.block, s->f0.d_map, k, ev.cslide, s->sC)) return -1;
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
    if (s2_plan(e, s, s->voice, lane.owner, &p2)) return -1;
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
  if (s2_plan(e, s, s->voice, lane.owner, &p2)) return -1;
  cudaEvent_t pe0 = nullptr, pe1 = nullptr;
  if (e->profile) { RYK_CUDA(cudaEventCreate(&pe0)); RYK_CUDA(cudaEventCreate(&pe1)); RYK_CUDA(cudaEventRecord(pe0, lane.stream)); }
  if (run_graph(e, lane.s2_layers, lane.stream, [&]() -> int { return unet_forward(e, p2, lane.stream, 1, 14); })) return -1;
  if (e->profile) { RYK_CUDA(cudaEventRecord(pe1, lane.stream)); e->prof_events.emplace_back(pe0, pe1); }
  return 0;
}

// the samples a step of parity b returns and their count: the synthesizer's blocks, or their device-rate resampling (synth_out), or
// with the output limiter its output for them
static double* synth_out(Session* s, int b) { return s->out.rate ? s->par[b].d_rout_fixed : s->par[b].d_out_fixed; }
static double* step_out(Session* s, int b) { return s->lim.on ? s->par[b].d_lim_out : synth_out(s, b); }
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
    if (s2_plan(e, s, s->voice, lane.owner, &p2)) return -1;
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
  // the limiter's and the pitch correction's settings: their pinned slots were last read by copies of step k - kRing, ahead of that
  // step's decode slides
  if (host_block_sync(s->lim.block, s->lim.w.params, k, ev.dslide, s->sD)) return -1;
  if (host_block_sync(s->pitch.block, s->pitch.w.params, k, ev.dslide, s->sD)) return -1;
  if (run_handoff_graph(e, s, k, &HandoffGraphs::dec_slide, s->sD, [&](int h) -> int {
        const HandoffSlot& o = s->ho[h];
        SlideBatch sb; sb.n = 0;
        slide_add<float>(sb, p.dw_f0, o.f0_out + pc, q.dw_f0, s->Td, s->n_feat, 1);
        slide_add<float>(sb, p.dw_ap, o.ap_out + (size_t)pc * s->nb, q.dw_ap, s->Td, s->n_feat, s->nb);
        slide_add<float>(sb, p.dw_sp, o.sp_out + (size_t)pc * s->nb, q.dw_sp, s->Td, s->n_feat, s->nb);
        if (slide_batch(sb, s->sD)) return -1;
        // P4: the rows this step appended, corrected once each in stream order; older rows were corrected when they were appended
        if (s->pitch.on && pitch_run(s->pitch.w, q.dw_f0 + (s->Td - s->n_feat), s->n_feat, s->sD)) return -1;
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
        if (!s->lim.on) return 0;
        // the limiter last, at the output rate: it changes no upstream state
        return limiter_run(s->lim.w, p.lim, q.lim, synth_out(s, b), step_n_out(s, b), p.d_lim_out, s->sD);
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
int group_enqueue(Engine* e, Group* G, const float* const* d_chunks) {
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
// host chunk -> pinned slot -> input[kMic].d_fixed on stream E, in front of the step's wave slides
int stage_in(Session* s, HostSlot& io, const float* wave) {
  memcpy(io.h_in, wave, sizeof(float) * s->n_in);
  RYK_CUDA(cudaMemcpyAsync(s->input[kMic].d_fixed, io.h_in, sizeof(float) * s->n_in, cudaMemcpyHostToDevice, s->sE));
  return 0;
}

// after a step of s was enqueued: copy its samples and sample count to out / n_out (kind: to the host slot or to device buffers) behind
// the decode stream and record io.dec.  The output buffers are those of the parity of the session's own step, which differs from the
// group's for a member that joined at a group step of the other parity.
int stage_out(Session* s, HostSlot& io, double* out, int* n_out, cudaMemcpyKind kind) {
  const int b = (int)((s->step - 1) & 1);
  RYK_CUDA(cudaMemcpyAsync(n_out, step_n_out(s, b), sizeof(int), kind, s->sD));
  RYK_CUDA(cudaMemcpyAsync(out, step_out(s, b), sizeof(double) * s->max_out, kind, s->sD));
  RYK_CUDA(cudaEventRecord(io.dec, s->sD));
  return 0;
}

// wait for the step staged in io and copy its samples out of the host slot
int collect_out(Session* s, HostSlot& io, double* out, int out_capacity, int* n_out) {
  RYK_CUDA(cudaEventSynchronize(io.dec));
  const int produced = *io.h_n;
  RYK_CHECK(produced <= out_capacity, "output buffer too small for the produced blocks");
  memcpy(out, io.h_out, sizeof(double) * produced);
  *n_out = produced;
  s->collected++;
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
  F0Map f0_map = voice_f0_map(s->voice);
  f0_map.formant = 1.0;
  if (host_block_alloc(m, s->f0.block, &s->f0.d_map, f0_map) || m.device(&s->f0.d_stats, 1)) return -1;
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
  RYK_CUDA(cudaDeviceSynchronize());
  s->precision = e->precision; s->s1_fused = e->s1_fused;
  for (int j = 0; j < kHandoffGraphs; ++j) if (stage1_build_switch(e, s, s->voice, s->s1_owner, j, s->hgraphs[j].s1)) return -1;
  return 0;
}

int session_create(Engine* e, const ryk_session_config* cfg, int voice_id, int f0_method, int* session_id) {
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

}  // namespace ryk

using namespace ryk;

extern "C" {


int ryk_session_create_voice(ryk_engine* h, const ryk_session_config* cfg, int voice_id, int* session_id) {
  return session_create(&h->impl, cfg, voice_id, h->impl.f0_method, session_id);
}

int ryk_session_create(ryk_engine* h, const ryk_session_config* cfg, int* session_id) { return ryk_session_create_voice(h, cfg, 0, session_id); }

int ryk_session_voice(ryk_engine* h, int id) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  return s->voice_id;
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
  side.rate = rate; side.up = up; side.down = down; side.n_taps = n_taps;
  if (input) {
    s->n_in = (int)lrint(s->cfg.buffer_time * rate);
    s->delay_in = half / down;
  } else {
    s->max_out = (int)(((long long)s->max_blocks * s->cfg.vocoder_buffer_size * up + down - 1) / down);
    if (s->lim.on && limiter_alloc(s, s->lim.block.next)) return -1;     // the limiter's L, R and buffers at the new rate and max_out
  }
  RYK_CUDA(cudaStreamSynchronize(e->stream));      // the zero-fills and the taps: the session's streams do not wait for the engine stream
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
  if (delay_in) *delay_in = s->delay_in + (s->dn.on || s->aec.on ? kDnDelay : 0);
  if (in_rate) *in_rate = s->in.rate ? s->in.rate : s->cfg.fs;
  if (out_rate) *out_rate = s->out.rate ? s->out.rate : s->cfg.fs;
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

}  // extern "C"
