// reblock.cu -- output re-blocker + silence gate (SURVEY 8(f) rank 2; realtime_voice_conversion/worker/decode_worker.py:38-59).
// The reference's decode worker concatenates the synthesizer blocks into `wave_fragment`, cuts one out_audio_chunk off its
// front whenever enough samples are queued (at most one per step) and drops the chunk when its mean STFT power is below
// -output_silent_threshold dB.  Here the fragment lives in HBM (ping-pong buffers), the sample count of a step is read from
// device memory (no host sync) and the gate kernels (world_synth.cu) are predicated on the device-side "chunk emitted" flag.
#include "../../include/ryk.h"
#include "engine.h"
#include "features.h"
#include "snapshot.h"

namespace ryk {

constexpr int kRing = 8;          // result slots: a push's results stay readable for 8 pushes

struct ReblockState { int len, sel, overflow; };
static_assert(sizeof(ReblockState) == 12, "snapshot layout: bump kSnapVersion (snapshot.h)");
struct Reblock {
  int chunk = 0, max_in = 0, cap = 0, n_fft = 2048, hop = 512;
  double threshold_db = 80.0;
  ReblockState* d_state = nullptr;
  double* d_frag[2] = {nullptr, nullptr};
  double* d_scratch = nullptr;
  double* d_chunk[kRing] = {}; int* d_nvalid[kRing] = {}; int* d_status[kRing] = {}; double* d_power[kRing] = {};
  double* h_chunk[kRing] = {}; int* h_status[kRing] = {}; double* h_power[kRing] = {}; int* h_overflow[kRing] = {};
  cudaEvent_t ev[kRing] = {};
  double* d_stage_in = nullptr; int* d_stage_n = nullptr;     // staging for the host-buffer entry point
  long long pushed = 0;
  BufferSet mem;
  ~Reblock() { for (cudaEvent_t x : ev) if (x) cudaEventDestroy(x); }
};

void reblock_destroy_all(Engine* e) {
  for (Reblock* R : e->reblocks) delete R;
  e->reblocks.clear();
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

static Reblock* get_reblock(Engine* e, int id) { return (id >= 0 && id < (int)e->reblocks.size()) ? e->reblocks[id] : nullptr; }

}  // namespace ryk

using namespace ryk;

extern "C" {

int ryk_reblock_create(ryk_engine* h, int out_audio_chunk, int max_in, int n_fft, int hop, double threshold_db, int* reblock_id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(out_audio_chunk > n_fft / 2 && max_in > 0, "out_audio_chunk must exceed n_fft / 2 (reflect-centred STFT)");
  RYK_CHECK(n_fft >= 64 && n_fft <= 4096 && (n_fft & (n_fft - 1)) == 0 && hop > 0, "unsupported STFT geometry");
  Reblock* R = new Reblock();
  R->chunk = out_audio_chunk; R->max_in = max_in; R->n_fft = n_fft; R->hop = hop; R->threshold_db = threshold_db;
  R->cap = 2 * out_audio_chunk + 2 * max_in;
  BufferSet& m = R->mem;
  m.stream = e->stream;
  int rc = m.device(&R->d_state, 1) || m.device(&R->d_frag[0], R->cap) || m.device(&R->d_frag[1], R->cap) ||
           m.device(&R->d_scratch, output_gate_scratch_doubles(out_audio_chunk, n_fft, hop)) || m.device(&R->d_stage_in, max_in) ||
           m.device(&R->d_stage_n, 1);
  for (int i = 0; i < kRing && !rc; ++i) {
    rc = m.device(&R->d_chunk[i], out_audio_chunk) || m.device(&R->d_nvalid[i], 1) || m.device(&R->d_status[i], 1) ||
         m.device(&R->d_power[i], 1) || m.pinned(&R->h_chunk[i], out_audio_chunk) || m.pinned(&R->h_status[i], 1) ||
         m.pinned(&R->h_power[i], 1) || m.pinned(&R->h_overflow[i], 1);
    if (!rc && cudaEventCreateWithFlags(&R->ev[i], cudaEventDisableTiming) != cudaSuccess) rc = 1;
  }
  if (rc) { delete R; return -1; }
  RYK_CUDA(cudaStreamSynchronize(e->stream));     // pushes attached to a session run on its (non-blocking) decode stream
  e->reblocks.push_back(R);
  *reblock_id = (int)e->reblocks.size() - 1;
  return 0;
}

int ryk_reblock_destroy(ryk_engine* h, int id) {
  Engine* e = &h->impl;
  Reblock* R = get_reblock(e, id);
  RYK_CHECK(R != nullptr, "no such re-blocker");
  RYK_CUDA(cudaDeviceSynchronize());
  delete R;
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
    const double* s_out = nullptr; const int* s_n = nullptr; int max_out = 0;
    if (int rc = session_last_output(e, session_id, &s_out, &s_n, &max_out, &st)) return rc;
    if (!wave_dev) {
      RYK_CHECK(max_out <= R->max_in, "re-blocker max_in is smaller than the most samples a session step returns");
      wave_dev = s_out; n_dev = s_n;
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

// ---- snapshot and restore (DESIGN.md §4k): RCNF (ryk_snapshot_reblock), RSTA ({len, sel, overflow}), RFR0 / RFR1 (the fragments).
// The result slots are not carried: a restored re-blocker's pushes continue the ticket numbering from the recorded push count.
static void reblock_conf(const Reblock* R, ryk_snapshot_reblock* c) {
  memset(c, 0, sizeof(*c));
  c->out_audio_chunk = R->chunk; c->max_in = R->max_in; c->n_fft = R->n_fft; c->hop = R->hop; c->threshold_db = R->threshold_db;
  c->pushed = R->pushed;
}
static size_t reblock_blob_size(const Reblock* R) {
  return snap_size({sizeof(ryk_snapshot_reblock), sizeof(ReblockState), sizeof(double) * R->cap, sizeof(double) * R->cap});
}

int ryk_reblock_snapshot_size(ryk_engine* h, int id, size_t* bytes) {
  Reblock* R = get_reblock(&h->impl, id);
  RYK_CHECK(R != nullptr && bytes != nullptr, "no such re-blocker");
  *bytes = reblock_blob_size(R);
  return 0;
}

int ryk_reblock_snapshot(ryk_engine* h, int id, void* buf, size_t bytes) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Reblock* R = get_reblock(e, id);
  RYK_CHECK(R != nullptr && buf != nullptr, "no such re-blocker");
  RYK_CHECK(bytes == reblock_blob_size(R), "the buffer must be exactly ryk_reblock_snapshot_size bytes");
  if (R->pushed > 0) RYK_CUDA(cudaEventSynchronize(R->ev[(R->pushed - 1) % kRing]));     // pushes run in order on one stream each
  const size_t frag = sizeof(double) * R->cap;
  ReblockState* st;
  double *fr0, *fr1;
  if (engine_pinned_layout(e, [&](Arena& a) { st = a.take<ReblockState>(1); fr0 = a.take<double>(R->cap); fr1 = a.take<double>(R->cap); }))
    return -1;
  RYK_CUDA(cudaMemcpyAsync(st, R->d_state, sizeof(ReblockState), cudaMemcpyDeviceToHost, e->stream));
  RYK_CUDA(cudaMemcpyAsync(fr0, R->d_frag[0], frag, cudaMemcpyDeviceToHost, e->stream));
  RYK_CUDA(cudaMemcpyAsync(fr1, R->d_frag[1], frag, cudaMemcpyDeviceToHost, e->stream));
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  ryk_snapshot_reblock c;
  reblock_conf(R, &c);
  uint8_t* cur = snap_begin(buf, kSnapReblock);
  memcpy(snap_section(&cur, snap_tag("RCNF"), sizeof(c)), &c, sizeof(c));
  memcpy(snap_section(&cur, snap_tag("RSTA"), sizeof(ReblockState)), st, sizeof(ReblockState));
  memcpy(snap_section(&cur, snap_tag("RFR0"), frag), fr0, frag);
  memcpy(snap_section(&cur, snap_tag("RFR1"), frag), fr1, frag);
  snap_finish(buf, bytes);
  return 0;
}

int ryk_reblock_restore(ryk_engine* h, const void* buf, size_t bytes, int* reblock_id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(reblock_id != nullptr, "null argument");
  uint32_t kind = 0, version = 0;
  std::vector<SnapSection> sec;
  if (const char* refusal = snap_parse(buf, bytes, &kind, &version, &sec)) { set_error(refusal); return -2; }
  RYK_CHECK(kind == kSnapReblock, "not a re-blocker snapshot");
  RYK_CHECK(sec.size() == 4 && sec[0].tag == snap_tag("RCNF") && sec[0].bytes == sizeof(ryk_snapshot_reblock) && sec[1].tag == snap_tag("RSTA") &&
                sec[1].bytes == sizeof(ReblockState) && sec[2].tag == snap_tag("RFR0") && sec[3].tag == snap_tag("RFR1"),
            "malformed re-blocker snapshot");
  ryk_snapshot_reblock c;
  memcpy(&c, sec[0].data, sizeof(c));
  const size_t frag = sizeof(double) * (2 * (size_t)c.out_audio_chunk + 2 * (size_t)c.max_in);
  RYK_CHECK(c.pushed >= 0 && sec[2].bytes == frag && sec[3].bytes == frag, "malformed re-blocker snapshot");
  int id = -1;
  if (int rc = ryk_reblock_create(h, c.out_audio_chunk, c.max_in, c.n_fft, c.hop, c.threshold_db, &id)) return rc;
  Reblock* R = e->reblocks[id];
  ReblockState* st;
  double *fr0, *fr1;
  int rc = engine_pinned_layout(e, [&](Arena& a) { st = a.take<ReblockState>(1); fr0 = a.take<double>(R->cap); fr1 = a.take<double>(R->cap); });
  if (!rc) {
    memcpy(st, sec[1].data, sizeof(ReblockState));
    memcpy(fr0, sec[2].data, frag);
    memcpy(fr1, sec[3].data, frag);
    const cudaError_t err[4] = {cudaMemcpyAsync(R->d_state, st, sizeof(ReblockState), cudaMemcpyHostToDevice, e->stream),
                                cudaMemcpyAsync(R->d_frag[0], fr0, frag, cudaMemcpyHostToDevice, e->stream),
                                cudaMemcpyAsync(R->d_frag[1], fr1, frag, cudaMemcpyHostToDevice, e->stream),
                                cudaStreamSynchronize(e->stream)};
    for (cudaError_t x : err) if (x != cudaSuccess && !rc) { set_error(std::string("re-blocker restore copy failed: ") + cudaGetErrorString(x)); rc = -1; }
  }
  if (rc) {
    const std::string cause = ryk_last_error();
    ryk_reblock_destroy(h, id);
    set_error(cause);
    return rc;
  }
  R->pushed = c.pushed;
  *reblock_id = id;
  return 0;
}

}  // extern "C"
