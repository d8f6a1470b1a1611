// drift.cu -- the clock drift stage (DESIGN.md §4l, DECIDE D1-D4): an asynchronous resampler on the played stream.  The read position
// is an int64 in 2^-32 samples that every output advances by inc = llrint(2^32 / (1 + ppm 1e-6)); each output interpolates a 512-phase
// windowed-sinc table linearly between adjacent phases and sums its 32 taps in FP64, with explicit round-to-nearest operations only, so
// tests/drift_oracle.py gives its bits.  One launch per push, one thread per output; the output count is decided on the device.
#include <math.h>
#include <string.h>

#include <vector>

#include "../../include/ryk.h"
#include "drift.h"
#include "engine.h"
#include "snapshot.h"

namespace ryk {

constexpr long long kOne = 1ll << 32;
constexpr int kDriftThreads = 256;

// DSTA: the device state of the current parity with the setting of the next push
struct DriftSnap { long long pos, consumed, produced, inc; double ppm; };
static_assert(sizeof(DriftState) == 40 && sizeof(DriftSnap) == 40 && sizeof(ryk_snapshot_drift) == 32,
              "snapshot layout: bump kSnapVersion (snapshot.h)");

struct Drift {
  int max_in = 0;
  double max_ppm = 0.0;
  double ppm = 0.0;                   // the setting of the next push
  long long inc = kOne;
  long long pushed = 0;               // pushes since creation: push k reads parity k & 1
  std::vector<double> table;          // the prototype filter as uploaded (carried by a snapshot)
  DriftState* d_state = nullptr;      // [2]
  double* d_hist[2] = {nullptr, nullptr};   // [2W]: the last 2W samples before the push (the delayed stream's)
  double* d_x = nullptr;              // [max_in]
  double* d_y = nullptr;              // [drift_capacity(max_in)]
  double* d_table = nullptr;          // [kDriftTable]
  double* h_x = nullptr;
  double* h_y = nullptr;
  DriftState* h_state = nullptr;      // the state the last push wrote (totals for ryk_drift_stats)
  BufferSet mem;
};

long long drift_inc(double ppm) { return llrint(4294967296.0 / (1.0 + ppm * 1e-6)); }

long long drift_capacity(long long n, double max_ppm) { return n + (long long)ceil((double)n * max_ppm * 1e-6) + 2; }

void drift_destroy_all(Engine* e) {
  for (Drift* D : e->drifts) delete D;
  e->drifts.clear();
}

// One push: the n samples in x follow the 2W kept ones in hist; output k (k < count) reads at pos + k inc.  Every thread derives the
// count from the state; block 0 writes the next parity's history and state, which no thread of this launch reads.
__global__ void __launch_bounds__(kDriftThreads) k_drift(const DriftState* __restrict__ cur, DriftState* __restrict__ next,
                                                         const double* __restrict__ hist, double* __restrict__ hist_next,
                                                         const double* __restrict__ x, int n, long long inc,
                                                         const double* __restrict__ table, double* __restrict__ y) {
  const long long pos = cur->pos;
  const long long num = (long long)n * kOne - pos;
  const long long count = num > 0 ? (num + inc - 1) / inc : 0;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < count) {
    const long long q = pos + (long long)k * inc;
    const int i = (int)(q >> 32);                                   // z[i] with 0 <= i < n: taps z[i - W + 1 .. i + W]
    const unsigned f = (unsigned)(q & (kOne - 1));
    const int phi = (int)(f >> 23);
    const double w = __dmul_rn((double)(f & 0x7fffffu), 0x1p-23);  // exact
    double acc = 0.0;
#pragma unroll 8
    for (int t = 0; t < kDriftTaps; ++t) {
      const int base = (kDriftTaps - 1 - t) * kDriftPhases + phi;
      const double h0 = __ldg(table + base), h1 = __ldg(table + base + 1);
      const double c = __dadd_rn(h0, __dmul_rn(w, __dsub_rn(h1, h0)));
      const int s = i + 1 + t;                                      // b[s], b = concat(hist, x)
      const double v = s < kDriftTaps ? hist[s] : x[s - kDriftTaps];
      acc = __dadd_rn(acc, __dmul_rn(c, v));
    }
    y[k] = acc;
  }
  if (blockIdx.x == 0) {
    for (int t = threadIdx.x; t < kDriftTaps; t += blockDim.x) {
      const int s = n + t;
      hist_next[t] = s < kDriftTaps ? hist[s] : x[s - kDriftTaps];
    }
    if (threadIdx.x == 0) {
      next->pos = pos + count * inc - (long long)n * kOne;
      next->consumed = cur->consumed + n;
      next->produced = cur->produced + count;
      next->inc = inc;
      next->count = count;
    }
  }
}

static int drift_launch(const DriftState* cur, DriftState* next, const double* hist, double* hist_next, const double* x, int n,
                        long long inc, const double* table, double* y, long long capacity, cudaStream_t st) {
  const int blocks = (int)((capacity + kDriftThreads - 1) / kDriftThreads);
  k_drift<<<blocks > 0 ? blocks : 1, kDriftThreads, 0, st>>>(cur, next, hist, hist_next, x, n, inc, table, y);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

static int drift_check_table(const double* table, int phases, int half_width) {
  RYK_CHECK(table != nullptr, "null filter table");
  RYK_CHECK(phases == kDriftPhases && half_width == kDriftHalfWidth,
            "the drift filter table must hold 2 * 16 * 512 + 1 entries: phases 512, half_width 16");
  for (int k = 0; k < kDriftTable; ++k) RYK_CHECK(isfinite(table[k]), "the drift filter table holds a value that is not finite");
  return 0;
}

static int drift_check_ppm(double ppm, double max_ppm) {
  RYK_CHECK(isfinite(ppm) && fabs(ppm) <= max_ppm, "|ppm| must not exceed the drift object's max_ppm");
  return 0;
}

static Drift* get_drift(Engine* e, int id) { return (id >= 0 && id < (int)e->drifts.size()) ? e->drifts[id] : nullptr; }

}  // namespace ryk

using namespace ryk;

extern "C" {

int ryk_drift_create(ryk_engine* h, int max_in, double max_ppm, const double* table, int phases, int half_width, int* drift_id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(drift_id != nullptr, "null argument");
  RYK_CHECK(max_in > 0 && max_in <= kDriftMaxIn, "max_in must be within [1, 2^24]");
  RYK_CHECK(isfinite(max_ppm) && max_ppm > 0.0 && max_ppm <= kDriftMaxPpm, "max_ppm must be within (0, 2000]");
  if (int rc = drift_check_table(table, phases, half_width)) return rc;
  Drift* D = new Drift();
  D->max_in = max_in; D->max_ppm = max_ppm;
  D->table.assign(table, table + kDriftTable);
  const long long cap = drift_capacity(max_in, max_ppm);
  BufferSet& m = D->mem;
  m.stream = e->stream;
  int rc = m.device(&D->d_state, 2) || m.device(&D->d_hist[0], kDriftTaps) || m.device(&D->d_hist[1], kDriftTaps) ||
           m.device(&D->d_x, max_in) || m.device(&D->d_y, cap) || m.device(&D->d_table, kDriftTable) || m.pinned(&D->h_x, max_in) ||
           m.pinned(&D->h_y, cap) || m.pinned(&D->h_state, 1);
  if (!rc && cudaMemcpyAsync(D->d_table, D->table.data(), sizeof(double) * kDriftTable, cudaMemcpyHostToDevice, e->stream) != cudaSuccess) rc = 1;
  if (!rc && cudaStreamSynchronize(e->stream) != cudaSuccess) rc = 1;
  if (rc) {
    const std::string cause = ryk_last_error();
    delete D;
    set_error(cause.empty() ? "drift object allocation failed" : cause);
    return -1;
  }
  D->h_state->inc = kOne;
  e->drifts.push_back(D);
  *drift_id = (int)e->drifts.size() - 1;
  return 0;
}

int ryk_drift_destroy(ryk_engine* h, int id) {
  Engine* e = &h->impl;
  Drift* D = get_drift(e, id);
  RYK_CHECK(D != nullptr, "no such drift object");
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  delete D;
  e->drifts[id] = nullptr;
  return 0;
}

int ryk_drift_set(ryk_engine* h, int id, double ppm) {
  Drift* D = get_drift(&h->impl, id);
  RYK_CHECK(D != nullptr, "no such drift object");
  if (int rc = drift_check_ppm(ppm, D->max_ppm)) return rc;
  D->ppm = ppm;
  D->inc = drift_inc(ppm);
  return 0;
}

int ryk_drift_get(ryk_engine* h, int id, double* ppm, long long* inc) {
  Drift* D = get_drift(&h->impl, id);
  RYK_CHECK(D != nullptr, "no such drift object");
  if (ppm) *ppm = D->ppm;
  if (inc) *inc = D->inc;
  return 0;
}

int ryk_drift_push(ryk_engine* h, int id, const double* x, int n, double* y, int y_capacity, int* n_out) {
  Engine* e = &h->impl;
  Drift* D = get_drift(e, id);
  RYK_CHECK(D != nullptr, "no such drift object");
  RYK_CHECK(n >= 0 && n <= D->max_in, "more samples than the drift object's max_in");
  RYK_CHECK((x != nullptr || n == 0) && y != nullptr && n_out != nullptr, "null argument");
  const long long cap = drift_capacity(n, D->max_ppm);
  RYK_CHECK(y_capacity >= cap, "the output buffer must hold n + ceil(n max_ppm 1e-6) + 2 samples");
  RYK_CUDA(cudaSetDevice(e->device));
  cudaStream_t st = e->stream;
  const int p = (int)(D->pushed & 1);
  if (n > 0) {
    memcpy(D->h_x, x, sizeof(double) * n);
    RYK_CUDA(cudaMemcpyAsync(D->d_x, D->h_x, sizeof(double) * n, cudaMemcpyHostToDevice, st));
  }
  if (drift_launch(D->d_state + p, D->d_state + (p ^ 1), D->d_hist[p], D->d_hist[p ^ 1], D->d_x, n, D->inc, D->d_table, D->d_y, cap, st))
    return -1;
  RYK_CUDA(cudaMemcpyAsync(D->h_state, D->d_state + (p ^ 1), sizeof(DriftState), cudaMemcpyDeviceToHost, st));
  RYK_CUDA(cudaMemcpyAsync(D->h_y, D->d_y, sizeof(double) * cap, cudaMemcpyDeviceToHost, st));
  RYK_CUDA(cudaStreamSynchronize(st));
  D->pushed++;
  const int count = (int)D->h_state->count;
  memcpy(y, D->h_y, sizeof(double) * count);
  *n_out = count;
  return 0;
}

int ryk_drift_stats(ryk_engine* h, int id, long long* consumed, long long* produced) {
  Drift* D = get_drift(&h->impl, id);
  RYK_CHECK(D != nullptr, "no such drift object");
  if (consumed) *consumed = D->h_state->consumed;
  if (produced) *produced = D->h_state->produced;
  return 0;
}

// The whole signal: one push of x followed by W zeros from a fresh state, on the engine's scratch.
int ryk_drift_resample(ryk_engine* h, const double* x, int n, double ppm, const double* table, int phases, int half_width, double* y,
                       int y_capacity, int* n_out) {
  Engine* e = &h->impl;
  RYK_CHECK(x != nullptr && y != nullptr && n_out != nullptr && n > 0, "null argument or empty signal");
  RYK_CHECK(n <= kDriftMaxIn - kDriftHalfWidth, "signal longer than 2^24 - 16 samples");
  RYK_CHECK(isfinite(ppm) && fabs(ppm) <= kDriftMaxPpm, "|ppm| must not exceed 2000");
  if (int rc = drift_check_table(table, phases, half_width)) return rc;
  const int len = n + kDriftHalfWidth;
  const long long cap = drift_capacity(len, fabs(ppm));
  RYK_CHECK(y_capacity >= cap, "the output buffer must hold len + ceil(len |ppm| 1e-6) + 2 samples, len = n + 16");
  RYK_CUDA(cudaSetDevice(e->device));
  DriftState* d_st;
  double *d_hist, *d_table, *d_x, *d_y;
  if (engine_scratch(e, [&](Arena& a) {
        d_st = a.take<DriftState>(2);
        d_hist = a.take<double>(2 * kDriftTaps);
        d_table = a.take<double>(kDriftTable);
        d_x = a.take<double>(len);
        d_y = a.take<double>(cap);
      })) return -1;
  double *h_table, *h_x, *h_y;
  DriftState* h_st;
  if (engine_pinned_layout(e, [&](Arena& a) {
        h_table = a.take<double>(kDriftTable);
        h_x = a.take<double>(len);
        h_y = a.take<double>(cap);
        h_st = a.take<DriftState>(1);
      })) return -1;
  memcpy(h_table, table, sizeof(double) * kDriftTable);
  memcpy(h_x, x, sizeof(double) * n);
  memset(h_x + n, 0, sizeof(double) * kDriftHalfWidth);
  cudaStream_t st = e->stream;
  // a fresh state: position 0, zeros before the signal
  RYK_CUDA(cudaMemsetAsync(d_st, 0, 2 * sizeof(DriftState), st));
  RYK_CUDA(cudaMemsetAsync(d_hist, 0, 2 * kDriftTaps * sizeof(double), st));
  RYK_CUDA(cudaMemcpyAsync(d_table, h_table, sizeof(double) * kDriftTable, cudaMemcpyHostToDevice, st));
  RYK_CUDA(cudaMemcpyAsync(d_x, h_x, sizeof(double) * len, cudaMemcpyHostToDevice, st));
  if (drift_launch(d_st, d_st + 1, d_hist, d_hist + kDriftTaps, d_x, len, drift_inc(ppm), d_table, d_y, cap, st)) return -1;
  RYK_CUDA(cudaMemcpyAsync(h_st, d_st + 1, sizeof(DriftState), cudaMemcpyDeviceToHost, st));
  RYK_CUDA(cudaMemcpyAsync(h_y, d_y, sizeof(double) * cap, cudaMemcpyDeviceToHost, st));
  RYK_CUDA(cudaStreamSynchronize(st));
  memcpy(y, h_y, sizeof(double) * h_st->count);
  *n_out = (int)h_st->count;
  return 0;
}

// ---- snapshot and restore (DESIGN.md §4l): DCNF (ryk_snapshot_drift, then the table), DSTA (DriftSnap), DHIS (the 2W kept samples).
static size_t drift_blob_size() {
  return snap_size({sizeof(ryk_snapshot_drift) + sizeof(double) * kDriftTable, sizeof(DriftSnap), sizeof(double) * kDriftTaps});
}

int ryk_drift_snapshot_size(ryk_engine* h, int id, size_t* bytes) {
  RYK_CHECK(get_drift(&h->impl, id) != nullptr && bytes != nullptr, "no such drift object");
  *bytes = drift_blob_size();
  return 0;
}

int ryk_drift_snapshot(ryk_engine* h, int id, void* buf, size_t bytes) {
  Engine* e = &h->impl;
  Drift* D = get_drift(e, id);
  RYK_CHECK(D != nullptr && buf != nullptr, "no such drift object");
  RYK_CHECK(bytes == drift_blob_size(), "the buffer must be exactly ryk_drift_snapshot_size bytes");
  RYK_CUDA(cudaSetDevice(e->device));
  const int p = (int)(D->pushed & 1);
  DriftState* st;
  double* hist;
  if (engine_pinned_layout(e, [&](Arena& a) { st = a.take<DriftState>(1); hist = a.take<double>(kDriftTaps); })) return -1;
  RYK_CUDA(cudaMemcpyAsync(st, D->d_state + p, sizeof(DriftState), cudaMemcpyDeviceToHost, e->stream));
  RYK_CUDA(cudaMemcpyAsync(hist, D->d_hist[p], sizeof(double) * kDriftTaps, cudaMemcpyDeviceToHost, e->stream));
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  ryk_snapshot_drift c;
  memset(&c, 0, sizeof(c));
  c.max_in = D->max_in; c.phases = kDriftPhases; c.half_width = kDriftHalfWidth; c.max_ppm = D->max_ppm; c.pushed = D->pushed;
  const DriftSnap s = {st->pos, st->consumed, st->produced, D->inc, D->ppm};
  uint8_t* cur = snap_begin(buf, kSnapDrift);
  uint8_t* conf = snap_section(&cur, snap_tag("DCNF"), sizeof(c) + sizeof(double) * kDriftTable);
  memcpy(conf, &c, sizeof(c));
  memcpy(conf + sizeof(c), D->table.data(), sizeof(double) * kDriftTable);
  memcpy(snap_section(&cur, snap_tag("DSTA"), sizeof(s)), &s, sizeof(s));
  memcpy(snap_section(&cur, snap_tag("DHIS"), sizeof(double) * kDriftTaps), hist, sizeof(double) * kDriftTaps);
  snap_finish(buf, bytes);
  return 0;
}

int ryk_drift_restore(ryk_engine* h, const void* buf, size_t bytes, int* drift_id) {
  Engine* e = &h->impl;
  RYK_CHECK(drift_id != nullptr, "null argument");
  uint32_t kind = 0, version = 0;
  std::vector<SnapSection> sec;
  if (const char* refusal = snap_parse(buf, bytes, &kind, &version, &sec)) { set_error(refusal); return -2; }
  RYK_CHECK(kind == kSnapDrift, "not a drift snapshot");
  RYK_CHECK(sec.size() == 3 && sec[0].tag == snap_tag("DCNF") && sec[0].bytes == sizeof(ryk_snapshot_drift) + sizeof(double) * kDriftTable &&
                sec[1].tag == snap_tag("DSTA") && sec[1].bytes == sizeof(DriftSnap) && sec[2].tag == snap_tag("DHIS") &&
                sec[2].bytes == sizeof(double) * kDriftTaps,
            "malformed drift snapshot");
  ryk_snapshot_drift c;
  DriftSnap s;
  memcpy(&c, sec[0].data, sizeof(c));
  memcpy(&s, sec[1].data, sizeof(s));
  std::vector<double> table(kDriftTable), hist(kDriftTaps);
  memcpy(table.data(), sec[0].data + sizeof(c), sizeof(double) * kDriftTable);
  memcpy(hist.data(), sec[2].data, sizeof(double) * kDriftTaps);
  RYK_CHECK(c.max_in > 0 && c.max_in <= kDriftMaxIn && isfinite(c.max_ppm) && c.max_ppm > 0.0 && c.max_ppm <= kDriftMaxPpm && c.pushed >= 0,
            "malformed drift snapshot: its configuration");
  if (int rc = drift_check_table(table.data(), c.phases, c.half_width)) return rc;
  if (int rc = drift_check_ppm(s.ppm, c.max_ppm)) return rc;
  RYK_CHECK(s.inc == drift_inc(s.ppm) && s.pos >= 0 && s.pos < 2 * kOne && s.consumed >= 0 && s.produced >= 0,
            "malformed drift snapshot: its state");
  for (double v : hist) RYK_CHECK(isfinite(v), "malformed drift snapshot: its history");
  int id = -1;
  if (int rc = ryk_drift_create(h, c.max_in, c.max_ppm, table.data(), c.phases, c.half_width, &id)) return rc;
  Drift* D = e->drifts[id];
  const int p = (int)(c.pushed & 1);   // the parity the next push reads
  DriftState st = {s.pos, s.consumed, s.produced, s.inc, 0};
  const cudaError_t err[3] = {cudaMemcpyAsync(D->d_state + p, &st, sizeof(st), cudaMemcpyHostToDevice, e->stream),
                              cudaMemcpyAsync(D->d_hist[p], hist.data(), sizeof(double) * kDriftTaps, cudaMemcpyHostToDevice, e->stream),
                              cudaStreamSynchronize(e->stream)};
  for (cudaError_t x : err)
    if (x != cudaSuccess) {
      const std::string cause = std::string("drift restore copy failed: ") + cudaGetErrorString(x);
      ryk_drift_destroy(h, id);
      set_error(cause);
      return -1;
    }
  *D->h_state = st;
  D->ppm = s.ppm; D->inc = s.inc;
  D->pushed = c.pushed;
  *drift_id = id;
  return 0;
}

}  // extern "C"
