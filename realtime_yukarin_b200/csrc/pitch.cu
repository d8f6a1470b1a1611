// pitch.cu -- pitch correction (DESIGN.md §4m, DECIDE P1-P4) of the converted f0 a streaming session hands its synthesizer, and the
// whole-signal ryk_pitch_correct.  In FP64 on the frames f0 (0: unvoiced), in stream order:
//   P1  a voiced frame (0 < f0 < inf) sits at s = 69 + 12 (log2 f0 - log2 a4) MIDI semitones (finite for every such f0); its target n is the nearest note whose pitch
//       class (n - key) mod 12 is in the scale (ties to the lower note), unless the previous target n_prev is still in the scale and
//       |s - n_prev| < 0.5 + 0.15, which keeps n = n_prev: a note sung between two scale notes does not flap between them
//   P2  d = n - s;  c = d on the first voiced frame after an unvoiced one (no glide from a stale note), else c += beta (d - c),
//       beta = -expm1(-hop_ms / retune_ms) (1 for retune_ms = 0: a hard snap)
//   P3  f0' = f0 exp2(amount c / 12); amount = 0 gives f0 bit for bit.  Any other frame is returned as it is and keeps c and n_prev.
//   P4  a session corrects the n_feat rows each step's decode slide appends to its decode window, once each, in the dec_slide graph on
//       stream D; later slides carry them on unchanged and the synthesizer's FP64 copy of the window reads them (session.cu).
// One kernel per step, one CTA, over tiles of kPitchTile frames:
//   phase 1  every thread takes s and the nearest scale note of its frames (the independent work: log2 and the scale search)
//   phase 2  thread 0 runs the hysteresis and the glide over the tile in order, and the meter
//   phase 3  every thread applies the correction to its frames
// The recursion is written with explicit round-to-nearest intrinsics, so nothing can be contracted into an FMA (DESIGN.md §5, lesson
// 2): a stream cut into steps gives the whole signal's bits, and a session gives those of the whole-signal call.
#include <math.h>
#include <string.h>

#include "../../include/ryk.h"
#include "engine.h"
#include "pitch.h"

namespace ryk {

constexpr int kPitchThreads = 256;
constexpr int kPitchTile = 1024;            // frames per pass of the three phases (shared: 12 KB)

__device__ __forceinline__ bool pitch_voiced(double f) { return f > 0.0 && f < HUGE_VAL; }
__device__ __forceinline__ int pitch_in_scale(int n, int key, int scale) { return (scale >> (((n - key) % 12 + 12) % 12)) & 1; }

template <typename T>
__global__ void __launch_bounds__(kPitchThreads) k_pitch(const PitchParams* __restrict__ par, PitchState* __restrict__ st,
                                                         T* __restrict__ f0, int n) {
  __shared__ double ss[kPitchTile];         // s of each voiced frame, then its correction c
  __shared__ int sn[kPitchTile];            // its nearest scale note
  const PitchParams P = *par;
  double c = 0.0, sum = 0.0, mx = 0.0;
  int n_prev = 0, voiced_prev = 0;
  long long voiced = 0;
  if (threadIdx.x == 0) { c = st->c; n_prev = st->n_prev; voiced_prev = st->voiced_prev; }
  for (int base = 0; base < n; base += kPitchTile) {
    const int m = min(kPitchTile, n - base);
    for (int i = threadIdx.x; i < m; i += blockDim.x) {
      const double f = (double)f0[base + i];
      if (!pitch_voiced(f)) continue;
      const double s = __dadd_rn(69.0, __dmul_rn(12.0, __dsub_rn(log2(f), P.log2_a4)));
      // every 12 consecutive notes hold a scale note, so the nearest is within 6 of s: in [floor(s) - 6, floor(s) + 7]
      const int lo = (int)floor(s);
      int best = lo;
      double bd = HUGE_VAL;
      for (int k = lo - 6; k <= lo + 7; ++k) {
        if (!pitch_in_scale(k, P.key, P.scale)) continue;
        const double dist = fabs(__dsub_rn(s, (double)k));
        if (dist < bd) { bd = dist; best = k; }          // ascending k, strictly nearer: a tie keeps the lower note
      }
      ss[i] = s;
      sn[i] = best;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int i = 0; i < m; ++i) {
        if (!pitch_voiced((double)f0[base + i])) { voiced_prev = 0; continue; }
        const double s = ss[i];
        int note = sn[i];
        if (pitch_in_scale(n_prev, P.key, P.scale) && fabs(__dsub_rn(s, (double)n_prev)) < kPitchHold) note = n_prev;
        const double d = __dsub_rn((double)note, s);
        c = voiced_prev ? __dadd_rn(c, __dmul_rn(P.beta, __dsub_rn(d, c))) : d;
        n_prev = note;
        voiced_prev = 1;
        ss[i] = c;
        const double cents = __dmul_rn(fabs(__dmul_rn(P.amount, c)), 100.0);
        ++voiced;
        sum = __dadd_rn(sum, cents);
        mx = fmax(mx, cents);
      }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < m; i += blockDim.x) {
      const double f = (double)f0[base + i];
      if (pitch_voiced(f)) f0[base + i] = (T)__dmul_rn(f, exp2(__ddiv_rn(__dmul_rn(P.amount, ss[i]), 12.0)));
    }
    __syncthreads();                        // the next tile's phase 1 overwrites ss and sn
  }
  if (threadIdx.x == 0) {
    st->c = c; st->n_prev = n_prev; st->voiced_prev = voiced_prev;
    st->voiced = voiced; st->sum_cents = sum; st->max_cents = mx;
  }
}

int pitch_check(int key, int scale, double a4_hz, double retune_ms, double amount) {
  RYK_CHECK(key >= 0 && key <= 11, "key must be a pitch class within [0, 11] (0 is C)");
  RYK_CHECK(scale >= 1 && scale <= 0xfff, "the scale must be a nonzero 12-bit mask of pitch classes");
  RYK_CHECK(isfinite(a4_hz) && a4_hz >= 400.0 && a4_hz <= 480.0, "a4_hz must be finite and within [400, 480]");
  RYK_CHECK(isfinite(retune_ms) && retune_ms >= 0.0 && retune_ms <= 1000.0, "retune_ms must be finite and within [0, 1000]");
  RYK_CHECK(isfinite(amount) && amount >= 0.0 && amount <= 1.0, "amount must be finite and within [0, 1]");
  return 0;
}

PitchParams pitch_params(double hop_ms, int key, int scale, double a4_hz, double retune_ms, double amount) {
  PitchParams p;
  p.a4 = a4_hz;
  p.log2_a4 = log2(a4_hz);
  p.retune_ms = retune_ms;
  p.amount = amount;
  p.beta = retune_ms == 0.0 ? 1.0 : -expm1(-hop_ms / retune_ms);
  p.key = key;
  p.scale = scale;
  return p;
}

void pitch_state_init(PitchState* st) {
  memset(st, 0, sizeof(*st));
  st->n_prev = kPitchNoNote;
}

template <typename T>
static int pitch_launch(const PitchWork& w, T* d_f0, int n, cudaStream_t stream) {
  k_pitch<T><<<1, kPitchThreads, 0, stream>>>(w.params, w.state, d_f0, n);
  RYK_CUDA(cudaGetLastError());
  return 0;
}
int pitch_run(const PitchWork& w, float* d_f0, int n, cudaStream_t stream) { return pitch_launch(w, d_f0, n, stream); }
int pitch_run(const PitchWork& w, double* d_f0, int n, cudaStream_t stream) { return pitch_launch(w, d_f0, n, stream); }

}  // namespace ryk

using namespace ryk;

extern "C" {

// The whole-signal correction: one launch over every frame from a fresh state, on the kernel a session runs.
int ryk_pitch_correct(ryk_engine* h, const double* f0, int n, int fs, double frame_period, int key, int scale_mask, double a4_hz,
                      double retune_ms, double amount, double* out) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(f0 && out && n > 0, "null argument or empty signal");
  RYK_CHECK(fs > 0, "fs must be positive");
  RYK_CHECK(isfinite(frame_period) && frame_period > 0.0, "frame_period must be finite and positive");
  if (int rc = pitch_check(key, scale_mask, a4_hz, retune_ms, amount)) return rc;
  PitchWork w;
  double* d_f0;
  if (engine_scratch(e, [&](Arena& a) { w.params = a.take<PitchParams>(1); w.state = a.take<PitchState>(1); d_f0 = a.take<double>(n); }))
    return -1;
  PitchParams* h_par;
  PitchState* h_st;
  double* h_f0;
  if (engine_pinned_layout(e, [&](Arena& a) { h_par = a.take<PitchParams>(1); h_st = a.take<PitchState>(1); h_f0 = a.take<double>(n); }))
    return -1;
  *h_par = pitch_params(frame_period, key, scale_mask, a4_hz, retune_ms, amount);
  pitch_state_init(h_st);
  memcpy(h_f0, f0, sizeof(double) * n);
  cudaStream_t s = e->stream;
  RYK_CUDA(cudaMemcpyAsync(w.params, h_par, sizeof(PitchParams), cudaMemcpyHostToDevice, s));
  RYK_CUDA(cudaMemcpyAsync(w.state, h_st, sizeof(PitchState), cudaMemcpyHostToDevice, s));
  RYK_CUDA(cudaMemcpyAsync(d_f0, h_f0, sizeof(double) * n, cudaMemcpyHostToDevice, s));
  if (pitch_run(w, d_f0, n, s)) return -1;
  RYK_CUDA(cudaMemcpyAsync(out, d_f0, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
  RYK_CUDA(cudaStreamSynchronize(s));
  return 0;
}

}  // extern "C"
