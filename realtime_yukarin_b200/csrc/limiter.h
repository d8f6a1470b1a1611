// limiter.h -- the look-ahead peak limiter on a streaming session's output and the whole-signal ryk_limit (limiter.cu; DESIGN.md §4i,
// DECIDE L1-L4).
#pragma once
#include "common.cuh"

namespace ryk {

struct Engine;

// What the host sets: written only by host-to-device copies.
struct LimParams {
  double ceiling;                     // c = 10^(ceiling_db / 20)
  double gain;                        // G: the ceiling applies to G y (L1)
};
// The stream position one step reads and the next step's copy it writes (double-buffered by step parity).
struct LimState {
  long long pos;                      // samples of y received before the step
};
// What the last step measured (L4): the smallest gain of its samples as the bits of a positive double (they order like the value, so
// an integer atomicMin takes the exact minimum) and how many of them had a gain below 1.
struct LimMeter {
  unsigned long long min_bits;
  unsigned long long limited;
};
// The history one step reads from its parity and writes for the next step into the other parity's.
struct LimHist {
  double* g0 = nullptr;               // [R + 2L - 1]: g0 of the samples before pos
  double* y = nullptr;                // [L]: y of the samples before pos
  LimState* st = nullptr;
};
// One limiter's shape, settings, meter and per-step scratch (a session's, or a whole-signal call's).
struct LimWork {
  int L = 0, R = 0;                   // look-ahead and hold in samples (L1)
  int max_n = 0;                      // most samples one step can bring
  LimParams* params = nullptr;
  LimMeter* meter = nullptr;
  double* g0 = nullptr;               // [R + 2L - 1 + max_n]: the step's g0 window, history first
  double* t32 = nullptr;              // minima of its tiles of 32 samples
  double* t1k = nullptr;              // ... and of 1024 samples
  double* m = nullptr;                // [max_n + L - 1]: the windowed minima m[s] the step's box sums read
};

// refuses a non-finite look-ahead outside [0.5, 10] ms or hold outside [0, 500] ms
int limiter_check_shape(double lookahead_ms, double hold_ms);
// refuses a non-finite ceiling outside [-24, 0] dB or a gain that is not finite and positive
int limiter_check_settings(double ceiling_db, double gain);
// L = max(1, round(lookahead_ms * rate / 1000)), R = round(hold_ms * rate / 1000), rounded half to even
void limiter_shape(int rate, double lookahead_ms, double hold_ms, int* L, int* R);
// the device block of the settings (L1)
LimParams limiter_params(double ceiling_db, double gain);
// elements of the scratch arrays of w's shape: g0, t32, t1k, m
void limiter_scratch_sizes(const LimWork& w, size_t* n_g0, size_t* n_t32, size_t* n_t1k, size_t* n_m);
// One step: *d_n (at most w.max_n) new samples of y in d_y -> as many samples of concat(zeros(L), z) in d_z.  Three kernels; every
// size is fixed and the sample count and stream position are read on the device, so the launches can sit in a captured graph.
int limiter_run(const LimWork& w, const LimHist& cur, const LimHist& next, const double* d_y, const int* d_n, double* d_z,
                cudaStream_t stream);

}  // namespace ryk
