// drift.h -- the clock drift stage: an asynchronous resampler on the played stream whose ratio the host trims between chunks
// (drift.cu; DESIGN.md §4l, DECIDE D1-D4).
#pragma once
#include "common.cuh"

namespace ryk {

struct Engine;
struct Drift;

constexpr int kDriftPhases = 512;                                   // D3: phases per input sample (the top 9 bits of the fraction)
constexpr int kDriftHalfWidth = 16;                                 // D3: W, half-width in input samples: 2W taps per output
constexpr int kDriftTaps = 2 * kDriftHalfWidth;
constexpr int kDriftTable = 2 * kDriftHalfWidth * kDriftPhases + 1; // prototype filter entries, t = k / P - W for k = 0 .. 2WP
constexpr int kDriftMaxIn = 1 << 24;                                // most samples of one push: n 2^32 stays far below 2^63
constexpr double kDriftMaxPpm = 2000.0;

// The stream position one push reads and the next push's copy it writes (double-buffered by push parity).
struct DriftState {
  long long pos;          // read position of the next output in 2^-32 samples, relative to the samples consumed: in [0, inc)
  long long consumed;     // input samples pushed since creation
  long long produced;     // outputs emitted since creation
  long long inc;          // the increment of the push that wrote this state
  long long count;        // outputs of that push
};

// inc = llrint(2^32 / (1 + ppm 1e-6)) (D2)
long long drift_inc(double ppm);
// the documented bound of one push's outputs: n + ceil(n max_ppm 1e-6) + 2
long long drift_capacity(long long n, double max_ppm);
void drift_destroy_all(Engine* e);

}  // namespace ryk
