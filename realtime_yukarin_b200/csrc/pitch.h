// pitch.h -- pitch correction of a streaming session's converted f0 and the whole-signal ryk_pitch_correct (pitch.cu; DESIGN.md §4m,
// DECIDE P1-P4).
#pragma once
#include "common.cuh"

namespace ryk {

constexpr double kPitchHold = 0.5 + 0.15;   // P1: the previous target is kept while |s - n_prev| is under this many semitones
constexpr int kPitchNoNote = -(1 << 28);    // n_prev before the first voiced frame: no s is within kPitchHold of it

// What the host sets: written only by host-to-device copies.  The settings as given, and the glide coefficient they make at the
// stream's frame period.
struct PitchParams {
  double a4;                          // Hz of MIDI note 69, in [400, 480]
  double log2_a4;                     // its log2, computed with the host's libm
  double retune_ms;                   // in [0, 1000]; 0 is a hard snap
  double amount;                      // in [0, 1]; 0 returns the input bit for bit
  double beta;                        // -expm1(-hop_ms / retune_ms), 1 when retune_ms is 0 (P2)
  int key;                            // pitch class of the scale's root, 0 (C) .. 11 (B)
  int scale;                          // 12-bit mask: bit j set when pitch class (key + j) mod 12 is in the scale
};
// The recursion state and the meter of the last launch, one block per session updated in place (every step's decode slide runs on
// stream D in step order).
struct PitchState {
  double c;                           // the correction of the last voiced frame, in semitones (P2)
  int n_prev;                         // its target note (kPitchNoNote before the first voiced frame)
  int voiced_prev;                    // the last frame was voiced
  long long voiced;                   // meter: voiced frames of the last launch
  double sum_cents, max_cents;        // ... and the sum and largest of |amount c| over them, in cents
};
struct PitchWork {
  PitchParams* params = nullptr;
  PitchState* state = nullptr;
};

// refuses settings that are not finite or out of range, and an empty scale
int pitch_check(int key, int scale, double a4_hz, double retune_ms, double amount);
// the device block of the settings at frame period hop_ms (P2), computed with the host's libm
PitchParams pitch_params(double hop_ms, int key, int scale, double a4_hz, double retune_ms, double amount);
// a fresh state: no voiced frame yet, an empty meter
void pitch_state_init(PitchState* st);
// n frames of f0 in d_f0, corrected in place in stream order, continuing the recursion in *w.state.  One kernel, one CTA; n is fixed and
// the settings are read on the device, so the launch can sit in a captured graph.
int pitch_run(const PitchWork& w, float* d_f0, int n, cudaStream_t stream);
int pitch_run(const PitchWork& w, double* d_f0, int n, cudaStream_t stream);

}  // namespace ryk
