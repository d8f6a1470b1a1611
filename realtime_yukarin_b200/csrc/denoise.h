// denoise.h -- input noise suppression of a streaming session and of the whole-signal ryk_denoise (denoise.cu; DESIGN.md §4f,
// DECIDE N1-N3).
#pragma once
#include "common.cuh"

namespace ryk {

struct Engine;

constexpr int kDnN = 512;                   // frame length (N1)
constexpr int kDnHop = 128;                 // hop (N1)
constexpr int kDnBins = kDnN / 2 + 1;       // rfft bins
constexpr int kDnDelay = kDnN - 1;          // model samples a session delays its filtered input by (N3)
constexpr double kDnAlpha = 0.98;           // decision-directed smoothing (N2)

// What the host sets: written only by host-to-device copies (a learning kernel never writes here, so a host copy never overwrites what
// the device learned).  A serial that differs from the one the device last applied marks a new request.
struct DenoiseParams {
  double gain_floor;                  // g = 10^(-reduction_db / 20)
  long long profile_serial;           // phi below is a new profile
  long long learn_serial, learn_frames;   // learn from the next learn_frames frames (0: cancel a learning in progress)
  double phi[kDnBins];
};
// What the device owns: written only by the gain scan.
struct DenoiseLearn {
  long long profile_serial, learn_serial;   // the host requests already applied
  long long remaining, total;               // frames still to learn, frames of the learning
  double sum[kDnBins];                      // per-bin power sums of the frames learned so far
  double phi[kDnBins];                      // the noise profile in use
};
// The stream state one step reads and the next step's copy it writes (double-buffered by step parity).
struct DenoiseState {
  long long in_end;                   // model samples received before the step
  double gain[kDnBins], power[kDnBins];   // G and P of the last frame processed (G_{-1} = 1, P_{-1} = 0)
  double carry[kDnDelay];             // overlap-add sums of the samples not yet emitted, from in_end - kDnDelay on
  float hist[kDnDelay];               // the last kDnDelay input samples before in_end
};
// Per-step scratch of one filter (a session's, or a whole-signal call's).
struct DenoiseWork {
  DenoiseParams* params = nullptr;
  DenoiseLearn* learn = nullptr;
  double2* spec = nullptr;            // [max_frames][kDnBins]: X_m, then G_m X_m
  double* frames = nullptr;           // [max_frames][kDnN]: windowed inverse transforms
  unsigned* done = nullptr;           // CTAs of the inverse kernel finished (the last one overlap-adds and resets it)
  int max_frames = 0;
};

// frames a step of n samples can hold: floor((k + 1) n / H) - floor(k n / H) <= ceil(n / H)
inline int denoise_max_frames(int n) { return (n + kDnHop - 1) / kDnHop; }
// the state of a fresh filter: G_{-1} = 1, everything else zero
void denoise_state_init(DenoiseState* host);
// refuses a reduction outside [0, 40] dB or a profile (phi: kDnBins values, may be null) with a negative or non-finite entry
int denoise_check(double reduction_db, const double* phi);
// One step: n new samples in d_x -> n filtered samples in d_z, delayed by kDnDelay.  Three kernels (forward transforms, gain scan,
// inverse transforms + overlap-add); every size is fixed, the frame range is read from st on the device, so the launches can sit in a
// captured graph.  denoise_run is the three launches below in order; the echo canceller runs its own scan between the first and last.
int denoise_run(Engine* e, const DenoiseWork& w, const DenoiseState* st, DenoiseState* st_next, const float* d_x, int n, float* d_z,
                cudaStream_t stream);
// k_dn_forward: X_m of the step's frames into spec ([max_frames][kDnBins]); writes st_next's history and in_end
int denoise_forward(Engine* e, int max_frames, const DenoiseState* st, DenoiseState* st_next, const float* d_x, int n, double2* spec,
                    cudaStream_t stream);
// k_dn_scan: the gain recursion on w.spec
int denoise_scan(const DenoiseWork& w, const DenoiseState* st, DenoiseState* st_next, int n, cudaStream_t stream);
// k_dn_inverse: inverse transforms of w.spec and the ordered overlap-add into d_z
int denoise_inverse(Engine* e, const DenoiseWork& w, const DenoiseState* st, DenoiseState* st_next, int n, float* d_z, cudaStream_t stream);

}  // namespace ryk
