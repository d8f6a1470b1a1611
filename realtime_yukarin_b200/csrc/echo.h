// echo.h -- echo cancellation of a streaming session and of the whole-signal ryk_echo_cancel (echo.cu; DESIGN.md §4g, DECIDE E1-E4).
// It works in the frame domain of the input noise suppression (denoise.h): the same forward and inverse transforms, one more kernel.
#pragma once
#include "denoise.h"

namespace ryk {

constexpr int kAecMaxTaps = 64;             // filter length in frames (E2)
constexpr int kAecMaxDelay = 256;           // bulk delay of the far end in frames (E2)
constexpr double kAecMu = 0.5;              // NLMS step (E2)
constexpr double kAecDelta = 1e-6;          // NLMS regularisation (E2)
constexpr double kAecLambda = 0.9;          // power smoothing (E3, E4)
constexpr double kAecCopyRatio = 0.5;       // B -> F when S_b < 0.5 S_f and S_b < S_d ...
constexpr int kAecCopyFrames = 3;           // ... for 3 consecutive frames (E3)
constexpr double kAecResetRatio = 4.0;      // F -> B, no update that frame, when S_b > 4 S_f (E3)
constexpr double kAecDivergedRatio = 1.0;   // F -> 0 when S_f > S_d: F would make the output louder than the microphone (E3)
constexpr double kAecRho = 1.0;             // residual suppression G = max(g_e, 1 - rho Yhat / (Ehat + eps)) (E4)
constexpr double kAecEps = 1e-12;

// What the host sets: written only by host-to-device copies.
struct EchoParams {
  double gain_floor;                  // g_e = 10^(-suppression_db / 20)
};
// What the last step measured (ryk_session_echo_stats): per-bin sums over its frames, added on the host in bin order.
struct EchoStats {
  double sum_d[kDnBins], sum_z[kDnBins];   // sum of |D|^2 and |Z|^2
  long long frames;
};
// What the device owns: written only by k_aec_scan, in place (every step's scan runs on one stream in step order).
struct EchoFilter {
  double2 b[kDnBins][kAecMaxTaps];    // background filter B: adapts every frame
  double2 f[kDnBins][kAecMaxTaps];    // foreground filter F: produces the output
  double sb[kDnBins], sf[kDnBins], sd[kDnBins];   // smoothed |E^b|^2, |E^f|^2, |D|^2
  double yh[kDnBins], eh[kDnBins];    // smoothed |Y^f|^2, |E^f|^2 of the residual suppression
  int cnt[kDnBins];                   // consecutive frames the B -> F condition held
  EchoStats stats;
};
// One canceller's device blocks and shape.
struct EchoWork {
  EchoParams* params = nullptr;
  EchoFilter* filter = nullptr;
  double2* ring = nullptr;            // [taps + delay][kDnBins]: X_m of the far end at slot m mod (taps + delay)
  double2* far_spec = nullptr;        // [max_frames][kDnBins]: the step's far-end spectra (k_dn_forward)
  int taps = 0, delay = 0;
};

// refuses taps outside [1, 64], delay_frames outside [0, 256] or a suppression outside [0, 40] dB
int echo_check(int taps, int delay_frames, double suppression_db);
// The canceller's scan over the step's frames (frame range from st, as the noise suppression reads it): the far end's spectra in
// w.far_spec, the microphone's in spec, which it overwrites with Z.  One kernel; every size is fixed, so it can sit in a captured graph.
int echo_scan(const EchoWork& w, const DenoiseState* st, int n, double2* spec, cudaStream_t stream);

}  // namespace ryk
