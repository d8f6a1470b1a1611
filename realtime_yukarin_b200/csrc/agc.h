// agc.h -- the automatic gain control of a streaming session's model-rate input and the whole-signal ryk_agc (agc.cu; DESIGN.md §4j,
// DECIDE A1-A4).
#pragma once
#include "common.cuh"

namespace ryk {

constexpr int kAgcBlock = 256;              // B: model samples per level block (A1)
constexpr int kAgcThreads = 1024;           // k_agc: one CTA per step

// What the host sets (A2): written only by host-to-device copies.
struct AgcParams {
  double target;                      // T = 10^(target_db / 10), a mean square
  double gate;                        // Gt = 10^(gate_db / 10): a block is active when its mean square exceeds it
  double gmax, ginv;                  // 10^(max_gain_db / 20) and 1 / gmax
  double a;                           // level smoothing -expm1(-B / (0.4 s fs))
  double s_up, s_dn;                  // gain slew per block: 10^(6 B / (20 fs)), 10^(-24 B / (20 fs))
};
// The stream state one step reads and the next step's copy it writes (double-buffered by step parity).
struct AgcState {
  long long pos;                      // model samples received before the step
  double level;                       // E (meaningful once started)
  double g1, g2;                      // gains of the last two completed blocks, g_{m-1} and g_{m-2} (1 before block 0)
  int started;                        // an active block has set E
  float hist[kAgcBlock];              // the pos % B samples of the block in progress
};
// What the last step measured (A4), one per session: written by the step's recursion.
struct AgcMeter {
  double level;                       // E after the step
  double gain;                        // the gain of the last completed block
  int started;                        // an active block has set E
  int active;                         // active blocks that completed in the step
};
struct AgcWork {
  AgcParams* params = nullptr;
  AgcMeter* meter = nullptr;
};

// refuses settings that are not finite or outside target [-40, -6], max_gain [0, 30], gate [-80, -20] dB
int agc_check(double target_db, double max_gain_db, double gate_db);
// the device block of the settings at model rate fs (A2), computed with the host's libm
AgcParams agc_params(int fs, double target_db, double max_gain_db, double gate_db);
// a fresh state (position 0, gains 1, no level) and the meter before any step
void agc_state_init(AgcState* st);
void agc_meter_init(AgcMeter* m);
// One step: n new samples of x in d_x -> n samples of z in d_z, no delay.  One kernel; n and the shared memory are fixed by n and the
// stream position is read from st on the device, so the launch can sit in a captured graph.
int agc_run(const AgcWork& w, const AgcState* st, AgcState* st_next, const float* d_x, int n, float* d_z, cudaStream_t stream);

}  // namespace ryk
