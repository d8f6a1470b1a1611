// agc.cu -- the automatic gain control (DESIGN.md §4j, DECIDE A1-A4) of a streaming session's model-rate input, after the frame stage
// of noise suppression and echo cancellation and ahead of the wave slide, and the whole-signal ryk_agc.  In FP64 on the input x:
//   P_m = (x[mB]^2 + ... + x[mB + B - 1]^2) / B, summed in ascending order from 0.0 (blocks of B = 256 at global positions)
//   on an active block (P_m > Gt): E = P_m for the first one, else E += a (P_m - E);
//                                  g_m = min(max(min(max(sqrt(T / E), 1 / gmax), gmax), g_{m-1} s_dn), g_{m-1} s_up)
//   on an inactive block:          E and g_m = g_{m-1} stay                                           (g_m = 1 for m < 0)
//   z[t] = (float)((g_{m-2} + (g_{m-1} - g_{m-2}) ((j + 1) / B)) x[t]),  t = mB + j
// Every sample uses the gains of the two blocks completed before its own, so the gain adds no delay, and the recursion over blocks
// carries E and g from step to step: a stream cut into steps gives the whole signal's bits.  One kernel per step, one CTA:
//   phase 1  P of each block that completes in the step, one thread per block (the first continues the kept history)
//   phase 2  thread 0 runs the recursion over them in order and writes the next step's state and the meter
//   phase 3  every thread applies the ramped gain to its samples
// Every floating-point operation is an explicit round-to-nearest intrinsic, so nothing can be contracted into an FMA and the device
// matches an FP64 numpy restatement bit for bit (DESIGN.md §5, lesson 2).
#include <math.h>
#include <string.h>
#include <algorithm>

#include "../../include/ryk.h"
#include "agc.h"
#include "engine.h"

namespace ryk {

constexpr int kAgcPiece = 1 << 18;  // ryk_agc: samples per launch (a shared array of 1026 gains)

// blocks that complete in a step of n samples: floor((r + n) / B) with r < B, at most (B - 1 + n) / B
static int agc_max_blocks(int n) { return (kAgcBlock - 1 + n) / kAgcBlock; }

__global__ void __launch_bounds__(kAgcThreads) k_agc(const AgcParams* __restrict__ par, const AgcState* __restrict__ st,
                                                     AgcState* __restrict__ st_next, const float* __restrict__ x, int n,
                                                     float* __restrict__ z, AgcMeter* __restrict__ meter) {
  extern __shared__ double sg[];    // sg[0] = g_{m0-2}, sg[1] = g_{m0-1}, sg[2 + i]: P, then g, of block m0 + i
  const long long pos = st->pos;
  const long long m0 = pos / kAgcBlock;     // the block of the step's first sample
  const int r = (int)(pos - m0 * kAgcBlock); // its samples before the step, in st->hist
  const int nc = (r + n) / kAgcBlock;       // blocks that complete in the step
  for (int i = threadIdx.x; i < nc; i += blockDim.x) {
    const int base = i * kAgcBlock - r;     // step index of the block's first sample
    double acc = 0.0;
#pragma unroll 8
    for (int j = 0; j < kAgcBlock; ++j) {
      const double v = (double)(base + j < 0 ? st->hist[j] : x[base + j]);
      acc = __dadd_rn(acc, __dmul_rn(v, v));
    }
    sg[2 + i] = __ddiv_rn(acc, (double)kAgcBlock);
  }
  // the next step's history: the (r + n) % B samples of the block in progress at its end
  const int r_next = (r + n) % kAgcBlock;
  for (int j = threadIdx.x; j < r_next; j += blockDim.x) {
    const int t = nc * kAgcBlock + j - r;   // negative only when no block completes: then the sample is in the kept history
    st_next->hist[j] = t < 0 ? st->hist[j] : x[t];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const AgcParams P = *par;
    double E = st->level, g = st->g1;
    int started = st->started, active = 0;
    sg[0] = st->g2;
    sg[1] = g;
    for (int i = 0; i < nc; ++i) {
      const double p = sg[2 + i];
      if (p > P.gate) {
        E = started ? __dadd_rn(E, __dmul_rn(P.a, __dsub_rn(p, E))) : p;
        started = 1;
        ++active;
        const double want = fmin(fmax(__dsqrt_rn(__ddiv_rn(P.target, E)), P.ginv), P.gmax);
        g = fmin(fmax(want, __dmul_rn(g, P.s_dn)), __dmul_rn(g, P.s_up));
      }
      sg[2 + i] = g;
    }
    st_next->pos = pos + n;
    st_next->level = E;
    st_next->started = started;
    st_next->g1 = sg[nc + 1];
    st_next->g2 = sg[nc];
    meter->level = E;
    meter->gain = g;
    meter->started = started;
    meter->active = active;
  }
  __syncthreads();
  for (int t = threadIdx.x; t < n; t += blockDim.x) {
    const long long s = pos + t, m = s / kAgcBlock;
    const int i = (int)(m - m0), j = (int)(s - m * kAgcBlock);
    const double ga = sg[i], gb = sg[i + 1];
    const double g = __dadd_rn(ga, __dmul_rn(__dsub_rn(gb, ga), __ddiv_rn((double)(j + 1), (double)kAgcBlock)));
    z[t] = (float)__dmul_rn(g, (double)x[t]);
  }
}

int agc_check(double target_db, double max_gain_db, double gate_db) {
  RYK_CHECK(isfinite(target_db) && target_db >= -40.0 && target_db <= -6.0, "target_db must be finite and within [-40, -6]");
  RYK_CHECK(isfinite(max_gain_db) && max_gain_db >= 0.0 && max_gain_db <= 30.0, "max_gain_db must be finite and within [0, 30]");
  RYK_CHECK(isfinite(gate_db) && gate_db >= -80.0 && gate_db <= -20.0, "gate_db must be finite and within [-80, -20]");
  return 0;
}

AgcParams agc_params(int fs, double target_db, double max_gain_db, double gate_db) {
  AgcParams p;
  p.target = pow(10.0, target_db / 10.0);
  p.gate = pow(10.0, gate_db / 10.0);
  p.gmax = pow(10.0, max_gain_db / 20.0);
  p.ginv = 1.0 / p.gmax;
  p.a = -expm1(-(double)kAgcBlock / (0.4 * fs));
  p.s_up = pow(10.0, 6.0 * kAgcBlock / (20.0 * fs));
  p.s_dn = pow(10.0, -24.0 * kAgcBlock / (20.0 * fs));
  return p;
}

void agc_state_init(AgcState* st) {
  memset(st, 0, sizeof(*st));
  st->g1 = st->g2 = 1.0;
}

void agc_meter_init(AgcMeter* m) {
  memset(m, 0, sizeof(*m));
  m->gain = 1.0;
}

int agc_run(const AgcWork& w, const AgcState* st, AgcState* st_next, const float* d_x, int n, float* d_z, cudaStream_t stream) {
  const size_t smem = sizeof(double) * (agc_max_blocks(n) + 2);
  k_agc<<<1, kAgcThreads, smem, stream>>>(w.params, st, st_next, d_x, n, d_z, w.meter);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace ryk

using namespace ryk;

extern "C" {

// The whole-signal gain control: from a fresh state, pieces of kAgcPiece samples that carry the state from one to the next, as the
// steps of a session do.
int ryk_agc(ryk_engine* h, const float* x, int n, int fs, double target_db, double max_gain_db, double gate_db, float* z) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(x && z && n > 0, "null argument or empty signal");
  RYK_CHECK(fs > 0, "fs must be positive");
  if (int rc = agc_check(target_db, max_gain_db, gate_db)) return rc;
  AgcWork w;
  AgcState* st[2];
  float *d_x, *d_z;
  if (engine_scratch(e, [&](Arena& a) {
        w.params = a.take<AgcParams>(1);
        w.meter = a.take<AgcMeter>(1);
        st[0] = a.take<AgcState>(1);
        st[1] = a.take<AgcState>(1);
        d_x = a.take<float>(n);
        d_z = a.take<float>(n);
      })) return -1;
  // host staging: the settings, a fresh state and x
  AgcParams* h_par;
  AgcState* h_st;
  float* h_x;
  if (engine_pinned_layout(e, [&](Arena& a) { h_par = a.take<AgcParams>(1); h_st = a.take<AgcState>(1); h_x = a.take<float>(n); })) return -1;
  *h_par = agc_params(fs, target_db, max_gain_db, gate_db);
  agc_state_init(h_st);
  memcpy(h_x, x, sizeof(float) * n);
  cudaStream_t s = e->stream;
  RYK_CUDA(cudaMemcpyAsync(w.params, h_par, sizeof(AgcParams), cudaMemcpyHostToDevice, s));
  RYK_CUDA(cudaMemcpyAsync(st[0], h_st, sizeof(AgcState), cudaMemcpyHostToDevice, s));
  RYK_CUDA(cudaMemcpyAsync(d_x, h_x, sizeof(float) * n, cudaMemcpyHostToDevice, s));
  for (int a = 0, k = 0; a < n; a += kAgcPiece, k ^= 1)
    if (agc_run(w, st[k], st[k ^ 1], d_x + a, std::min(kAgcPiece, n - a), d_z + a, s)) return -1;
  RYK_CUDA(cudaMemcpyAsync(z, d_z, sizeof(float) * n, cudaMemcpyDeviceToHost, s));
  RYK_CUDA(cudaStreamSynchronize(s));
  return 0;
}

}  // extern "C"
