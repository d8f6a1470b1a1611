// echo.cu -- echo cancellation (DESIGN.md §4g, DECIDE E1-E4): a per-bin two-path NLMS filter over the frames of the far end (the audio
// the host played), in FP64, in the frame domain of the input noise suppression (denoise.cu), ahead of the WORLD analysis of a
// streaming session and in the whole-signal ryk_echo_cancel.
//
// A step frames the microphone and the far end with k_dn_forward (each with its own DenoiseState pair), then
//   k_aec_scan    one warp per bin: the frames of the step in ascending order; Y = sum_p W_p X_{m-d-p} for the background filter B
//                 and the foreground filter F, E = D - Y, the two-path control (E3) and the residual suppression (E4); D_m <- Z_m
// then, with noise suppression on, k_dn_scan on Z, and k_dn_inverse overlap-adds the frames.  Each lane holds taps j and j + 32 of B
// and F in registers for the whole step; the sums over taps are a fixed xor butterfly, so every lane sees the same bitwise E and the
// result does not depend on launch or step boundaries.
#include <math.h>
#include <string.h>

#include "../../include/ryk.h"
#include "echo.h"
#include "engine.h"

namespace ryk {

constexpr int kAecWarps = 4;                // bins per CTA: 65 CTAs spread the 257 bins over the SMs

__device__ inline double2 cmul(double2 a, double2 b) { return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ inline double cabs2(double2 a) { return a.x * a.x + a.y * a.y; }

__global__ void __launch_bounds__(kAecWarps * 32) k_aec_scan(const EchoParams* __restrict__ par, EchoFilter* __restrict__ flt,
                                                            double2* __restrict__ ring, const double2* __restrict__ far_spec, int P, int d,
                                                            const DenoiseState* __restrict__ st, int n, double2* __restrict__ spec) {
  const int lane = threadIdx.x & 31;
  const int k = blockIdx.x * kAecWarps + (threadIdx.x >> 5);
  const long long in_end = st->in_end;
  const long long f0 = in_end / kDnHop, f1 = (in_end + n) / kDnHop;
  if (blockIdx.x == 0 && threadIdx.x == 0) flt->stats.frames = f1 - f0;
  if (k >= kDnBins) return;
  const int L = P + d;
  const bool on0 = lane < P, on1 = lane + 32 < P;
  // X_q of the far end: this step's frames from far_spec, earlier ones from the ring, zero before frame 0
  auto far_at = [&](long long q) -> double2 {
    if (q < 0) return make_double2(0.0, 0.0);
    return q >= f0 ? far_spec[(size_t)(q - f0) * kDnBins + k] : ring[(size_t)(q % L) * kDnBins + k];
  };
  const double ge = par->gain_floor, lam = kAecLambda, mix = 1.0 - kAecLambda;
  double2 B0 = flt->b[k][lane], B1 = flt->b[k][lane + 32], F0 = flt->f[k][lane], F1 = flt->f[k][lane + 32];
  double sb = flt->sb[k], sf = flt->sf[k], sd = flt->sd[k], yh = flt->yh[k], eh = flt->eh[k];
  int cnt = flt->cnt[k];
  double sum_d = 0.0, sum_z = 0.0;
  const double2 zero = make_double2(0.0, 0.0);
  // frame m + 1's loads are issued before frame m's sums: the frame loop is sequential and bound by latency
  double2 xa = on0 ? far_at(f0 - d - lane) : zero, xb = on1 ? far_at(f0 - d - lane - 32) : zero;
  double2 dn = f0 < f1 ? spec[k] : zero;
  for (long long m = f0; m < f1; ++m) {
    const double2 x0 = xa, x1 = xb, D = dn;
    if (m + 1 < f1) {
      xa = on0 ? far_at(m + 1 - d - lane) : zero;
      xb = on1 ? far_at(m + 1 - d - lane - 32) : zero;
      dn = spec[(size_t)(m + 1 - f0) * kDnBins + k];
    }
    // warp_sum (common.cuh) is an xor butterfly: every lane ends with the same bits, as a + b == b + a
    const double2 b0 = cmul(B0, x0), b1 = cmul(B1, x1), g0 = cmul(F0, x0), g1 = cmul(F1, x1);
    const double ybr = warp_sum(b0.x + b1.x), ybi = warp_sum(b0.y + b1.y);
    const double yfr = warp_sum(g0.x + g1.x), yfi = warp_sum(g0.y + g1.y);
    const double px = warp_sum(cabs2(x0) + cabs2(x1));
    const double2 Eb = make_double2(D.x - ybr, D.y - ybi), Ef = make_double2(D.x - yfr, D.y - yfi);
    sb = lam * sb + mix * cabs2(Eb);
    sf = lam * sf + mix * cabs2(Ef);
    sd = lam * sd + mix * cabs2(D);
    yh = lam * yh + mix * (yfr * yfr + yfi * yfi);
    eh = lam * eh + mix * cabs2(Ef);
    const double G = fmax(ge, 1.0 - kAecRho * yh / (eh + kAecEps));
    const double2 Z = make_double2(G * Ef.x, G * Ef.y);
    sum_d += cabs2(D);
    sum_z += cabs2(Z);
    if (lane == 0) {
      spec[(size_t)(m - f0) * kDnBins + k] = Z;
      // slot m mod L held X_{m-L}, which no frame from m on reads
      ring[(size_t)(m % L) * kDnBins + k] = far_spec[(size_t)(m - f0) * kDnBins + k];
    }
    // the filters, in the oracle's order: clear a diverged F, reset B from F (no update), else count, copy B into F, update B
    if (sf > kAecDivergedRatio * sd) { F0 = zero; F1 = zero; }
    if (sb > kAecResetRatio * sf) {
      B0 = F0; B1 = F1; cnt = 0;
    } else {
      cnt = (sb < kAecCopyRatio * sf && sb < sd) ? cnt + 1 : 0;
      if (cnt >= kAecCopyFrames) { F0 = B0; F1 = B1; cnt = 0; }
      const double c = kAecMu / (px + kAecDelta);
      const double er = c * Eb.x, ei = c * Eb.y;
      // B_p += c E conj(X_p)
      B0 = make_double2(B0.x + (er * x0.x + ei * x0.y), B0.y + (ei * x0.x - er * x0.y));
      B1 = make_double2(B1.x + (er * x1.x + ei * x1.y), B1.y + (ei * x1.x - er * x1.y));
    }
  }
  flt->b[k][lane] = B0; flt->b[k][lane + 32] = B1; flt->f[k][lane] = F0; flt->f[k][lane + 32] = F1;
  if (lane == 0) {
    flt->sb[k] = sb; flt->sf[k] = sf; flt->sd[k] = sd; flt->yh[k] = yh; flt->eh[k] = eh;
    flt->cnt[k] = cnt;
    flt->stats.sum_d[k] = sum_d; flt->stats.sum_z[k] = sum_z;
  }
}

int echo_scan(const EchoWork& w, const DenoiseState* st, int n, double2* spec, cudaStream_t stream) {
  k_aec_scan<<<(kDnBins + kAecWarps - 1) / kAecWarps, kAecWarps * 32, 0, stream>>>(w.params, w.filter, w.ring, w.far_spec, w.taps, w.delay,
                                                                                   st, n, spec);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

int echo_check(int taps, int delay_frames, double suppression_db) {
  RYK_CHECK(taps >= 1 && taps <= kAecMaxTaps, "taps must be within [1, 64]");
  RYK_CHECK(delay_frames >= 0 && delay_frames <= kAecMaxDelay, "delay_frames must be within [0, 256]");
  RYK_CHECK(isfinite(suppression_db) && suppression_db >= 0.0 && suppression_db <= 40.0, "suppression_db must be finite and within [0, 40]");
  return 0;
}

}  // namespace ryk

using namespace ryk;

extern "C" {

// The whole-signal canceller: one step over mic / far followed by kDnDelay zeros from a fresh state; its output from kDnDelay on is z.
int ryk_echo_cancel(ryk_engine* h, const float* mic, const float* far, int n, int taps, int delay_frames, double suppression_db,
                    double reduction_db, const double* phi, float* z) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(mic && far && z && n > 0, "null argument or empty signal");
  if (int rc = echo_check(taps, delay_frames, suppression_db)) return rc;
  if (int rc = denoise_check(reduction_db, phi)) return rc;
  const int len = n + kDnDelay;
  DenoiseWork w;
  EchoWork a;
  w.max_frames = denoise_max_frames(len);
  a.taps = taps; a.delay = delay_frames;
  DenoiseState *st, *st_next, *fst, *fst_next;
  float *d_mic, *d_far, *d_z;
  if (engine_scratch(e, [&](Arena& ar) {
        w.params = ar.take<DenoiseParams>(1);
        w.learn = ar.take<DenoiseLearn>(1);
        st = ar.take<DenoiseState>(1);
        st_next = ar.take<DenoiseState>(1);
        fst = ar.take<DenoiseState>(1);
        fst_next = ar.take<DenoiseState>(1);
        w.spec = ar.take<double2>((size_t)kDnBins * w.max_frames);
        a.far_spec = ar.take<double2>((size_t)kDnBins * w.max_frames);
        w.frames = ar.take<double>((size_t)kDnN * w.max_frames);
        d_mic = ar.take<float>(len);
        d_far = ar.take<float>(len);
        d_z = ar.take<float>(len);
        a.params = ar.take<EchoParams>(1);
        a.filter = ar.take<EchoFilter>(1);
        a.ring = ar.take<double2>((size_t)kDnBins * (taps + delay_frames));
        w.done = ar.take<unsigned>(1);
      })) return -1;
  // host staging: both parameter blocks, the fresh state, and mic / far followed by zeros
  DenoiseParams* h_par;
  DenoiseState* h_st;
  EchoParams* h_epar;
  float *h_mic, *h_far;
  if (engine_pinned_layout(e, [&](Arena& ar) {
        h_par = ar.take<DenoiseParams>(1);
        h_st = ar.take<DenoiseState>(1);
        h_epar = ar.take<EchoParams>(1);
        h_mic = ar.take<float>(len);
        h_far = ar.take<float>(len);
      })) return -1;
  memset(h_par, 0, sizeof(DenoiseParams));
  h_par->gain_floor = pow(10.0, -reduction_db / 20.0);
  h_par->profile_serial = 1;
  if (phi) memcpy(h_par->phi, phi, sizeof(double) * kDnBins);
  denoise_state_init(h_st);
  h_epar->gain_floor = pow(10.0, -suppression_db / 20.0);
  memcpy(h_mic, mic, sizeof(float) * n);
  memset(h_mic + n, 0, sizeof(float) * kDnDelay);
  memcpy(h_far, far, sizeof(float) * n);
  memset(h_far + n, 0, sizeof(float) * kDnDelay);
  cudaStream_t s = e->stream;
  RYK_CUDA(cudaMemcpyAsync(w.params, h_par, sizeof(DenoiseParams), cudaMemcpyHostToDevice, s));
  RYK_CUDA(cudaMemsetAsync(w.learn, 0, sizeof(DenoiseLearn), s));
  RYK_CUDA(cudaMemcpyAsync(st, h_st, sizeof(DenoiseState), cudaMemcpyHostToDevice, s));
  RYK_CUDA(cudaMemcpyAsync(fst, h_st, sizeof(DenoiseState), cudaMemcpyHostToDevice, s));
  RYK_CUDA(cudaMemcpyAsync(d_mic, h_mic, sizeof(float) * len, cudaMemcpyHostToDevice, s));
  RYK_CUDA(cudaMemcpyAsync(d_far, h_far, sizeof(float) * len, cudaMemcpyHostToDevice, s));
  RYK_CUDA(cudaMemcpyAsync(a.params, h_epar, sizeof(EchoParams), cudaMemcpyHostToDevice, s));
  RYK_CUDA(cudaMemsetAsync(a.filter, 0, sizeof(EchoFilter), s));
  RYK_CUDA(cudaMemsetAsync(a.ring, 0, sizeof(double2) * kDnBins * (taps + delay_frames), s));
  RYK_CUDA(cudaMemsetAsync(w.done, 0, sizeof(unsigned), s));
  if (denoise_forward(e, w.max_frames, st, st_next, d_mic, len, w.spec, s)) return -1;
  if (denoise_forward(e, w.max_frames, fst, fst_next, d_far, len, a.far_spec, s)) return -1;
  if (echo_scan(a, st, len, w.spec, s)) return -1;
  if (phi && denoise_scan(w, st, st_next, len, s)) return -1;
  if (denoise_inverse(e, w, st, st_next, len, d_z, s)) return -1;
  RYK_CUDA(cudaMemcpyAsync(z, d_z + kDnDelay, sizeof(float) * n, cudaMemcpyDeviceToHost, s));
  RYK_CUDA(cudaStreamSynchronize(s));
  return 0;
}

}  // extern "C"
