// denoise.cu -- input noise suppression (DESIGN.md §4f, DECIDE N1-N3): a decision-directed Wiener filter on 512-sample sqrt-Hann
// frames at a 128-sample hop, in FP64, ahead of the WORLD analysis of a streaming session and in the whole-signal ryk_denoise.
//
// A step hands in n new model-rate samples x[in_end, in_end + n) and takes out n filtered samples delayed by kDnDelay:
//   k_dn_forward   one CTA per frame m in [floor(in_end / H), floor((in_end + n) / H)), the frames whose last sample arrives in the
//                  step: X_m = rfft(w * x[mH - (N - H), mH + H)) from the kept history and the new samples
//   k_dn_scan      one thread per bin: the gain recursion (N2) over the step's frames in ascending order, with the profile learning
//                  folded into the same loop; X_m <- G_m X_m
//   k_dn_inverse   one CTA per frame: w * irfft(G_m X_m); the last CTA to finish overlap-adds the step's frames into the samples
//                  [in_end - kDnDelay, floor((in_end + n) / H) H) in ascending frame order, continuing the FP64 sums carried from the
//                  previous step, and emits the first n of them
// Every sample's sum runs over the same frames in the same order whatever the step boundaries, and every frame's arithmetic depends on
// the frame alone, so a stream of steps is bitwise the whole-signal call (one step over x followed by kDnDelay zeros).
#include <math.h>
#include <string.h>

#include <vector>

#include "../../include/ryk.h"
#include "denoise.h"
#include "engine.h"
#include "fft.cuh"

namespace ryk {

constexpr int kDnLog2N = 9;
constexpr int kDnThreads = 256;

// periodic sqrt-Hann: sqrt(0.5 - 0.5 cos(2 pi j / N))
__device__ inline double dn_window(int j) { return sqrt(0.5 - 0.5 * cospi((double)j / (kDnN / 2))); }

__device__ inline long long dn_floordiv(long long a, long long b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }

// sample t of the stream for a step that starts at in_end: zero before 0, from the kept history before in_end, else the step's input
__device__ inline float dn_sample(const DenoiseState* __restrict__ st, long long in_end, const float* __restrict__ x, long long t) {
  if (t < 0) return 0.f;
  return t < in_end ? st->hist[t - (in_end - kDnDelay)] : x[t - in_end];
}

__global__ void __launch_bounds__(kDnThreads) k_dn_forward(const DenoiseState* __restrict__ st, DenoiseState* __restrict__ st_next,
                                                          const float* __restrict__ x, int n, double2* __restrict__ spec,
                                                          const double2* __restrict__ tw) {
  __shared__ double2 a[kDnN];
  const long long in_end = st->in_end;
  if (blockIdx.x == 0) {
    for (int i = threadIdx.x; i < kDnDelay; i += blockDim.x) st_next->hist[i] = dn_sample(st, in_end, x, in_end + n - kDnDelay + i);
    if (threadIdx.x == 0) st_next->in_end = in_end + n;
  }
  const long long m = in_end / kDnHop + blockIdx.x;
  if (m >= (in_end + n) / kDnHop) return;
  const long long s = m * kDnHop - (kDnN - kDnHop);
  for (int i = threadIdx.x; i < kDnN; i += blockDim.x) a[i] = make_double2(dn_window(i) * (double)dn_sample(st, in_end, x, s + i), 0.0);
  fft_smem(a, kDnN, kDnLog2N, -1, tw);
  for (int k = threadIdx.x; k < kDnBins; k += blockDim.x) spec[(size_t)blockIdx.x * kDnBins + k] = a[k];
}

// N2 per bin k: xi_m = alpha G_{m-1}^2 P_{m-1} / Phi + (1 - alpha) max(P_m / Phi - 1, 0), G_m = max(xi_m / (1 + xi_m), g); G = 1 where
// Phi == 0.  A new host profile applies to the whole step; a learning adds P_m of its first `total` frames to the sums, and the
// profile they give applies from the next step.  Thread 0 writes the shared scalars after every thread has read them.
__global__ void __launch_bounds__(288) k_dn_scan(const DenoiseParams* __restrict__ par, DenoiseLearn* __restrict__ learn,
                                                 const DenoiseState* __restrict__ st, DenoiseState* __restrict__ st_next, int n,
                                                 double2* __restrict__ spec) {
  const int k = threadIdx.x;
  const long long in_end = st->in_end;
  const long long f0 = in_end / kDnHop, f1 = (in_end + n) / kDnHop;
  const bool new_profile = par->profile_serial != learn->profile_serial;
  const bool new_learn = par->learn_serial != learn->learn_serial;
  long long rem = new_learn ? par->learn_frames : learn->remaining;
  const long long total = new_learn ? par->learn_frames : learn->total;
  const double g = par->gain_floor;
  if (k < kDnBins) {
    const double phi = new_profile ? par->phi[k] : learn->phi[k];
    double sum = new_learn ? 0.0 : learn->sum[k];
    double G = st->gain[k], Pp = st->power[k];
    bool learned = false;
    for (long long m = f0; m < f1; ++m) {
      double2* X = &spec[(size_t)(m - f0) * kDnBins + k];
      const double2 v = *X;
      const double P = v.x * v.x + v.y * v.y;
      if (phi > 0.0) {
        const double xi = kDnAlpha * (G * G) * Pp / phi + (1.0 - kDnAlpha) * fmax(P / phi - 1.0, 0.0);
        G = fmax(xi / (1.0 + xi), g);
      } else {
        G = 1.0;
      }
      *X = make_double2(G * v.x, G * v.y);
      Pp = P;
      if (rem > 0) {
        sum += P;
        learned = --rem == 0;
      }
    }
    st_next->gain[k] = G; st_next->power[k] = Pp;
    learn->sum[k] = sum;
    learn->phi[k] = learned ? sum / (double)total : phi;
  }
  __syncthreads();
  if (k == 0) {
    learn->profile_serial = par->profile_serial; learn->learn_serial = par->learn_serial;
    learn->remaining = rem; learn->total = total;
  }
}

__global__ void __launch_bounds__(kDnThreads) k_dn_inverse(const DenoiseState* __restrict__ st, DenoiseState* __restrict__ st_next, int n,
                                                          const double2* __restrict__ spec, double* frames, unsigned* done,
                                                          float* __restrict__ z, const double2* __restrict__ tw) {
  __shared__ double2 a[kDnN];
  __shared__ bool last;
  const long long in_end = st->in_end;
  const long long f0 = in_end / kDnHop, f1 = (in_end + n) / kDnHop;
  if (f0 + blockIdx.x < f1) {
    for (int k = threadIdx.x; k < kDnBins; k += blockDim.x) a[k] = spec[(size_t)blockIdx.x * kDnBins + k];
    irfft_smem(a, kDnN, kDnLog2N, tw);
    for (int i = threadIdx.x; i < kDnN; i += blockDim.x) frames[(size_t)blockIdx.x * kDnN + i] = dn_window(i) * (a[i].x * (1.0 / kDnN));
  }
  // the last CTA to finish sees every frame (the threadFenceReduction pattern)
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) last = atomicAdd(done, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!last) return;
  const long long t0 = in_end - kDnDelay, t_emit = in_end + n - kDnDelay, t1 = f1 * kDnHop;
  for (long long t = t0 + threadIdx.x; t < t1; t += blockDim.x) {
    double acc = t < f0 * kDnHop ? st->carry[t - t0] : 0.0;
    // the frames m covering t: m H - (N - H) <= t < m H + H
    long long lo = dn_floordiv(t - kDnHop, kDnHop) + 1, hi = dn_floordiv(t + (kDnN - kDnHop), kDnHop);
    if (lo < f0) lo = f0;
    if (hi > f1 - 1) hi = f1 - 1;
    for (long long m = lo; m <= hi; ++m) acc += __ldcg(&frames[(size_t)(m - f0) * kDnN + (size_t)(t - (m * kDnHop - (kDnN - kDnHop)))]);
    if (t < t_emit) z[t - t0] = t < 0 ? 0.f : (float)(0.5 * acc);
    else st_next->carry[t - t_emit] = acc;
  }
  if (threadIdx.x == 0) *done = 0;
}

void denoise_state_init(DenoiseState* host) {
  memset(host, 0, sizeof(DenoiseState));
  for (double& g : host->gain) g = 1.0;
}

int denoise_forward(Engine* e, int max_frames, const DenoiseState* st, DenoiseState* st_next, const float* d_x, int n, double2* spec,
                    cudaStream_t stream) {
  k_dn_forward<<<max_frames, kDnThreads, 0, stream>>>(st, st_next, d_x, n, spec, e->d_twiddle);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

int denoise_scan(const DenoiseWork& w, const DenoiseState* st, DenoiseState* st_next, int n, cudaStream_t stream) {
  k_dn_scan<<<1, 288, 0, stream>>>(w.params, w.learn, st, st_next, n, w.spec);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

int denoise_inverse(Engine* e, const DenoiseWork& w, const DenoiseState* st, DenoiseState* st_next, int n, float* d_z, cudaStream_t stream) {
  k_dn_inverse<<<w.max_frames, kDnThreads, 0, stream>>>(st, st_next, n, w.spec, w.frames, w.done, d_z, e->d_twiddle);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

int denoise_run(Engine* e, const DenoiseWork& w, const DenoiseState* st, DenoiseState* st_next, const float* d_x, int n, float* d_z,
                cudaStream_t stream) {
  if (denoise_forward(e, w.max_frames, st, st_next, d_x, n, w.spec, stream)) return -1;
  if (denoise_scan(w, st, st_next, n, stream)) return -1;
  return denoise_inverse(e, w, st, st_next, n, d_z, stream);
}

// the refusals every entry point that takes a reduction or a profile shares
int denoise_check(double reduction_db, const double* phi) {
  RYK_CHECK(isfinite(reduction_db) && reduction_db >= 0.0 && reduction_db <= 40.0, "reduction_db must be finite and within [0, 40]");
  if (phi)
    for (int k = 0; k < kDnBins; ++k) RYK_CHECK(isfinite(phi[k]) && phi[k] >= 0.0, "noise profile entries must be finite and >= 0");
  return 0;
}

}  // namespace ryk

using namespace ryk;

extern "C" {

// The whole-signal filter: one step over x followed by kDnDelay zeros from a fresh state; its output from kDnDelay on is z.
int ryk_denoise(ryk_engine* h, const float* x, int n, double reduction_db, const double* phi, float* z) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(x && z && n > 0, "null argument or empty signal");
  if (int rc = denoise_check(reduction_db, phi)) return rc;
  const int len = n + kDnDelay;
  DenoiseWork w;
  w.max_frames = denoise_max_frames(len);
  DenoiseState *st, *st_next;
  float *d_x, *d_z;
  if (engine_scratch(e, [&](Arena& a) {
        w.params = a.take<DenoiseParams>(1);
        w.learn = a.take<DenoiseLearn>(1);
        st = a.take<DenoiseState>(1);
        st_next = a.take<DenoiseState>(1);
        w.spec = a.take<double2>((size_t)kDnBins * w.max_frames);
        w.frames = a.take<double>((size_t)kDnN * w.max_frames);
        d_x = a.take<float>(len);
        d_z = a.take<float>(len);
        w.done = a.take<unsigned>(1);
      })) return -1;
  // host staging: the parameter block (a profile set, no learning), the fresh state and x followed by zeros
  DenoiseParams* h_par;
  DenoiseState* h_st;
  float* h_x;
  if (engine_pinned_layout(e, [&](Arena& a) { h_par = a.take<DenoiseParams>(1); h_st = a.take<DenoiseState>(1); h_x = a.take<float>(len); }))
    return -1;
  memset(h_par, 0, sizeof(DenoiseParams));
  h_par->gain_floor = pow(10.0, -reduction_db / 20.0);
  h_par->profile_serial = 1;
  if (phi) memcpy(h_par->phi, phi, sizeof(double) * kDnBins);
  denoise_state_init(h_st);
  memcpy(h_x, x, sizeof(float) * n);
  memset(h_x + n, 0, sizeof(float) * kDnDelay);
  cudaStream_t s = e->stream;
  RYK_CUDA(cudaMemcpyAsync(w.params, h_par, sizeof(DenoiseParams), cudaMemcpyHostToDevice, s));
  RYK_CUDA(cudaMemsetAsync(w.learn, 0, sizeof(DenoiseLearn), s));
  RYK_CUDA(cudaMemcpyAsync(st, h_st, sizeof(DenoiseState), cudaMemcpyHostToDevice, s));
  RYK_CUDA(cudaMemcpyAsync(d_x, h_x, sizeof(float) * len, cudaMemcpyHostToDevice, s));
  RYK_CUDA(cudaMemsetAsync(w.done, 0, sizeof(unsigned), s));
  if (denoise_run(e, w, st, st_next, d_x, len, d_z, s)) return -1;
  RYK_CUDA(cudaMemcpyAsync(z, d_z + kDnDelay, sizeof(float) * n, cudaMemcpyDeviceToHost, s));
  RYK_CUDA(cudaStreamSynchronize(s));
  return 0;
}

}  // extern "C"
