// limiter.cu -- the look-ahead peak limiter (DESIGN.md §4i, DECIDE L1-L4) on a streaming session's output, after the NaN scrub and the
// output resampler, and in the whole-signal ryk_limit.  In FP64 on the output stream y:
//   g0[u] = 1 if G |y[u]| <= c, else c / (G |y[u]|)            (1 for u < 0)
//   m[s]  = min of g0[u] over u in [s - R, s + L - 1]
//   g[t]  = (m[t - L + 1] + ... + m[t]) / L, summed in ascending s from 0.0
//   z[t]  = g[t] y[t]
// A step that brings n samples y[pos .. pos + n) returns z[pos - L .. pos + n - L): the L-sample look-ahead is the limiter's delay.
// Every output depends on a bounded window of y, with no recursion from sample to sample, so each kernel is parallel over samples and
// a stream cut into steps gives the bits of the whole signal.  Three kernels per step:
//   k_lim_g0     g0 over the step's window [pos - (R + 2L - 1), pos + n): the kept history, then the new samples with the step's
//                settings; the minima of its tiles of 32 and 1024 samples; the history and position for the next step; resets the meter
//   k_lim_min    m[s] for s in [pos - 2L + 1, pos + n - L) as a two-level blocked minimum: at most 31 samples at each end, then at
//                most 31 tiles of 32 at each end, then whole tiles of 1024 -- at most 148 loads for any window up to R + L = 24,480
//   k_lim_apply  g and z of the step's outputs (the box sum per output, ascending), and the meter
// The minimum is exact, so the blocked evaluation gives the bits of any other order.  Nothing offers an FMA contraction: the box sum
// only adds, and g0 and z are one product and one quotient each, so the device matches an FP64 numpy restatement bit for bit.
#include <math.h>
#include <string.h>

#include "../../include/ryk.h"
#include "engine.h"
#include "limiter.h"

namespace ryk {

constexpr int kLimTile = 1024;      // k_lim_g0: one CTA per tile of 1024 samples (the t1k tile)
constexpr int kLimThreads = 256;    // k_lim_min, k_lim_apply

__global__ void __launch_bounds__(kLimTile) k_lim_g0(const LimParams* __restrict__ par, LimHist cur, LimHist next,
                                                     const double* __restrict__ y, const int* __restrict__ n_new, int L, int R,
                                                     double* __restrict__ g0, double* __restrict__ t32, double* __restrict__ t1k,
                                                     LimMeter* __restrict__ meter) {
  const int H = R + 2 * L - 1;
  const int n = *n_new > 0 ? *n_new : 0;
  const long long pos = cur.st->pos;
  const double c = par->ceiling, G = par->gain;
  // g0 at index j of the window: u = pos - H + j
  auto g0_at = [&](int j) -> double {
    if (pos - H + j < 0) return 1.0;
    if (j < H) return cur.g0[j];
    const double a = G * fabs(y[j - H]);
    return a <= c ? 1.0 : c / a;
  };
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double v = 1.0;                   // beyond the window: neutral in the tile minima
  if (i < H + n) { v = g0_at(i); g0[i] = v; }
  if (i < H) next.g0[i] = g0_at(n + i);
  if (i < L) next.y[i] = n + i < L ? cur.y[n + i] : y[n + i - L];
  if (i == 0) {
    next.st->pos = pos + n;
    meter->min_bits = (unsigned long long)__double_as_longlong(1.0);
    meter->limited = 0;
  }
  for (int o = 16; o; o >>= 1) v = fmin(v, __shfl_xor_sync(0xffffffffu, v, o));
  __shared__ double warp_min[kLimTile / 32];
  if ((threadIdx.x & 31) == 0) { t32[i >> 5] = v; warp_min[threadIdx.x >> 5] = v; }
  __syncthreads();
  if (threadIdx.x < 32) {
    double w = warp_min[threadIdx.x];
    for (int o = 16; o; o >>= 1) w = fmin(w, __shfl_xor_sync(0xffffffffu, w, o));
    if (threadIdx.x == 0) t1k[blockIdx.x] = w;
  }
}

// min of a[lo .. hi) (hi > lo): single samples up to a 32 boundary at each end, then tiles of 32 up to a 1024 boundary, then tiles of 1024
__device__ inline double lim_range_min(const double* __restrict__ a, const double* __restrict__ t32, const double* __restrict__ t1k,
                                       int lo, int hi) {
  double v = 1.0;                   // every g0 is at most 1
  while (lo < hi && (lo & 31)) v = fmin(v, a[lo++]);
  while (lo < hi && (hi & 31)) v = fmin(v, a[--hi]);
  lo >>= 5; hi >>= 5;
  while (lo < hi && (lo & 31)) v = fmin(v, t32[lo++]);
  while (lo < hi && (hi & 31)) v = fmin(v, t32[--hi]);
  for (lo >>= 5, hi >>= 5; lo < hi; ++lo) v = fmin(v, t1k[lo]);
  return v;
}

// m at index q of the step (s = pos - 2L + 1 + q) covers window indices [q, q + R + L)
__global__ void __launch_bounds__(kLimThreads) k_lim_min(const int* __restrict__ n_new, int L, int R, const double* __restrict__ g0,
                                                         const double* __restrict__ t32, const double* __restrict__ t1k, double* __restrict__ m) {
  const int n = *n_new > 0 ? *n_new : 0;
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (n == 0 || q >= n + L - 1) return;
  m[q] = lim_range_min(g0, t32, t1k, q, q + R + L);
}

// output j of the step is z[t], t = pos + j - L; its box sum reads m at indices j .. j + L - 1
__global__ void __launch_bounds__(kLimThreads) k_lim_apply(LimHist cur, const double* __restrict__ y, const int* __restrict__ n_new, int L,
                                                           const double* __restrict__ m, double* __restrict__ z, LimMeter* __restrict__ meter) {
  const int n = *n_new > 0 ? *n_new : 0;
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  double g = 1.0;
  if (j < n) {
    if (cur.st->pos + j - L < 0) {
      z[j] = 0.0;                   // the leading zeros of the delay
    } else {
      double acc = 0.0;
      for (int q = j; q < j + L; ++q) acc += m[q];
      g = acc / (double)L;
      z[j] = g * (j < L ? cur.y[j] : y[j - L]);
    }
  }
  unsigned limited = g < 1.0;
  for (int o = 16; o; o >>= 1) {
    g = fmin(g, __shfl_xor_sync(0xffffffffu, g, o));
    limited += __shfl_xor_sync(0xffffffffu, limited, o);
  }
  if ((threadIdx.x & 31) == 0 && limited) {
    atomicMin(&meter->min_bits, (unsigned long long)__double_as_longlong(g));
    atomicAdd(&meter->limited, (unsigned long long)limited);
  }
}

int limiter_check_shape(double lookahead_ms, double hold_ms) {
  RYK_CHECK(isfinite(lookahead_ms) && lookahead_ms >= 0.5 && lookahead_ms <= 10.0, "lookahead_ms must be finite and within [0.5, 10]");
  RYK_CHECK(isfinite(hold_ms) && hold_ms >= 0.0 && hold_ms <= 500.0, "hold_ms must be finite and within [0, 500]");
  return 0;
}

int limiter_check_settings(double ceiling_db, double gain) {
  RYK_CHECK(isfinite(ceiling_db) && ceiling_db >= -24.0 && ceiling_db <= 0.0, "ceiling_db must be finite and within [-24, 0]");
  RYK_CHECK(isfinite(gain) && gain > 0.0, "gain must be finite and positive");
  return 0;
}

void limiter_shape(int rate, double lookahead_ms, double hold_ms, int* L, int* R) {
  const long l = lrint(lookahead_ms * rate / 1000.0);
  *L = l < 1 ? 1 : (int)l;
  *R = (int)lrint(hold_ms * rate / 1000.0);
}

LimParams limiter_params(double ceiling_db, double gain) { return LimParams{pow(10.0, ceiling_db / 20.0), gain}; }

void limiter_scratch_sizes(const LimWork& w, size_t* n_g0, size_t* n_t32, size_t* n_t1k, size_t* n_m) {
  const size_t window = (size_t)w.R + 2 * w.L - 1 + w.max_n;
  const size_t tiles = (window + kLimTile - 1) / kLimTile;
  *n_g0 = window;
  *n_t32 = tiles * (kLimTile / 32);
  *n_t1k = tiles;
  *n_m = (size_t)w.max_n + w.L - 1;
}

int limiter_run(const LimWork& w, const LimHist& cur, const LimHist& next, const double* d_y, const int* d_n, double* d_z,
                cudaStream_t stream) {
  size_t n_g0, n_t32, n_t1k, n_m;
  limiter_scratch_sizes(w, &n_g0, &n_t32, &n_t1k, &n_m);
  k_lim_g0<<<(int)n_t1k, kLimTile, 0, stream>>>(w.params, cur, next, d_y, d_n, w.L, w.R, w.g0, w.t32, w.t1k, w.meter);
  k_lim_min<<<(int)((n_m + kLimThreads - 1) / kLimThreads), kLimThreads, 0, stream>>>(d_n, w.L, w.R, w.g0, w.t32, w.t1k, w.m);
  k_lim_apply<<<(w.max_n + kLimThreads - 1) / kLimThreads, kLimThreads, 0, stream>>>(cur, d_y, d_n, w.L, w.m, d_z, w.meter);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace ryk

using namespace ryk;

extern "C" {

// The whole-signal limiter: one step over y followed by L zeros from a fresh state; its output from L on is z.
int ryk_limit(ryk_engine* h, const double* y, int n, int rate, double lookahead_ms, double hold_ms, double ceiling_db, double gain,
              double* z) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(y && z && n > 0, "null argument or empty signal");
  RYK_CHECK(rate > 0, "rate must be positive");
  if (int rc = limiter_check_shape(lookahead_ms, hold_ms)) return rc;
  if (int rc = limiter_check_settings(ceiling_db, gain)) return rc;
  LimWork w;
  limiter_shape(rate, lookahead_ms, hold_ms, &w.L, &w.R);
  const int len = n + w.L, H = w.R + 2 * w.L - 1;
  w.max_n = len;
  size_t n_g0, n_t32, n_t1k, n_m;
  limiter_scratch_sizes(w, &n_g0, &n_t32, &n_t1k, &n_m);
  LimHist cur, next;
  double *d_y, *d_z;
  int* d_n;
  if (engine_scratch(e, [&](Arena& a) {
        w.params = a.take<LimParams>(1);
        w.meter = a.take<LimMeter>(1);
        for (LimHist* hist : {&cur, &next}) {
          hist->st = a.take<LimState>(1);
          hist->g0 = a.take<double>(H);
          hist->y = a.take<double>(w.L);
        }
        d_y = a.take<double>(len);
        d_z = a.take<double>(len);
        w.g0 = a.take<double>(n_g0);
        w.t32 = a.take<double>(n_t32);
        w.t1k = a.take<double>(n_t1k);
        w.m = a.take<double>(n_m);
        d_n = a.take<int>(1);
      })) return -1;
  // host staging: the settings, the sample count, and y followed by L zeros
  LimParams* h_par;
  double* h_y;
  int* h_n;
  if (engine_pinned_layout(e, [&](Arena& a) { h_par = a.take<LimParams>(1); h_y = a.take<double>(len); h_n = a.take<int>(1); })) return -1;
  *h_par = limiter_params(ceiling_db, gain);
  memcpy(h_y, y, sizeof(double) * n);
  memset(h_y + n, 0, sizeof(double) * w.L);
  *h_n = len;
  cudaStream_t s = e->stream;
  RYK_CUDA(cudaMemcpyAsync(w.params, h_par, sizeof(LimParams), cudaMemcpyHostToDevice, s));
  RYK_CUDA(cudaMemcpyAsync(d_y, h_y, sizeof(double) * len, cudaMemcpyHostToDevice, s));
  RYK_CUDA(cudaMemcpyAsync(d_n, h_n, sizeof(int), cudaMemcpyHostToDevice, s));
  // a fresh state: position 0 (the history is never read before 0)
  RYK_CUDA(cudaMemsetAsync(cur.st, 0, sizeof(LimState), s));
  RYK_CUDA(cudaMemsetAsync(cur.g0, 0, sizeof(double) * H, s));
  RYK_CUDA(cudaMemsetAsync(cur.y, 0, sizeof(double) * w.L, s));
  if (limiter_run(w, cur, next, d_y, d_n, d_z, s)) return -1;
  RYK_CUDA(cudaMemcpyAsync(z, d_z + w.L, sizeof(double) * n, cudaMemcpyDeviceToHost, s));
  RYK_CUDA(cudaStreamSynchronize(s));
  return 0;
}

}  // extern "C"
