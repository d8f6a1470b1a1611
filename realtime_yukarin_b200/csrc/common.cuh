// common.cuh -- shared declarations for libryk (H100 / sm_90a hot path of realtime-yukarin).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>

namespace ryk {

constexpr double kPi = 3.1415926535897932384;
constexpr double kLog2 = 0.69314718055994529;
constexpr double kSafeMin = 0.000000000001;
constexpr double kEps = 0.00000000000000022204460492503131;
constexpr double kDefaultF0 = 500.0;
constexpr double kMaxValue = 100000.0;

void set_error(const std::string& msg);

#define RYK_CUDA(call)                                                                       \
  do {                                                                                       \
    cudaError_t _e = (call);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      ryk::set_error(std::string(#call) + " failed: " + cudaGetErrorString(_e) + " at " +    \
                     __FILE__ + ":" + std::to_string(__LINE__));                             \
      return -1;                                                                             \
    }                                                                                        \
  } while (0)

#define RYK_CHECK(cond, msg)                                                                 \
  do {                                                                                       \
    if (!(cond)) {                                                                           \
      ryk::set_error(std::string(msg) + " (" #cond ") at " + __FILE__ + ":" +                \
                     std::to_string(__LINE__));                                              \
      return -2;                                                                             \
    }                                                                                        \
  } while (0)

__host__ __device__ inline int matlab_round(double x) { return x > 0 ? (int)(x + 0.5) : (int)(x - 0.5); }
__host__ __device__ inline int imin(int a, int b) { return a < b ? a : b; }
__host__ __device__ inline int imax(int a, int b) { return a > b ? a : b; }

inline int suitable_fft_size(int sample) {
  return (int)pow(2.0, (int)(log((double)sample) / kLog2) + 1.0);
}
inline int cheaptrick_fft_size(int fs, double f0_floor) {
  return (int)pow(2.0, 1.0 + (int)(log(3.0 * fs / f0_floor + 1) / kLog2));
}

// ---- block-wide helpers (all threads of the CTA must call) ------------------------------------
__device__ inline double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// scratch: >= 32 doubles of shared memory. Result broadcast to every thread.
__device__ inline double block_sum(double v, double* scratch) {
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) scratch[w] = v;
  __syncthreads();
  double r = 0.0;
  if (w == 0) {
    r = lane < nw ? scratch[lane] : 0.0;
    r = warp_sum(r);
    if (lane == 0) scratch[0] = r;
  }
  __syncthreads();
  r = scratch[0];
  __syncthreads();
  return r;
}

// In-place inclusive prefix sum over smem array a[0..n) (doubles). scratch >= blockDim.x doubles.
__device__ inline void block_inclusive_scan(double* a, int n, double* scratch) {
  const int T = blockDim.x, lane = threadIdx.x & 31, nw = (T + 31) >> 5;
  // nvcc 12.9 miscompiles &scratch[threadIdx.x >> 5] here when block_sum() was inlined earlier in the same kernel: it re-uses block_sum's
  // address register, strength-reduced to base + (tid >> 2) under block_sum's `lane == 0` predicate, for accesses made by ALL lanes
  // (compute-sanitizer: misaligned shared accesses at base + 8 w + (lane >> 2)).  The empty asm makes the warp index opaque to that CSE.
  int w = threadIdx.x >> 5;
  asm volatile("" : "+r"(w));
  int per = (n + T - 1) / T;
  int lo = threadIdx.x * per, hi = min(lo + per, n);
  double s = 0.0;
  for (int i = lo; i < hi; ++i) { s += a[i]; a[i] = s; }
  // scan of the per-thread sums: shuffles inside a warp, one pass over the <= 32 warp totals (3 block barriers; the Hillis-Steele
  // form over all threads took 2 log2(T) + 2 of them, and these per-frame kernels are chains of barriers)
  double incl = s;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const double t = __shfl_up_sync(0xffffffffu, incl, off);
    if (lane >= off) incl += t;
  }
  double excl = __shfl_up_sync(0xffffffffu, incl, 1);      // exclusive prefix inside the warp (exact: no incl - s cancellation)
  if (lane == 0) excl = 0.0;
  const double wtot = __shfl_sync(0xffffffffu, incl, 31);
  if (lane == 0) scratch[w] = wtot;
  __syncthreads();
  if (w == 0) {
    double t = lane < nw ? scratch[lane] : 0.0;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const double u = __shfl_up_sync(0xffffffffu, t, off);
      if (lane >= off) t += u;
    }
    if (lane < nw) scratch[lane] = t;
  }
  __syncthreads();
  const double base = excl + (w > 0 ? scratch[w - 1] : 0.0);
  for (int i = lo; i < hi; ++i) a[i] += base;
  __syncthreads();
}

// interp1Q on an equally spaced grid (origin x0, spacing dx), y has n points (delta_y[n-1] = 0).
__device__ inline double interp1q(double x0, double dx, const double* y, int n, double xi) {
  double pos = (xi - x0) / dx;
  int base = (int)pos;
  double frac = pos - base;
  double dy = base + 1 < n ? y[base + 1] - y[base] : 0.0;
  return y[base] + dy * frac;
}

// matlab interp1 (histc + linear, extrapolating): k = clamp(#{x[j] <= xi}, 1, n-1)
__device__ inline double interp1_at(const double* x, const double* y, int n, double xi) {
  int lo = 0, hi = n;
  while (lo < hi) {
    int mid = (lo + hi) >> 1;
    if (x[mid] <= xi) lo = mid + 1; else hi = mid;
  }
  int k = lo < 1 ? 1 : (lo > n - 1 ? n - 1 : lo);
  double s = (xi - x[k - 1]) / (x[k] - x[k - 1]);
  return y[k - 1] + s * (y[k] - y[k - 1]);
}

}  // namespace ryk
