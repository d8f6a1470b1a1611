// world_analysis.cu -- WORLD analysis on the H100: DIO + StoneMask (f0), CheapTrick (spectral
// envelope, fused with SPTK sp2mc), D4C (aperiodicity).  Replaces the CPU pyworld/pysptk calls
// reached from realtime_voice_conversion/yukarin_wrapper/vocoder.py:26-48 ->
// acoustic_feature_wrapper.py:28-33 -> yukarin.AcousticFeature.extract (SURVEY rows a6, A-E).
//
// Mapping to the hardware (all FP64, no tensor cores: this is FFT / scan / sort work):
//   * DIO's whole-chunk FFTs (16k-64k points) go through cuFFT (D2Z once, batched Z2D for the bands);
//   * everything per-frame is ONE CTA per frame with the frame resident in shared memory:
//     window -> FFT -> smoothing (block scan) -> cepstral lifter -> FFT -> exp, so a frame's
//     intermediate spectra never reach HBM;
//   * zero-crossing extraction is an ordered block compaction (warp-shuffle scans);
//   * the sequential f0-contour repair (<= a few hundred frames) runs on a single thread.
#include <cufft.h>
#include <math.h>
#include <vector>

#include "analysis_shared.cuh"
#include "engine.h"
#include "fft.cuh"

namespace ryk {

// ------------------------------------------------------------------------------------ DIO
__global__ void k_dio_prepare(const float* __restrict__ x, int n, int y_length, int fft_size, double* __restrict__ y) {
  __shared__ double scratch[32];
  double s = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) s += (double)x[i];
  double mean = block_sum(s, scratch) / y_length;
  for (int i = threadIdx.x; i < fft_size; i += blockDim.x) {
    double v = 0.0;
    if (i < n) v = (double)x[i] - mean;
    else if (i < y_length) v = -mean;
    y[i] = v;
  }
}

// time-domain filters whose spectra are cached per plan: index 0 = low-cut, 1+b = band b Nuttall LPF
__global__ void k_dio_design_filters(double* __restrict__ filt, int fft_size, int cutoff_N, const int* __restrict__ half_avg) {
  int which = blockIdx.x;
  double* f = filt + (size_t)which * fft_size;
  if (which == 0) {
    __shared__ double scratch[32];
    int N = cutoff_N;
    double s = 0.0;
    for (int i = threadIdx.x; i < N; i += blockDim.x) s += 0.5 - 0.5 * cos((i + 1) * 2.0 * kPi / (N + 1));
    double sum = block_sum(s, scratch);
    int sh = (N - 1) / 2;
    // circularly centred: tap j of the normalised negated Hanning lands at (j - sh) mod fft_size
    for (int i = threadIdx.x; i < fft_size; i += blockDim.x) {
      int j;   // source tap
      if (i <= N - 1 - sh) j = i + sh; else if (i >= fft_size - sh) j = i - (fft_size - sh); else j = -1;
      double v = 0.0;
      if (j >= 0 && j < N) v = -(0.5 - 0.5 * cos((j + 1) * 2.0 * kPi / (N + 1))) / sum;
      if (i == 0) v += 1.0;
      f[i] = v;
    }
  } else {
    int len = half_avg[which - 1] * 4;
    for (int i = threadIdx.x; i < fft_size; i += blockDim.x) {
      double v = 0.0;
      if (i < len) {
        double tmp = i / (len - 1.0);
        v = 0.355768 - 0.487396 * cos(2.0 * kPi * tmp) + 0.144232 * cos(4.0 * kPi * tmp) - 0.012604 * cos(6.0 * kPi * tmp);
      }
      f[i] = v;
    }
  }
}

// Y *= F (low-cut), in place
__global__ void k_cmul_inplace(cufftDoubleComplex* __restrict__ y, const cufftDoubleComplex* __restrict__ f, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    cufftDoubleComplex a = y[i], b = f[i];
    y[i] = make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
  }
}

__global__ void k_dio_candidates(const double* __restrict__ loc, const double* __restrict__ itv, const int* __restrict__ counts,
                                 int y_length, int f0_length, int nbands, double frame_period, double f0_floor, double f0_ceil,
                                 const double* __restrict__ boundary, double* __restrict__ cand, double* __restrict__ score) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int b = blockIdx.y;
  if (i >= f0_length) return;
  const int* c = counts + b * 4;
  double cv = 0.0, sv = kMaxValue;
  if (c[0] > 2 && c[1] > 2 && c[2] > 2 && c[3] > 2) {
    double t = i * frame_period / 1000.0;
    double v[4];
    for (int e = 0; e < 4; ++e) {
      size_t slot = ((size_t)b * 4 + e) * y_length;
      v[e] = interp1_at(loc + slot, itv + slot, c[e], t);
    }
    cv = (v[0] + v[1] + v[2] + v[3]) / 4.0;
    sv = sqrt(((v[0] - cv) * (v[0] - cv) + (v[1] - cv) * (v[1] - cv) + (v[2] - cv) * (v[2] - cv) + (v[3] - cv) * (v[3] - cv)) / 3.0);
    double bf = boundary[b];
    if (cv > bf || cv < bf / 2.0 || cv > f0_ceil || cv < f0_floor) { cv = 0.0; sv = kMaxValue; }
  }
  cand[(size_t)b * f0_length + i] = cv;
  score[(size_t)b * f0_length + i] = sv / (cv + kSafeMin);
}

__device__ inline double dio_select_best(double cur, double past, const double* cand, int nbands, int f0_length, int target, double allowed) {
  double ref = (cur * 3.0 - past) / 2.0;
  double minerr = fabs(ref - cand[target]), best = cand[target];
  for (int b = 1; b < nbands; ++b) {
    double err = fabs(ref - cand[(size_t)b * f0_length + target]);
    if (err < minerr) { minerr = err; best = cand[(size_t)b * f0_length + target]; }
  }
  if (fabs(1.0 - best / ref) > allowed) return 0.0;
  return best;
}

// best-band selection (parallel) + FixF0Contour steps 1-4 (sequential, thread 0). scratch: 3*f0_length doubles + 2*f0_length ints
__global__ void k_dio_fix(const double* __restrict__ cand, const double* __restrict__ score, int nbands, int f0_length,
                          double frame_period, double f0_floor, double* __restrict__ scratch, int* __restrict__ iscratch,
                          double* __restrict__ f0) {
  const double allowed = 0.1;
  double* best = scratch;
  double* t1 = scratch + f0_length;
  double* t2 = scratch + 2 * (size_t)f0_length;
  for (int i = threadIdx.x; i < f0_length; i += blockDim.x) {
    double tmp = score[i], bv = cand[i];
    for (int b = 1; b < nbands; ++b) {
      double s = score[(size_t)b * f0_length + i];
      if (tmp > s) { tmp = s; bv = cand[(size_t)b * f0_length + i]; }
    }
    best[i] = bv;
    f0[i] = 0.0;
  }
  __syncthreads();
  int vrm = (int)(0.5 + 1000.0 / frame_period / f0_floor) * 2 + 1;
  if (f0_length <= vrm) return;
  // step 1 (parallel)
  for (int i = threadIdx.x; i < f0_length; i += blockDim.x) {
    double v = 0.0;
    if (i >= vrm) {
      double bi = (i < vrm || i >= f0_length - vrm) ? 0.0 : best[i];
      double bp = (i - 1 < vrm || i - 1 >= f0_length - vrm) ? 0.0 : best[i - 1];
      v = fabs((bi - bp) / (kSafeMin + bi)) < allowed ? bi : 0.0;
    }
    t1[i] = v;
  }
  __syncthreads();
  // step 2 (parallel)
  int center = (vrm - 1) / 2;
  for (int i = threadIdx.x; i < f0_length; i += blockDim.x) {
    double v = t1[i];
    if (i >= center && i < f0_length - center) {
      for (int j = -center; j <= center; ++j) if (t1[i + j] == 0) { v = 0.0; break; }
    }
    t2[i] = v;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  int* pos = iscratch; int* neg = iscratch + f0_length;
  int pc = 0, nc = 0;
  for (int i = 1; i < f0_length; ++i) {
    if (t2[i] == 0 && t2[i - 1] != 0) neg[nc++] = i - 1;
    else if (t2[i - 1] == 0 && t2[i] != 0) pos[pc++] = i;
  }
  // step 3: forward extension (t1 <- t2)
  for (int i = 0; i < f0_length; ++i) t1[i] = t2[i];
  for (int i = 0; i < nc; ++i) {
    int limit = i == nc - 1 ? f0_length - 1 : neg[i + 1];
    for (int j = neg[i]; j < limit; ++j) {
      double v = dio_select_best(t1[j], t1[j - 1], cand, nbands, f0_length, j + 1, allowed);
      t1[j + 1] = v;
      if (v == 0) break;
    }
  }
  // step 4: backward extension
  for (int i = 0; i < f0_length; ++i) f0[i] = t1[i];
  for (int i = pc - 1; i >= 0; --i) {
    int limit = i == 0 ? 1 : pos[i - 1];
    for (int j = pos[i]; j > limit; --j) {
      double v = dio_select_best(f0[j], f0[j + 1], cand, nbands, f0_length, j - 1, allowed);
      f0[j - 1] = v;
      if (v == 0) break;
    }
  }
}

// ------------------------------------------------------------------------------------ StoneMask
__device__ inline double stonemask_fix(const double* power, const double* numer, int fft_size, int fs, double f0i, int nh) {
  double num = 0.0, den = 0.0;
  for (int i = 0; i < nh; ++i) {
    int index = matlab_round(f0i * fft_size / fs * (i + 1));
    double p = power[index];
    double inst = p == 0.0 ? 0.0 : (double)index * fs / fft_size + numer[index] / p * fs / 2.0 / kPi;
    double amp = sqrt(p);
    num += amp * inst;
    den += amp * (i + 1);
  }
  return num / (den + kSafeMin);
}

// StoneMask's window half length and FFT size for an f0 estimate f0i (40 < f0i <= fs / 12).  WORLD's size is
// 2^(2 + floor(log2(2 half + 1))); 2 half + 1 is odd, never a power of two, so the integer bit length gives the same floor as
// log() / log(2) in any rounding, on the host and on the device alike.
__host__ __device__ inline int stonemask_half(int fs, double f0i) { return (int)(1.5 * fs / f0i + 1.0); }
__host__ __device__ inline int stonemask_fft_size(int half) {
  const unsigned m = 2u * (unsigned)half + 1u;
  int lg = 0;
  while (m >> (lg + 1)) ++lg;
  return 1 << (2 + lg);
}
// The largest FFT k_stonemask can form on a plan whose f0 contour is 0 or >= f0_min: the half length falls as f0i grows (correctly
// rounded division and the truncation are monotonic), and the kernel skips f0i <= 40, so f0_min below 40 bounds nothing.  The shared-
// memory FFT stops at kTwiddleN points; a frame that would need more (only from 27.3 kHz up, with f0 near 40 Hz) keeps its estimate.
static int stonemask_max_fft(int fs, double f0_min) {
  const int n = stonemask_fft_size(stonemask_half(fs, f0_min > 40.0 ? f0_min : 40.0));
  return n < kTwiddleN ? n : kTwiddleN;
}
static size_t stonemask_smem_bytes(int max_fft) { return sizeof(double2) * 2 * max_fft + sizeof(double) * 2 * (max_fft / 2 + 1) + 64; }

// one CTA per frame; smem: 2 * max_fft double2 (main / diff spectra) + 2 * (max_fft / 2 + 1) doubles, max_fft from stonemask_max_fft
__global__ void __launch_bounds__(256) k_stonemask(const float* __restrict__ x, int x_length, int fs, double frame_period,
                                                  const double* __restrict__ f0_in, double* __restrict__ f0_out,
                                                  const double2* __restrict__ tw, int max_fft) {
  extern __shared__ double2 sm2[];
  int frame = blockIdx.x;
  double f0i = f0_in[frame];
  if (f0i <= 40.0 || f0i > fs / 12.0) { if (threadIdx.x == 0) f0_out[frame] = 0.0; return; }
  double pos = frame * frame_period / 1000.0;
  int half = stonemask_half(fs, f0i);
  double wlen_time = (2.0 * half + 1.0) / fs;
  int blen = half * 2 + 1;
  int fft_size = stonemask_fft_size(half);
  // cannot happen for a contour within the plan's f0 range below 27.3 kHz (stonemask_max_fft); never write past the smem
  if (fft_size > max_fft) { if (threadIdx.x == 0) f0_out[frame] = f0i; return; }
  int lg = ilog2(fft_size);
  double2* A = sm2;                 // main
  double2* B = sm2 + max_fft;       // diff
  double* power = (double*)(sm2 + 2 * max_fft);
  double* numer = power + max_fft / 2 + 1;
  int basic_index = matlab_round((pos + (double)(-half) / fs) * fs + 0.001);
  auto mainw = [&](int i) {
    double tmp = ((basic_index + i) - 1.0) / fs - pos;
    return 0.42 + 0.5 * cos(2.0 * kPi * tmp / wlen_time) + 0.08 * cos(4.0 * kPi * tmp / wlen_time);
  };
  for (int i = threadIdx.x; i < fft_size; i += blockDim.x) {
    double a = 0.0, b = 0.0;
    if (i < blen) {
      double xv = (double)x[imax(0, imin(x_length - 1, basic_index + i - 1))];
      double mw = mainw(i), dw;
      if (i == 0) dw = -mainw(1) / 2.0;
      else if (i == blen - 1) dw = mainw(blen - 2) / 2.0;
      else dw = -(mainw(i + 1) - mainw(i - 1)) / 2.0;
      a = xv * mw; b = xv * dw;
    }
    A[i] = make_double2(a, 0.0);
    B[i] = make_double2(b, 0.0);
  }
  fft_smem(A, fft_size, lg, -1, tw);
  fft_smem(B, fft_size, lg, -1, tw);
  for (int j = threadIdx.x; j <= fft_size / 2; j += blockDim.x) {
    double2 m = A[j], d = B[j];
    numer[j] = m.x * d.y - m.y * d.x;
    power[j] = m.x * m.x + m.y * m.y;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double tentative = stonemask_fix(power, numer, fft_size, fs, f0i, 2);
    double mean_f0;
    if (tentative <= 0.0 || tentative > f0i * 2) mean_f0 = 0.0;
    else mean_f0 = stonemask_fix(power, numer, fft_size, fs, tentative, 6);
    if (fabs(mean_f0 - f0i) > f0i * 0.2) mean_f0 = f0i;
    f0_out[frame] = mean_f0;
  }
}

// ------------------------------------------------------------------------------------ shared smoothing helpers
// DCCorrection, in place on a[] (smem). All threads call.
__device__ inline void dc_correction_smem(double* a, double f0, int fs, int fft_size) {
  int upper_limit = 2 + (int)(f0 * fft_size / fs);
  int nrep = upper_limit - 1;
  double dx = -(double)fs / fft_size;
  double rep[2] = {0.0, 0.0};
  int c = 0;
  __syncthreads();
  for (int i = threadIdx.x; i < nrep; i += blockDim.x, ++c)
    rep[c] = interp1q(f0, dx, a, upper_limit + 1, (double)i * fs / fft_size);
  __syncthreads();
  c = 0;
  for (int i = threadIdx.x; i < nrep; i += blockDim.x, ++c) a[i] = a[i] + rep[c];
  __syncthreads();
}

// LinearSmoothing: in[0..half] -> out[0..half] (may alias). seg: scratch >= half + 2*boundary + 1, scan scratch >= blockDim.x
__device__ inline void linear_smoothing_smem(const double* in, double* out, double width, int fs, int fft_size,
                                             double* seg, double* scan_scratch) {
  int half = fft_size / 2;
  int boundary = (int)(width * fft_size / fs) + 1;
  int mlen = half + boundary * 2 + 1;
  __syncthreads();
  for (int i = threadIdx.x; i < mlen; i += blockDim.x) {
    double v;
    if (i < boundary) v = in[boundary - i];
    else if (i < half + boundary) v = in[i - boundary];
    else v = in[half - (i - (half + boundary))];
    seg[i] = v * fs / fft_size;
  }
  __syncthreads();
  block_inclusive_scan(seg, mlen, scan_scratch);
  double origin = -(boundary - 0.5) * fs / fft_size;
  double interval = (double)fs / fft_size;
  for (int i = threadIdx.x; i <= half; i += blockDim.x) {
    double axis = (double)i / fft_size * fs - width / 2.0;
    double low = interp1q(origin, interval, seg, mlen, axis);
    double high = interp1q(origin, interval, seg, mlen, axis + width);
    out[i] = (high - low) / width;
  }
  __syncthreads();
}

// ------------------------------------------------------------------------------------ CheapTrick (+ sp2mc)
// one CTA (256 threads) per frame. DECIDE (matches oracle): randn dither dropped, +eps constant.
constexpr int kCtMaxFft = 2048;
constexpr double kMaxF0Smem = 2000.0;   // StoneMask caps refined f0 at fs/12; scratch is sized for this
__host__ __device__ inline int ct_seg_len(int fft_size, int fs) { return fft_size / 2 + 1 + 2 * ((int)(kMaxF0Smem * 2.0 / 3.0 * fft_size / fs) + 2) + 2; }
__host__ __device__ inline int d4c_seg_len(int fft_d4c, int fs) { return fft_d4c / 2 + 1 + 2 * ((int)(kMaxF0Smem * fft_d4c / fs) + 2) + 2; }
__global__ void __launch_bounds__(256) k_cheaptrick(const float* __restrict__ x, int x_length, int fs, double frame_period,
                                                   const double* __restrict__ f0, int fft_size, double q1,
                                                   const double* __restrict__ G /*[ (order+1) ][nb]*/, int order,
                                                   int n_out, float* __restrict__ sp_out, float* __restrict__ mc_out,
                                                   double* __restrict__ sp_f64 /*nullable*/, const double2* __restrict__ tw) {
  extern __shared__ double2 sm2[];
  int frame = blockIdx.x;
  int half_fft = fft_size / 2, nb = half_fft + 1, lg = ilog2(fft_size);
  double2* A = sm2;                                   // fft_size
  double* ps = (double*)(sm2 + fft_size);             // nb (+1)
  double* seg = ps + nb + 1;                          // nb + 2*boundary + 1  (boundary <= ~ 0.67*f0*fft/fs + 1)
  double* scratch = seg + ct_seg_len(fft_size, fs);   // blockDim.x + 32
  double f0_floor = 3.0 * fs / (fft_size - 3.0);
  double cf0 = f0[frame] <= f0_floor ? kDefaultF0 : f0[frame];
  double pos = frame * frame_period / 1000.0;
  int half = matlab_round(1.5 * fs / cf0);
  int origin = matlab_round(pos * fs + 0.001);
  // window energy
  double acc = 0.0;
  for (int i = threadIdx.x; i <= half * 2; i += blockDim.x) {
    double p = (i - half) / 1.5 / fs;
    double w = 0.5 * cos(kPi * p * cf0) + 0.5;
    acc += w * w;
  }
  double average = sqrt(block_sum(acc, scratch));
  double w1 = 0.0, w2 = 0.0;
  for (int i = threadIdx.x; i < fft_size; i += blockDim.x) {
    double wv = 0.0, v = 0.0;
    if (i <= half * 2) {
      double p = (i - half) / 1.5 / fs;
      wv = (0.5 * cos(kPi * p * cf0) + 0.5) / average;
      int idx = imin(x_length - 1, imax(0, origin + i - half));
      v = (double)x[idx] * wv;
      w1 += v; w2 += wv;
    }
    A[i] = make_double2(v, wv);      // stash the window in .y until the DC removal
  }
  double s1 = block_sum(w1, scratch);
  double s2 = block_sum(w2, scratch);
  double coef = s1 / s2;
  for (int i = threadIdx.x; i < fft_size; i += blockDim.x) {
    double2 v = A[i];
    A[i] = make_double2(i <= half * 2 ? v.x - v.y * coef : 0.0, 0.0);
  }
  fft_smem(A, fft_size, lg, -1, tw);
  for (int i = threadIdx.x; i < nb; i += blockDim.x) { double2 v = A[i]; ps[i] = v.x * v.x + v.y * v.y; }
  if (threadIdx.x == 0) ps[nb] = 0.0;
  dc_correction_smem(ps, cf0, fs, fft_size);
  linear_smoothing_smem(ps, ps, cf0 * 2.0 / 3.0, fs, fft_size, seg, scratch);
  // SmoothingWithRecovery
  for (int i = threadIdx.x; i < fft_size; i += blockDim.x) {
    int k = i <= half_fft ? i : fft_size - i;
    A[i] = make_double2(log(ps[k] + kEps), 0.0);
  }
  fft_smem(A, fft_size, lg, -1, tw);
  for (int i = threadIdx.x; i <= half_fft; i += blockDim.x) {
    double sl, cl;
    if (i == 0) { sl = 1.0; cl = (1.0 - 2.0 * q1) + 2.0 * q1; }
    else {
      double quef = (double)i / fs;
      sl = sin(kPi * cf0 * quef) / (kPi * cf0 * quef);
      cl = (1.0 - 2.0 * q1) + 2.0 * q1 * cos(2.0 * kPi * quef * cf0);
    }
    A[i] = make_double2(A[i].x * sl * cl / fft_size, 0.0);
  }
  irfft_smem(A, fft_size, lg, tw);
  // envelope + fused sp2mc (mc = G . log(sp))
  for (int i = threadIdx.x; i < nb; i += blockDim.x) {
    double spv = exp(A[i].x);
    ps[i] = log(spv);
    if (frame < n_out) {
      sp_out[(size_t)frame * nb + i] = (float)spv;
      if (sp_f64) sp_f64[(size_t)frame * nb + i] = spv;
    }
  }
  __syncthreads();
  for (int j = 0; j <= order; ++j) {
    double a = 0.0;
    for (int i = threadIdx.x; i < nb; i += blockDim.x) a += G[(size_t)j * nb + i] * ps[i];
    double m = block_sum(a, scratch);
    if (threadIdx.x == 0 && frame < n_out) mc_out[(size_t)frame * (order + 1) + j] = (float)m;
  }
}

// ------------------------------------------------------------------------------------ D4C
// windowed waveform into A[i].x (i < fft), zero elsewhere; returns after DC-weight removal.
__device__ inline void d4c_window_smem(double2* A, int fft_size, const float* __restrict__ x, int x_length, int fs,
                                       double cf0, double pos, bool blackman, double ratio, double* scratch) {
  int half = matlab_round(ratio * fs / cf0 / 2.0);
  int origin = matlab_round(pos * fs + 0.001);
  double w1 = 0.0, w2 = 0.0;
  __syncthreads();
  for (int i = threadIdx.x; i < fft_size; i += blockDim.x) {
    double v = 0.0, wv = 0.0;
    if (i <= half * 2) {
      double p = (2.0 * (i - half) / ratio) / fs;
      wv = blackman ? 0.42 + 0.5 * cos(kPi * p * cf0) + 0.08 * cos(kPi * p * cf0 * 2) : 0.5 * cos(kPi * p * cf0) + 0.5;
      int idx = imin(x_length - 1, imax(0, origin + i - half));
      v = (double)x[idx] * wv;
      w1 += v; w2 += wv;
    }
    A[i] = make_double2(v, wv);
  }
  double s1 = block_sum(w1, scratch);
  double s2 = block_sum(w2, scratch);
  double coef = s1 / s2;
  for (int i = threadIdx.x; i < fft_size; i += blockDim.x) {
    double2 v = A[i];
    A[i] = make_double2(i <= half * 2 ? v.x - v.y * coef : 0.0, 0.0);
  }
  __syncthreads();
}

// centroid of the frame at `pos` accumulated into cen[] (+=). tmp: nb doubles x2
__device__ inline void d4c_centroid_smem(double2* A, int fft_size, int lg, const float* __restrict__ x, int x_length, int fs,
                                         double cf0, double pos, double* tr, double* ti, double* cen, bool accumulate,
                                         double* scratch, const double2* __restrict__ tw) {
  int nb = fft_size / 2 + 1;
  d4c_window_smem(A, fft_size, x, x_length, fs, cf0, pos, true, 4.0, scratch);
  int lim = matlab_round(2.0 * fs / cf0) * 2;
  double p = 0.0;
  for (int i = threadIdx.x; i <= lim; i += blockDim.x) p += A[i].x * A[i].x;
  double power = block_sum(p, scratch);
  double sq = sqrt(power);
  for (int i = threadIdx.x; i < fft_size; i += blockDim.x) {
    double v = A[i].x;
    if (i <= lim) v = v / sq;
    A[i] = make_double2(v, 0.0);
  }
  __syncthreads();
  // WORLD needs FFT(v) and FFT((n+1) v): one complex FFT of v + i (n+1) v yields both by Hermitian symmetry.
  for (int i = threadIdx.x; i < fft_size; i += blockDim.x) {
    double v = A[i].x;
    A[i] = make_double2(v, v * (i + 1.0));
  }
  fft_smem(A, fft_size, lg, -1, tw);
  // Z[k] = X[k] + i Y[k];  X[k] = (Z[k] + conj(Z[N-k]))/2,  Y[k] = (Z[k] - conj(Z[N-k]))/(2i)
  for (int k = threadIdx.x; k < nb; k += blockDim.x) {
    double2 z = A[k];
    double2 zc = A[(fft_size - k) & (fft_size - 1)];
    double xr = 0.5 * (z.x + zc.x), xi = 0.5 * (z.y - zc.y);
    double yr = 0.5 * (z.y + zc.y), yi = -0.5 * (z.x - zc.x);
    tr[k] = xr; ti[k] = xi;
    double c = yr * xr + xi * yi;
    cen[k] = accumulate ? cen[k] + c : c;
  }
  __syncthreads();
}

// Sums of the `need` smallest of v[0..n) and of all n values (1 <= need <= n; v >= 0 in smem), without sorting.  The bit patterns of
// non-negative doubles order like their values, so a radix select over them, 8 bits per pass from the top, finds t = the need-th
// smallest value; it stops early once one candidate is left.  sum_lo = sum(v < t) + (copies of t among the need smallest) * t is the
// same multiset sum as a cumulative sum over the sorted values, only in another order.  hist: 256 ints, sel: 4 ints (smem).
__device__ inline void select_sums_smem(const double* v, int n, int need, unsigned* hist, unsigned* sel, double* scratch,
                                        double* sum_lo, double* sum_all) {
  unsigned long long prefix = 0, mask = 0;
  unsigned k = (unsigned)need;          // rank of t among the values that match prefix under mask
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const unsigned long long u = (unsigned long long)__double_as_longlong(v[i]);
      if ((u & mask) == prefix) atomicAdd(&hist[(u >> shift) & 255], 1u);
    }
    __syncthreads();
    if (threadIdx.x < 32) {             // warp 0: the bin that holds rank k (lane l owns bins 8 l .. 8 l + 7)
      const int l = threadIdx.x;
      unsigned c[8], own = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) { c[j] = hist[l * 8 + j]; own += c[j]; }
      unsigned incl = own;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const unsigned y = __shfl_up_sync(0xffffffffu, incl, off);
        if (l >= off) incl += y;
      }
      unsigned run = incl - own;
      if (run < k && k <= incl) {
        for (int j = 0; j < 8; ++j) {
          if (k <= run + c[j]) { sel[0] = l * 8 + j; sel[1] = k - run; sel[2] = c[j]; break; }
          run += c[j];
        }
      }
    }
    __syncthreads();
    const unsigned digit = sel[0], cnt = sel[2];
    k = sel[1];
    prefix |= (unsigned long long)digit << shift;
    mask |= 255ull << shift;
    if (cnt == 1) break;                // block-uniform: read from smem
  }
  // t = the candidate left (unique), or every candidate (all equal once the mask is full)
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x)
    if (((unsigned long long)__double_as_longlong(v[i]) & mask) == prefix) scratch[0] = v[i];
  __syncthreads();
  const double t = scratch[0];
  double lo = 0.0, all = 0.0;
  for (int i = threadIdx.x; i < n; i += blockDim.x) { const double x = v[i]; all += x; if (x < t) lo += x; }
  // the values below t are need - k of the need smallest; k copies of t complete them
  const double s_lo = block_sum(lo, scratch);
  *sum_all = block_sum(all, scratch);
  *sum_lo = s_lo + (double)k * t;
}

// one CTA (512 threads) per frame
__global__ void __launch_bounds__(512) k_d4c(const float* __restrict__ x, int x_length, int fs, double frame_period,
                                            const double* __restrict__ f0, int fft_size_out, double threshold,
                                            int n_out, float* __restrict__ ap_out, const double2* __restrict__ tw,
                                            int fft_d4c, int lt_fft) {
  extern __shared__ double2 sm2[];
  int frame = blockIdx.x;
  if (frame >= n_out) return;
  const int nb_out = fft_size_out / 2 + 1;
  float* out = ap_out + (size_t)frame * nb_out;
  const int maxfft = fft_d4c > lt_fft ? fft_d4c : lt_fft;
  double2* A = sm2;
  double* base = (double*)(sm2 + maxfft);
  const int hb = fft_d4c / 2 + 1;
  const int alen = hb + 8;
  double* sc = base;                  // static centroid
  double* sps = sc + alen;            // smoothed power spectrum
  double* gd = sps + alen;            // group delay
  double* t1 = gd + alen;             // temp
  double* t2 = t1 + alen;             // temp
  double* seg = t2 + alen;            // smoothing scratch (hb + 2*boundary + 1)
  double* scratch = seg + d4c_seg_len(fft_d4c, fs);   // blockDim.x + 32
  double f0v = f0[frame];
  double pos = frame * frame_period / 1000.0;
  const float unvoiced = (float)(1.0 - kSafeMin);
  bool skip = f0v == 0.0;
  if (!skip) {
    // D4C LoveTrain
    int lg = ilog2(lt_fft);
    double cf0 = f0v > 40.0 ? f0v : 40.0;
    d4c_window_smem(A, lt_fft, x, x_length, fs, cf0, pos, true, 3.0, scratch);
    fft_smem(A, lt_fft, lg, -1, tw);
    int b0 = (int)ceil(100.0 * lt_fft / fs), b1 = (int)ceil(4000.0 * lt_fft / fs), b2 = (int)ceil(7900.0 * lt_fft / fs);
    double p1 = 0.0, p2 = 0.0;
    for (int i = b0 + 1 + threadIdx.x; i <= b2; i += blockDim.x) {
      double2 v = A[i];
      double pw = v.x * v.x + v.y * v.y;
      p2 += pw;
      if (i <= b1) p1 += pw;
    }
    double s1 = block_sum(p1, scratch), s2 = block_sum(p2, scratch);
    double ap0 = s1 / s2;
    skip = ap0 <= threshold;     // NaN compares false, exactly like the CPU code path
  }
  if (skip) {
    for (int i = threadIdx.x; i < nb_out; i += blockDim.x) out[i] = unvoiced;
    return;
  }
  int lg = ilog2(fft_d4c);
  double cf0 = f0v > 47.0 ? f0v : 47.0;
  d4c_centroid_smem(A, fft_d4c, lg, x, x_length, fs, cf0, pos - 0.25 / cf0, t1, t2, sc, false, scratch, tw);
  d4c_centroid_smem(A, fft_d4c, lg, x, x_length, fs, cf0, pos + 0.25 / cf0, t1, t2, sc, true, scratch, tw);
  if (threadIdx.x == 0) sc[hb] = 0.0;
  dc_correction_smem(sc, cf0, fs, fft_d4c);
  // smoothed power spectrum
  d4c_window_smem(A, fft_d4c, x, x_length, fs, cf0, pos, false, 4.0, scratch);
  fft_smem(A, fft_d4c, lg, -1, tw);
  for (int i = threadIdx.x; i < hb; i += blockDim.x) { double2 v = A[i]; sps[i] = v.x * v.x + v.y * v.y; }
  if (threadIdx.x == 0) sps[hb] = 0.0;
  dc_correction_smem(sps, cf0, fs, fft_d4c);
  linear_smoothing_smem(sps, sps, cf0, fs, fft_d4c, seg, scratch);
  // static group delay
  for (int i = threadIdx.x; i < hb; i += blockDim.x) gd[i] = sc[i] / sps[i];
  linear_smoothing_smem(gd, gd, cf0 / 2.0, fs, fft_d4c, seg, scratch);
  linear_smoothing_smem(gd, t1, cf0, fs, fft_d4c, seg, scratch);
  for (int i = threadIdx.x; i < hb; i += blockDim.x) gd[i] -= t1[i];
  __syncthreads();
  // coarse aperiodicity
  const int nap = (int)(fmin(15000.0, fs / 2.0 - 3000.0) / 3000.0);
  const int window_length = (int)(3000.0 * fft_d4c / fs) * 2 + 1;
  const int half_wl = window_length / 2;
  const int boundary = matlab_round(fft_d4c * 8.0 / window_length);
  double* coarse = t2;                // nap + 2 values
  unsigned* hist = (unsigned*)A;      // selection histogram (256) + result (4): A is free once the power spectrum is in t1
  if (threadIdx.x == 0) { coarse[0] = -60.0; coarse[nap + 1] = -kSafeMin; }
  for (int b = 0; b < nap; ++b) {
    int center = (int)(3000.0 * (b + 1) * fft_d4c / fs);
    __syncthreads();
    for (int i = threadIdx.x; i < fft_d4c; i += blockDim.x) {
      double v = 0.0;
      if (i <= half_wl * 2) {
        double tmp = i / (window_length - 1.0);
        double w = 0.355768 - 0.487396 * cos(2.0 * kPi * tmp) + 0.144232 * cos(4.0 * kPi * tmp) - 0.012604 * cos(6.0 * kPi * tmp);
        v = gd[center - half_wl + i] * w;
      }
      A[i] = make_double2(v, 0.0);
    }
    fft_smem(A, fft_d4c, lg, -1, tw);
    // power spectrum -> t1 (hb values); WORLD sorts it and takes the cumulative sums at fft / 2 - boundary - 1 and fft / 2 (= all):
    // the sum of all but the boundary + 1 largest values, and the sum of all of them
    for (int i = threadIdx.x; i < hb; i += blockDim.x) { double2 v = A[i]; t1[i] = v.x * v.x + v.y * v.y; }
    __syncthreads();
    double sa, sb;
    select_sums_smem(t1, hb, fft_d4c / 2 - boundary, hist, hist + 256, scratch, &sa, &sb);
    if (threadIdx.x == 0) {
      double ca = 10 * log10(sa / sb);
      coarse[1 + b] = fmin(0.0, ca + (cf0 - 100) / 50.0);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nb_out; i += blockDim.x) {
    double fx = (double)i * fs / fft_size_out;
    // coarse axis: k*3000 for k<=nap, fs/2 at nap+1
    int n = nap + 2;
    int lo = 0, hi = n;
    while (lo < hi) {
      int mid = (lo + hi) >> 1;
      double xm = mid <= nap ? mid * 3000.0 : fs / 2.0;
      if (xm <= fx) lo = mid + 1; else hi = mid;
    }
    int k = lo < 1 ? 1 : (lo > n - 1 ? n - 1 : lo);
    double x0 = (k - 1) <= nap ? (k - 1) * 3000.0 : fs / 2.0;
    double x1 = k <= nap ? k * 3000.0 : fs / 2.0;
    double s = (fx - x0) / (x1 - x0);
    double v = coarse[k - 1] + s * (coarse[k] - coarse[k - 1]);
    out[i] = (float)pow(10.0, v / 20.0);
  }
}

// f0 / voiced outputs (float32 / uint8), trimmed to n_out frames
__global__ void k_f0_out(const double* __restrict__ f0, int n_out, float* __restrict__ f0_out, uint8_t* __restrict__ voiced) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n_out) { double v = f0[i]; f0_out[i] = (float)v; voiced[i] = v != 0.0 ? 1 : 0; }
}

// ------------------------------------------------------------------------------------ host side
struct DioPlan {
  int n = 0, fs = 0, fft_size = 0, y_length = 0, f0_length = 0, nbands = 0;
  double frame_period = 0, f0_floor = 0, f0_ceil = 0;
  cufftHandle fwd = 0, inv = 0, fwd_filters = 0;
  double* d_y = nullptr; cufftDoubleComplex* d_Y = nullptr; cufftDoubleComplex* d_filt_spec = nullptr;   // [1+nbands][nbins]
  cufftDoubleComplex* d_Z = nullptr; double* d_filtered = nullptr;
  int* d_half_avg = nullptr; double* d_boundary = nullptr;
  int* d_edges = nullptr; double* d_loc = nullptr; double* d_itv = nullptr; int* d_counts = nullptr;
  double* d_cand = nullptr; double* d_score = nullptr; double* d_scratch = nullptr; int* d_iscratch = nullptr;
  double* d_f0 = nullptr; double* d_f0r = nullptr;
  HarvestPlan* harvest = nullptr;          // f0 method 1: Harvest writes d_f0 instead of DIO
  int sm_fft = 0;                          // largest FFT k_stonemask can form on this plan's f0 contours (its smem stride)
};


void dio_plan_free(DioPlan* p) {
  if (!p) return;
  harvest_plan_free(p->harvest);
  if (p->fwd) cufftDestroy(p->fwd);
  if (p->inv) cufftDestroy(p->inv);
  if (p->fwd_filters) cufftDestroy(p->fwd_filters);
  void* ptrs[] = {p->d_y, p->d_Y, p->d_filt_spec, p->d_Z, p->d_filtered, p->d_half_avg, p->d_boundary, p->d_edges, p->d_loc,
                  p->d_itv, p->d_counts, p->d_cand, p->d_score, p->d_scratch, p->d_iscratch, p->d_f0, p->d_f0r};
  for (void* q : ptrs) if (q) cudaFree(q);
  delete p;
}

int dio_plan_create(Engine* e, int n, int fs, double frame_period, double f0_floor, double f0_ceil, DioPlan** out, int f0_method) {
  DioPlan* p = new DioPlan();
  if (f0_method == 1 && harvest_plan_create(e, n, fs, frame_period, f0_floor, f0_ceil, &p->harvest)) { delete p; return -1; }
  p->n = n; p->fs = fs; p->frame_period = frame_period; p->f0_floor = f0_floor; p->f0_ceil = f0_ceil;
  // DIO's contour is 0 or a band candidate >= f0_floor (k_dio_candidates zeroes the rest; the repair only copies candidates).  Harvest's
  // lowest output is not bounded by f0_floor in a way this code shows, so its plans keep the bound of k_stonemask itself (40 Hz).
  p->sm_fft = stonemask_max_fft(fs, f0_method == 1 ? 40.0 : f0_floor);
  p->nbands = 1 + (int)(log(f0_ceil / f0_floor) / kLog2 * 2.0);
  std::vector<double> boundary(p->nbands);
  std::vector<int> half_avg(p->nbands);
  for (int i = 0; i < p->nbands; ++i) {
    boundary[i] = f0_floor * pow(2.0, (i + 1) / 2.0);
    half_avg[i] = matlab_round((double)fs / boundary[i] / 2.0);
  }
  p->y_length = n + 1;
  p->fft_size = suitable_fft_size(p->y_length + matlab_round((double)fs / 50.0) * 2 + 1 + (4 * (int)(1.0 + (double)fs / boundary[0] / 2.0)));
  p->f0_length = (int)(1000.0 * n / fs / frame_period) + 1;
  int nbins = p->fft_size / 2 + 1;
  size_t ev = (size_t)p->nbands * 4 * p->y_length;
  RYK_CUDA(cudaMalloc(&p->d_y, sizeof(double) * p->fft_size));
  RYK_CUDA(cudaMalloc(&p->d_Y, sizeof(cufftDoubleComplex) * nbins));
  RYK_CUDA(cudaMalloc(&p->d_filt_spec, sizeof(cufftDoubleComplex) * nbins * (1 + p->nbands)));
  RYK_CUDA(cudaMalloc(&p->d_Z, sizeof(cufftDoubleComplex) * nbins * p->nbands));
  RYK_CUDA(cudaMalloc(&p->d_filtered, sizeof(double) * (size_t)p->fft_size * (1 + p->nbands)));
  RYK_CUDA(cudaMalloc(&p->d_half_avg, sizeof(int) * p->nbands));
  RYK_CUDA(cudaMalloc(&p->d_boundary, sizeof(double) * p->nbands));
  RYK_CUDA(cudaMalloc(&p->d_edges, sizeof(int) * ev));
  RYK_CUDA(cudaMalloc(&p->d_loc, sizeof(double) * ev));
  RYK_CUDA(cudaMalloc(&p->d_itv, sizeof(double) * ev));
  RYK_CUDA(cudaMalloc(&p->d_counts, sizeof(int) * p->nbands * 4));
  RYK_CUDA(cudaMalloc(&p->d_cand, sizeof(double) * p->nbands * p->f0_length));
  RYK_CUDA(cudaMalloc(&p->d_score, sizeof(double) * p->nbands * p->f0_length));
  RYK_CUDA(cudaMalloc(&p->d_scratch, sizeof(double) * 3 * p->f0_length));
  RYK_CUDA(cudaMalloc(&p->d_iscratch, sizeof(int) * 2 * p->f0_length));
  RYK_CUDA(cudaMalloc(&p->d_f0, sizeof(double) * p->f0_length));
  RYK_CUDA(cudaMalloc(&p->d_f0r, sizeof(double) * p->f0_length));
  RYK_CUDA(cudaMemcpyAsync(p->d_half_avg, half_avg.data(), sizeof(int) * p->nbands, cudaMemcpyHostToDevice, e->stream));
  RYK_CUDA(cudaMemcpyAsync(p->d_boundary, boundary.data(), sizeof(double) * p->nbands, cudaMemcpyHostToDevice, e->stream));
  if (cufft_ok(cufftPlan1d(&p->fwd, p->fft_size, CUFFT_D2Z, 1), "plan D2Z")) return -1;
  if (cufft_ok(cufftPlan1d(&p->inv, p->fft_size, CUFFT_Z2D, p->nbands), "plan Z2D")) return -1;
  if (cufft_ok(cufftPlan1d(&p->fwd_filters, p->fft_size, CUFFT_D2Z, 1 + p->nbands), "plan D2Z filters")) return -1;
  // filter spectra, computed once (d_filtered doubles as the time-domain staging area)
  if (cufft_ok(cufftSetStream(p->fwd_filters, e->stream), "set stream")) return -1;
  k_dio_design_filters<<<1 + p->nbands, 256, 0, e->stream>>>(p->d_filtered, p->fft_size, matlab_round((double)fs / 50.0) * 2 + 1, p->d_half_avg);
  if (cufft_ok(cufftExecD2Z(p->fwd_filters, p->d_filtered, p->d_filt_spec), "exec filters")) return -1;
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  RYK_CUDA(cudaGetLastError());
  cufftDestroy(p->fwd_filters); p->fwd_filters = 0;
  *out = p;
  return 0;
}

// DIO + StoneMask: x (device float32, n samples) -> plan->d_f0r (double, f0_length frames). Stream-ordered, no sync.
int dio_stonemask_run(Engine* e, DioPlan* p, const float* d_x, cudaStream_t st) {
  const size_t sm_smem = stonemask_smem_bytes(p->sm_fft);
  if (p->harvest) {                                  // Harvest replaces DIO as the contour StoneMask refines
    if (harvest_run(e, p->harvest, d_x, p->d_f0, st)) return -1;
    k_stonemask<<<p->f0_length, 256, sm_smem, st>>>(d_x, p->n, p->fs, p->frame_period, p->d_f0, p->d_f0r, e->d_twiddle, p->sm_fft);
    RYK_CUDA(cudaGetLastError());
    return 0;
  }
  int nbins = p->fft_size / 2 + 1;
  if (cufft_ok(cufftSetStream(p->fwd, st), "set stream")) return -1;
  if (cufft_ok(cufftSetStream(p->inv, st), "set stream")) return -1;
  k_dio_prepare<<<1, 1024, 0, st>>>(d_x, p->n, p->y_length, p->fft_size, p->d_y);
  if (cufft_ok(cufftExecD2Z(p->fwd, p->d_y, p->d_Y), "exec D2Z")) return -1;
  k_cmul_inplace<<<(nbins + 255) / 256, 256, 0, st>>>(p->d_Y, p->d_filt_spec, nbins);
  k_band_mul<<<dim3((nbins + 255) / 256, p->nbands), 256, 0, st>>>(p->d_Y, p->d_filt_spec + nbins, p->d_Z, nbins);
  if (cufft_ok(cufftExecZ2D(p->inv, p->d_Z, p->d_filtered), "exec Z2D")) return -1;
  k_dio_zero_cross<<<dim3(4, p->nbands), 1024, 0, st>>>(p->d_filtered, p->fft_size, p->y_length, p->d_half_avg, 2, 0, (double)p->fs,
                                                      p->d_edges, p->d_loc, p->d_itv, p->d_counts);
  k_dio_candidates<<<dim3((p->f0_length + 127) / 128, p->nbands), 128, 0, st>>>(
      p->d_loc, p->d_itv, p->d_counts, p->y_length, p->f0_length, p->nbands, p->frame_period, p->f0_floor, p->f0_ceil,
      p->d_boundary, p->d_cand, p->d_score);
  k_dio_fix<<<1, 256, 0, st>>>(p->d_cand, p->d_score, p->nbands, p->f0_length, p->frame_period, p->f0_floor, p->d_scratch,
                               p->d_iscratch, p->d_f0);
  k_stonemask<<<p->f0_length, 256, sm_smem, st>>>(d_x, p->n, p->fs, p->frame_period, p->d_f0, p->d_f0r, e->d_twiddle, p->sm_fft);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

const double* dio_plan_f0(DioPlan* p) { return p->d_f0r; }
double* dio_plan_f0_mut(DioPlan* p) { return p->d_f0r; }
int dio_plan_frames(DioPlan* p) { return p->f0_length; }
HarvestPlan* dio_plan_harvest(DioPlan* p) { return p->harvest; }
const double* dio_plan_f0_raw(DioPlan* p) { return p->d_f0; }

size_t cheaptrick_smem_bytes(int fft_size, int fs) {
  int nb = fft_size / 2 + 1;
  return sizeof(double2) * fft_size + sizeof(double) * ((nb + 1) + ct_seg_len(fft_size, fs) + 256 + 64);
}

size_t d4c_smem_bytes(int fs) {
  int fft_d4c = (int)pow(2.0, 1.0 + (int)(log(4.0 * fs / 47.0 + 1) / kLog2));
  int lt_fft = (int)pow(2.0, 1.0 + (int)(log(3.0 * fs / 40.0 + 1) / kLog2));
  int maxfft = fft_d4c > lt_fft ? fft_d4c : lt_fft;
  int hb = fft_d4c / 2 + 1;
  return sizeof(double2) * maxfft + sizeof(double) * (5 * (hb + 8) + d4c_seg_len(fft_d4c, fs) + 512 + 64);
}

int analysis_kernels_init() {
  RYK_CUDA(cudaFuncSetAttribute(k_stonemask, cudaFuncAttributeMaxDynamicSharedMemorySize, 170 * 1024));
  RYK_CUDA(cudaFuncSetAttribute(k_cheaptrick, cudaFuncAttributeMaxDynamicSharedMemorySize, 100 * 1024));
  RYK_CUDA(cudaFuncSetAttribute(k_d4c, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  return 0;
}

// CheapTrick(+sp2mc) and D4C on the refined f0 in d_f0 (double, >= n_out frames). Stream-ordered.
// Both read only the wave and the f0 and write disjoint outputs.  With a side stream (st being captured) D4C is forked onto it and
// joined back, so the captured graph holds CheapTrick (+ f0 out) and D4C as two concurrent branches; otherwise they run in turn on st.
int spectral_analysis_run(Engine* e, const float* d_x, int n, int fs, double frame_period, const double* d_f0, int n_out,
                          int fft_size, int order, const double* d_G, float* d_sp, float* d_ap, float* d_mc, float* d_f0_out,
                          uint8_t* d_voiced, cudaStream_t st, cudaStream_t side) {
  RYK_CHECK(fft_size <= kCtMaxFft && fft_size >= 64, "unsupported CheapTrick fft size");
  if (n_out <= 0) return 0;
  const int fft_d4c = (int)pow(2.0, 1.0 + (int)(log(4.0 * fs / 47.0 + 1) / kLog2));   // host pow: exact
  const int lt_fft = (int)pow(2.0, 1.0 + (int)(log(3.0 * fs / 40.0 + 1) / kLog2));
  cudaEvent_t fork = nullptr, join = nullptr;
  cudaStream_t sd = st;
  if (side) {
    RYK_CUDA(cudaEventCreateWithFlags(&fork, cudaEventDisableTiming));
    RYK_CUDA(cudaEventCreateWithFlags(&join, cudaEventDisableTiming));
    RYK_CUDA(cudaEventRecord(fork, st));
    RYK_CUDA(cudaStreamWaitEvent(side, fork, 0));
    sd = side;
  }
  k_d4c<<<n_out, 512, d4c_smem_bytes(fs), sd>>>(d_x, n, fs, frame_period, d_f0, fft_size, 0.85, n_out, d_ap, e->d_twiddle, fft_d4c, lt_fft);
  k_cheaptrick<<<n_out, 256, cheaptrick_smem_bytes(fft_size, fs), st>>>(d_x, n, fs, frame_period, d_f0, fft_size, -0.15, d_G, order,
                                                                      n_out, d_sp, d_mc, nullptr, e->d_twiddle);
  k_f0_out<<<(n_out + 127) / 128, 128, 0, st>>>(d_f0, n_out, d_f0_out, d_voiced);
  RYK_CUDA(cudaGetLastError());
  if (side) {
    RYK_CUDA(cudaEventRecord(join, side));
    RYK_CUDA(cudaStreamWaitEvent(st, join, 0));
    RYK_CUDA(cudaEventDestroy(fork));           // the captured graph keeps the dependencies, not the events
    RYK_CUDA(cudaEventDestroy(join));
  }
  return 0;
}

}  // namespace ryk
