// world_harvest.cu -- WORLD Harvest f0 extraction on the H100 (pyworld.harvest; the f0 hook of yukarin.AcousticFeature.extract reached
// from realtime_voice_conversion/yukarin_wrapper/acoustic_feature_wrapper.py:28-33; f0_estimating_method='harvest', SURVEY A.2 / A.7).
// Selected with ryk_engine_set_f0_method(e, 1); the result feeds StoneMask exactly like DIO's does (DESIGN, DECIDE H3).
//
// Mapping to the hardware (FP64 throughout; FFT / scan / compare work, no tensor cores):
//   * decimation to ~8 kHz is WORLD's zero-phase 3rd-order Chebyshev IIR -- a sequential recurrence, cut into per-thread segments with
//     a warm-up prefix that the filter's pole radius makes exact to 1e-21 (hv_filter_for_decimate);
//   * the 40-channels-per-octave band-pass bank is ONE batched cuFFT Z2D over cached filter spectra (152 channels x 4096 points),
//     followed by the ordered zero-crossing extraction shared with DIO (analysis_shared.cuh), one CTA per (event type, channel);
//   * candidate detection / overlap / removal are one thread per frame or per (frame, candidate);
//   * refinement (GetRefinedF0) needs the spectra of two windowed segments at <= 6 harmonic bins only: one WARP per candidate
//     evaluates those bins directly (windowed DFT with table twiddles) instead of two full FFTs;
//   * FixF0Contour is inherently sequential over the 1 ms frames: one warp, with every SelectBestF0 / SearchScore scan over the
//     candidate columns done warp-parallel with the reference's tie-breaking (last minimal candidate wins);
//   * smoothing is the reference's forward-backward 2nd-order Butterworth per voiced section: one thread per section.
// Everything is stream-ordered without host synchronisation, so the session can capture it inside its analysis graph.
#include <cufft.h>
#include <math.h>

#include <vector>

#include "analysis_shared.cuh"
#include "engine.h"
#include "fft.cuh"

namespace ryk {

struct HarvestPlan {
  int n = 0, fs = 0, ratio = 1, y_length = 0, fft_size = 0, channels = 0, nf1 = 0, max_cand = 0, f0_length = 0, lag = 0, n_pad = 0, max_sections = 0;
  double frame_period = 0, f0_floor = 0, f0_ceil = 0, actual_fs = 0;
  cufftHandle fwd = 0, inv = 0;
  double *d_t1 = nullptr, *d_t2 = nullptr;          // decimation scratch (n_pad each)
  double* d_y = nullptr;                            // [fft_size]
  cufftDoubleComplex *d_Y = nullptr, *d_F = nullptr, *d_Z = nullptr;     // [nbins], [channels][nbins] x 2
  double* d_filtered = nullptr;                     // [channels][fft_size]
  int* d_flh = nullptr; double* d_boundary = nullptr;
  int* d_edges = nullptr; double *d_loc = nullptr, *d_itv = nullptr; int* d_counts = nullptr;
  double* d_raw = nullptr;                          // [channels][nf1]
  double *d_cand = nullptr, *d_score = nullptr, *d_tmpc = nullptr;      // [nf1][max_cand]
  int* d_nc = nullptr;                              // base candidates per frame (max over frames)
  double *d_best = nullptr, *d_basic = nullptr;     // [nf1]
  double* d_work = nullptr; int* d_iwork = nullptr; // contour / smoothing scratch
};

__constant__ double c_dec_a[13][3] = {{0, 0, 0}, {0, 0, 0},
  {0.041156734567757161, -0.42599112459189592, 0.041037215479961149},
  {0.95039378983237421, -0.67429146741526802, 0.15412211621346472},
  {1.4499664446880223, -0.98943497080950538, 0.24578252340690199},
  {1.761093965428056, -1.255491484385977, 0.32371865077882145},
  {1.9715352749512141, -1.4686795689225343, 0.38939084349657005},
  {2.1225239019534698, -1.6395144861046296, 0.44469707800587344},
  {2.2357462340187593, -1.7780899984041356, 0.49152555365968698},
  {2.3236003491759578, -1.89215456174636, 0.53148928133729068},
  {2.3936475118069382, -1.9873904075111852, 0.56588799790270516},
  {2.450743295230728, -2.0679490460197805, 0.59574774438332112},
  {2.4981398605924205, -2.1368928194784025, 0.62187513816221485}};
__constant__ double c_dec_b[13][2] = {{0, 0}, {0, 0},
  {0.16797464681802221, 0.50392394045406663},
  {0.071221945171178622, 0.21366583551353585},
  {0.03671075033932264, 0.11013225101796792},
  {0.021334858522387451, 0.064004575567162353},
  {0.013469181309343806, 0.04040754392803142},
  {0.0090366882681607811, 0.027110064804482345},
  {0.0063522763407111793, 0.019056829022133539},
  {0.0046331164041389242, 0.013899349212416773},
  {0.0034818622251927374, 0.010445586675578211},
  {0.0026822508007164039, 0.0080467524021492123},
  {0.0021097275904708771, 0.0063291827714126309}};

// FilterForDecimate, all threads of the CTA: the recurrence is sequential (4 dependent FP64 operations per sample: ~1 ms for the 15 k
// steps of a 0.3 s chunk on one thread), but the filter is stable with pole radius rho(r) <= 0.89, so thread t can start `warm` samples
// before its own segment from a zero state -- after `warm` steps the state differs from the true one by rho^warm < 1e-21 of the signal
// (c_dec_warm = 1.25 * 17 ln 10 / -ln rho) -- and then produces its segment with the CPU restatement's operation order (explicit
// rounding, no FMA contraction).  Thread 0 and every thread whose warm-up reaches the start of the signal are exact.
__constant__ int c_dec_warm[13] = {0, 0, 117, 130, 156, 186, 218, 250, 283, 317, 350, 384, 417};
__device__ inline void hv_filter_for_decimate(const double* __restrict__ x, int n, int r, double* __restrict__ y) {
  const double a0 = c_dec_a[r][0], a1 = c_dec_a[r][1], a2 = c_dec_a[r][2], b0 = c_dec_b[r][0], b1 = c_dec_b[r][1];
  const int seg = (n + blockDim.x - 1) / blockDim.x;
  const int lo = threadIdx.x * seg, hi = min(n, lo + seg);
  if (lo >= hi) return;
  double w0 = 0.0, w1 = 0.0, w2 = 0.0;
  for (int i = max(0, lo - c_dec_warm[r]); i < hi; ++i) {
    const double wt = __dadd_rn(__dadd_rn(__dadd_rn(x[i], __dmul_rn(a0, w0)), __dmul_rn(a1, w1)), __dmul_rn(a2, w2));
    if (i >= lo) y[i] = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(b0, wt), __dmul_rn(b1, w0)), __dmul_rn(b1, w1)), __dmul_rn(b0, w2));
    w2 = w1; w1 = w0; w0 = wt;
  }
}

// GetWaveformAndSpectrumSub + DC removal.  x: n float32 samples; y: fft_size doubles (decimated signal, mean removed, zero padded).
__global__ void __launch_bounds__(512) k_hv_decimate(const float* __restrict__ x, int n, int ratio, int lag, int y_length, int fft_size,
                                                    double* __restrict__ t1, double* __restrict__ t2, double* __restrict__ y) {
  __shared__ double scratch[32];
  const int T = blockDim.x, tid = threadIdx.x;
  if (ratio == 1) {
    for (int i = tid; i < fft_size; i += T) y[i] = i < n ? (double)x[i] : 0.0;
  } else {
    const int nx = n + 2 * lag;                       // new_x: x[0] * lag, x, x[n - 1] * lag
    const int nf = 9, np = nx + 2 * nf;               // decimate(): reflect 9 samples on both sides
    auto new_x = [&](int i) -> double { return (double)x[i < lag ? 0 : (i < lag + n ? i - lag : n - 1)]; };
    for (int i = tid; i < np; i += T) {
      double v;
      if (i < nf) v = 2 * new_x(0) - new_x(nf - i);
      else if (i < nf + nx) v = new_x(i - nf);
      else v = 2 * new_x(nx - 1) - new_x(nx - 2 - (i - (nf + nx)));
      t1[i] = v;
    }
    __syncthreads();
    hv_filter_for_decimate(t1, np, ratio, t2);
    __syncthreads();
    for (int i = tid; i < np; i += T) t1[i] = t2[np - i - 1];
    __syncthreads();
    hv_filter_for_decimate(t1, np, ratio, t2);
    __syncthreads();
    // tmp1[i] = t2[np - i - 1];  y_dec[count] = tmp1[nbeg + count * r + nf - 1];  y[i] = y_dec[lag / r + i]
    const int nout = (nx - 1) / ratio + 1;
    const int nbeg = ratio - ratio * nout + nx;
    for (int i = tid; i < fft_size; i += T) {
      double v = 0.0;
      if (i < y_length) {
        const int c = lag / ratio + i;
        const int src = nbeg + c * ratio + nf - 1;      // index into the twice-reversed array
        v = (c < nout && src < np) ? t2[np - src - 1] : 0.0;
      }
      y[i] = v;
    }
  }
  __syncthreads();
  double s = 0.0;
  for (int i = tid; i < y_length; i += T) s += y[i];
  const double mean = block_sum(s, scratch) / y_length;
  for (int i = tid; i < y_length; i += T) y[i] -= mean;
}

// time-domain band-pass filters (Nuttall window x cosine carrier), one CTA per channel; spectra are cached in the plan
__global__ void k_hv_design_filters(double* __restrict__ filt, int fft_size, const int* __restrict__ flh, const double* __restrict__ boundary,
                                    double fs) {
  const int ch = blockIdx.x, h = flh[ch], len = 2 * h + 1;
  double* f = filt + (size_t)ch * fft_size;
  const double bf = boundary[ch];
  for (int i = threadIdx.x; i < fft_size; i += blockDim.x) {
    double v = 0.0;
    if (i < len) {
      const double tmp = i / (len - 1.0);
      v = 0.355768 - 0.487396 * cos(2.0 * kPi * tmp) + 0.144232 * cos(4.0 * kPi * tmp) - 0.012604 * cos(6.0 * kPi * tmp);
      v *= cos(2 * kPi * bf * (i - h) / fs);
    }
    f[i] = v;
  }
}

// GetF0CandidateContour: raw[ch][i] at the 1 ms basic frames
__global__ void k_hv_raw_candidates(const double* __restrict__ loc, const double* __restrict__ itv, const int* __restrict__ counts, int y_length,
                                    int nf1, double f0_floor, double f0_ceil, const double* __restrict__ boundary, double* __restrict__ raw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, ch = blockIdx.y;
  if (i >= nf1) return;
  const int* c = counts + ch * 4;
  double cv = 0.0;
  if (c[0] > 2 && c[1] > 2 && c[2] > 2 && c[3] > 2) {
    const double t = i * 1.0 / 1000.0;
    double v[4];
    for (int e = 0; e < 4; ++e) {
      const size_t slot = ((size_t)ch * 4 + e) * y_length;
      v[e] = interp1_at(loc + slot, itv + slot, c[e], t);
    }
    cv = (v[0] + v[1] + v[2] + v[3]) / 4.0;
    const double bf = boundary[ch], upper = bf * 1.1, lower = bf * 0.9;
    if (cv > upper || cv < lower || cv > f0_ceil || cv < f0_floor) cv = 0.0;
  }
  raw[(size_t)ch * nf1 + i] = cv;
}

// DetectOfficialF0Candidates: one thread per frame walks the channels; candidate = mean over a run of >= 10 agreeing channels
__global__ void k_hv_detect(const double* __restrict__ raw, int channels, int nf1, int max_cand, double* __restrict__ cand,
                            double* __restrict__ score, int* __restrict__ nc_max) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nf1) return;
  double* row = cand + (size_t)i * max_cand;
  for (int j = 0; j < max_cand; ++j) { row[j] = 0.0; score[(size_t)i * max_cand + j] = 0.0; }
  int nc = 0, st = 0, prev = 0;
  for (int j = 1; j < channels; ++j) {
    const int cur = (j == channels - 1) ? 0 : (raw[(size_t)j * nf1 + i] > 0 ? 1 : 0);      // vuv[0] = vuv[channels - 1] = 0
    if (cur - prev == 1) st = j;
    if (cur - prev == -1) {
      const int ed = j;
      if (ed - st >= 10) {
        double s = 0.0;
        for (int k = st; k < ed; ++k) s += raw[(size_t)k * nf1 + i];
        s /= (ed - st);
        if (nc < max_cand / 7) row[nc++] = s;
      }
    }
    prev = cur;
  }
  if (nc > 0) atomicMax(nc_max, nc);
}

// OverlapF0Candidates: columns [nc .. 7 nc) are the base columns of frames k -+ 1..3
__global__ void k_hv_overlap(double* __restrict__ cand, int nf1, int max_cand, const int* __restrict__ nc_max) {
  const int nc = *nc_max;
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nf1 || nc <= 0) return;
  for (int i = 1; i <= 3; ++i)
    for (int j = 0; j < nc; ++j) {
      cand[(size_t)k * max_cand + j + nc * i] = k >= i ? cand[(size_t)(k - i) * max_cand + j] : 0.0;
      cand[(size_t)k * max_cand + j + nc * (i + 3)] = k < nf1 - i ? cand[(size_t)(k + i) * max_cand + j] : 0.0;
    }
}

// GetRefinedF0: one warp per (frame, candidate column).  Only the <= 6 harmonic bins of the two windowed spectra are needed, so they
// are evaluated directly: X[k] = sum_n x[n] w[n] exp(-2 pi i k n / N), twiddles from the engine's exact table (N <= 4096 divides it).
__global__ void __launch_bounds__(128) k_hv_refine(const double* __restrict__ y, int y_length, double fs, int nf1, int max_cand,
                                                  const int* __restrict__ nc_max, double f0_floor, double f0_ceil, double* __restrict__ cand,
                                                  double* __restrict__ score, const double2* __restrict__ tw) {
  const int nc_all = *nc_max * 7;
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * 4 + (threadIdx.x >> 5), frame = blockIdx.y;
  if (j >= nc_all || frame >= nf1) return;
  const size_t at = (size_t)frame * max_cand + j;
  const double f0c = cand[at];
  if (f0c <= 0.0) { if (lane == 0) { cand[at] = 0.0; score[at] = 0.0; } return; }
  const double pos = frame * 1.0 / 1000.0;
  const int half = (int)(1.5 * fs / f0c + 1.0);
  const double wlen_time = (2.0 * half + 1.0) / fs;
  const int blen = half * 2 + 1;
  const int fft_size = 1 << (2 + (int)(log(half * 2.0 + 1.0) / kLog2));
  const int basic_index = matlab_round((pos + (double)(-half) / fs) * fs + 0.001);
  const int nh = imin((int)(fs / 2.0 / f0c), 6);
  int index[6];
#pragma unroll
  for (int h = 0; h < 6; ++h) index[h] = imin(matlab_round(f0c * fft_size / fs * (h + 1)), fft_size / 2);
  auto mainw = [&](int i) {
    const double tmp = ((basic_index + i) - 1.0) / fs - pos;
    return 0.42 + 0.5 * cos(2.0 * kPi * tmp / wlen_time) + 0.08 * cos(4.0 * kPi * tmp / wlen_time);
  };
  double mr[6], mi[6], dr[6], di[6];
#pragma unroll
  for (int h = 0; h < 6; ++h) { mr[h] = mi[h] = dr[h] = di[h] = 0.0; }
  const int tstep = kTwiddleN / fft_size;           // table holds exp(-2 pi i k / kTwiddleN), k < kTwiddleN / 2
  for (int i = lane; i < blen; i += 32) {
    const double xv = y[imax(0, imin(y_length - 1, basic_index + i - 1))];
    const double mw = mainw(i);
    double dw;
    if (i == 0) dw = -mainw(1) / 2.0;
    else if (i == blen - 1) dw = mainw(blen - 2) / 2.0;
    else dw = -(mainw(i + 1) - mainw(i - 1)) / 2.0;
    const double a = xv * mw, b = xv * dw;
#pragma unroll
    for (int h = 0; h < 6; ++h) {
      if (h < nh) {
        int q = (int)(((long long)index[h] * i) % fft_size) * tstep;      // angle index in [0, kTwiddleN)
        double2 w;
        if (q < kTwiddleN / 2) w = __ldg(&tw[q]); else { w = __ldg(&tw[q - kTwiddleN / 2]); w.x = -w.x; w.y = -w.y; }
        mr[h] += a * w.x; mi[h] += a * w.y;
        dr[h] += b * w.x; di[h] += b * w.y;
      }
    }
  }
#pragma unroll
  for (int h = 0; h < 6; ++h) { mr[h] = warp_sum(mr[h]); mi[h] = warp_sum(mi[h]); dr[h] = warp_sum(dr[h]); di[h] = warp_sum(di[h]); }
  if (lane != 0) return;
  double numerator = 0.0, denominator = 0.0, sc = 0.0;
  for (int h = 0; h < nh; ++h) {
    const double power = mr[h] * mr[h] + mi[h] * mi[h];
    const double numer_i = mr[h] * di[h] - mi[h] * dr[h];
    const double inst = power == 0.0 ? 0.0 : (double)index[h] * fs / fft_size + numer_i / power * fs / 2.0 / kPi;
    const double amp = sqrt(power);
    numerator += amp * inst;
    denominator += amp * (h + 1.0);
    sc += fabs((inst / (h + 1.0) - f0c) / f0c);
  }
  double rf = numerator / (denominator + kSafeMin);
  double rs = 1.0 / (sc / nh + kSafeMin);
  if (rf < f0_floor || rf > f0_ceil || rs < 2.5) { rf = 0.0; rs = 0.0; }
  cand[at] = rf; score[at] = rs;
}

// SelectBestF0's error only (RemoveUnreliableCandidates needs no winner): min(allowed, min_i |ref - c_i| / ref)
__device__ inline double hv_best_error(double ref, const double* __restrict__ c, int n, double allowed) {
  double best = allowed;
  for (int i = 0; i < n; ++i) {
    const double tmp = fabs(ref - c[i]) / ref;
    if (tmp > best) continue;
    best = tmp;
  }
  return best;
}

__global__ void k_hv_remove(const double* __restrict__ tmpc, int nf1, int max_cand, const int* __restrict__ nc_max, double* __restrict__ cand,
                            double* __restrict__ score) {
  const int nc_all = *nc_max * 7;
  const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
  if (j >= nc_all || i < 1 || i >= nf1 - 1) return;
  const double ref = tmpc[(size_t)i * max_cand + j];
  if (ref == 0) return;
  const double e1 = hv_best_error(ref, tmpc + (size_t)(i + 1) * max_cand, nc_all, 1.0);
  const double e2 = hv_best_error(ref, tmpc + (size_t)(i - 1) * max_cand, nc_all, 1.0);
  if (fmin(e1, e2) <= 0.05) return;
  cand[(size_t)i * max_cand + j] = 0; score[(size_t)i * max_cand + j] = 0;
}

// ---- FixF0Contour: one warp ---------------------------------------------------------------------------------------------------
// SelectBestF0 over n candidate columns, warp-parallel, with the sequential loop's result: among the candidates whose error equals the
// minimum (and does not exceed `allowed`) the LAST one wins; 0 when none qualifies.
__device__ inline double hv_select_best_warp(double ref, const double* __restrict__ c, int n, double allowed) {
  const int lane = threadIdx.x & 31;
  double best_err = allowed; int best_idx = -1;
  for (int i = lane; i < n; i += 32) {
    const double tmp = fabs(ref - c[i]) / ref;
    if (tmp > best_err) continue;
    best_err = tmp; best_idx = i;                  // increasing i within a lane: ties keep the later index
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double oe = __shfl_xor_sync(0xffffffffu, best_err, o);
    const int oi = __shfl_xor_sync(0xffffffffu, best_idx, o);
    if (oi >= 0 && (best_idx < 0 || oe < best_err || (oe == best_err && oi > best_idx))) { best_err = oe; best_idx = oi; }
  }
  return best_idx >= 0 ? c[best_idx] : 0.0;
}

__device__ inline double hv_search_score_warp(double f0, const double* __restrict__ c, const double* __restrict__ s, int n) {
  const int lane = threadIdx.x & 31;
  double sc = 0.0;
  for (int i = lane; i < n; i += 32)
    if (f0 == c[i] && sc < s[i]) sc = s[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sc = fmax(sc, __shfl_xor_sync(0xffffffffu, sc, o));
  return sc;
}

// GetBoundaryList (lane 0); returns the number of boundaries to every lane
__device__ inline int hv_boundary_list_warp(const double* __restrict__ f0, int n, int* __restrict__ bl) {
  int nb = 0;
  if ((threadIdx.x & 31) == 0) {
    int prev = 0;
    for (int i = 1; i < n; ++i) {
      const int cur = (i == n - 1) ? 0 : (f0[i] > 0 ? 1 : 0);
      if (cur - prev != 0) { bl[nb] = i - nb % 2; nb++; }
      prev = cur;
    }
  }
  return __shfl_sync(0xffffffffu, nb, 0);
}

__device__ inline int hv_extend_warp(int origin, int last_point, int shift, const double* __restrict__ cand, int stride, int nc, double* ext) {
  const int lane = threadIdx.x & 31;
  double tmp_f0 = ext[origin];
  int shifted_origin = origin, count = 0;
  const int distance = abs(last_point - origin);
  for (int i = 0; i <= distance; ++i) {
    const int idx = origin + shift * i + shift;
    const double v = hv_select_best_warp(tmp_f0, cand + (size_t)idx * stride, nc, 0.18);
    if (lane == 0) ext[idx] = v;
    if (v == 0.0) count++;
    else { tmp_f0 = v; count = 0; shifted_origin = idx; }
    if (count == 4) break;
  }
  __syncwarp();
  return shifted_origin;
}

// work: c1[nf], c2[nf], mc[max_sections][nf];  iwork: bl[nf + 2], order / sel [max_sections], sb[2 max_sections]
__global__ void __launch_bounds__(32) k_hv_fix_contour(const double* __restrict__ cand, const double* __restrict__ score, int nf, int stride,
                                                      const int* __restrict__ nc_max, int max_sections, double* __restrict__ work,
                                                      int* __restrict__ iwork, double* __restrict__ best) {
  const int lane = threadIdx.x;
  const int nc = *nc_max * 7;
  double* c1 = work; double* c2 = work + nf; double* mc = work + 2 * (size_t)nf;
  int* bl = iwork; int* order = iwork + nf + 2; int* sel = order + max_sections; int* sb = sel + max_sections;    // sb: 2 * max_sections
  // SearchF0Base
  for (int i = lane; i < nf; i += 32) {
    double bs = 0.0, v = 0.0;
    for (int j = 0; j < nc; ++j) {
      const double s = score[(size_t)i * stride + j];
      if (s > bs) { v = cand[(size_t)i * stride + j]; bs = s; }
    }
    c1[i] = v;
  }
  __syncwarp();
  // FixStep1
  for (int i = lane; i < nf; i += 32) {
    double v = 0.0;
    if (i >= 2 && c1[i] != 0.0) {
      const double ref = c1[i - 1] * 2 - c1[i - 2];
      v = (fabs((c1[i] - ref) / ref) > 0.008 && fabs((c1[i] - c1[i - 1])) / c1[i - 1] > 0.008) ? 0.0 : c1[i];
    }
    c2[i] = v;
  }
  __syncwarp();
  // FixStep2
  for (int i = lane; i < nf; i += 32) c1[i] = c2[i];
  __syncwarp();
  int nb = hv_boundary_list_warp(c2, nf, bl);
  __syncwarp();
  for (int s = 0; s < nb / 2; ++s) {
    const int st = bl[s * 2], ed = bl[s * 2 + 1];
    if (ed - st >= 6) continue;
    for (int j = st + lane; j <= ed; j += 32) c1[j] = 0.0;
  }
  __syncwarp();
  // FixStep3
  for (int i = lane; i < nf; i += 32) c2[i] = c1[i];
  __syncwarp();
  nb = hv_boundary_list_warp(c1, nf, bl);
  __syncwarp();
  int ns = nb / 2;
  if (ns > max_sections) ns = max_sections;          // cannot happen: sections are >= 6 frames long and separated (max_sections = nf / 7 + 2)
  if (ns > 0) {
    for (int s = 0; s < ns; ++s) {                   // GetMultiChannelF0
      const int st = bl[s * 2], ed = bl[s * 2 + 1];
      for (int j = lane; j < nf; j += 32) mc[(size_t)s * nf + j] = (j >= st && j <= ed) ? c1[j] : 0.0;
    }
    __syncwarp();
    for (int s = 0; s < ns; ++s) {                   // Extend
      double* row = mc + (size_t)s * nf;
      const int ed = hv_extend_warp(bl[s * 2 + 1], imin(nf - 2, bl[s * 2 + 1] + 100), 1, cand, stride, nc, row);
      const int st = hv_extend_warp(bl[s * 2], imax(1, bl[s * 2] - 100), -1, cand, stride, nc, row);
      if (lane == 0) { bl[s * 2 + 1] = ed; bl[s * 2] = st; }
      __syncwarp();
    }
    // ExtendSub (running mean carried across sections, as in the published source).  The published code compacts the selected
    // sections to the front of its row / boundary arrays; here sel[] maps compact slot -> row and sb[] holds the compacted boundaries.
    int count = 0;
    if (lane == 0) {
      double mean_f0 = 0.0;
      for (int s = 0; s < ns; ++s) {
        const int st = bl[s * 2], ed = bl[s * 2 + 1];
        for (int j = st; j < ed; ++j) mean_f0 += mc[(size_t)s * nf + j];
        mean_f0 /= ed - st;
        if (2200.0 / mean_f0 < ed - st) { sel[count] = s; sb[count * 2] = st; sb[count * 2 + 1] = ed; count++; }
      }
      // MakeSortedOrder, literally (an insertion pass that compares against the moving entry order[i])
      for (int i = 0; i < count; ++i) order[i] = i;
      for (int i = 1; i < count; ++i)
        for (int j = i - 1; j >= 0; --j) {
          if (sb[order[j] * 2] > sb[order[i] * 2]) { const int t = order[i]; order[i] = order[j]; order[j] = t; }
          else break;
        }
    }
    count = __shfl_sync(0xffffffffu, count, 0);
    __syncwarp();
    if (count != 0) {                                // MergeF0: sb[0], sb[1] double as the running boundaries of the merged contour
      const double* r0 = mc + (size_t)sel[0] * nf;
      for (int i = lane; i < nf; i += 32) c2[i] = r0[i];
      __syncwarp();
      for (int q = 1; q < count; ++q) {
        const int o = order[q];
        const double* row = mc + (size_t)sel[o] * nf;
        const int st2 = sb[o * 2], ed2 = sb[o * 2 + 1], b0 = sb[0], b1 = sb[1];
        __syncwarp();
        int new_b0 = b0, new_b1;
        if (st2 - b1 > 0) {
          for (int j = st2 + lane; j <= ed2; j += 32) c2[j] = row[j];
          new_b0 = st2; new_b1 = ed2;
        } else if (b0 <= st2 && b1 >= ed2) {         // MergeF0Sub: the new section lies inside the merged one
          new_b1 = b1;
        } else {
          double score1 = 0.0, score2 = 0.0;
          for (int i = st2; i <= b1; ++i) {
            score1 += hv_search_score_warp(c2[i], cand + (size_t)i * stride, score + (size_t)i * stride, nc);
            score2 += hv_search_score_warp(row[i], cand + (size_t)i * stride, score + (size_t)i * stride, nc);
          }
          const int from = score1 > score2 ? b1 : st2;
          for (int j = from + lane; j <= ed2; j += 32) c2[j] = row[j];
          new_b1 = ed2;
        }
        __syncwarp();
        if (lane == 0) { sb[0] = new_b0; sb[1] = new_b1; }
        __syncwarp();
      }
    }
  }
  __syncwarp();
  // FixStep4
  for (int i = lane; i < nf; i += 32) best[i] = c2[i];
  __syncwarp();
  nb = hv_boundary_list_warp(c2, nf, bl);
  __syncwarp();
  for (int s = 0; s < nb / 2 - 1; ++s) {
    const int e0 = bl[s * 2 + 1], s1 = bl[(s + 1) * 2];
    const int distance = s1 - e0 - 1;
    if (distance >= 9) continue;
    const double tmp0 = c2[e0] + 1, tmp1 = c2[s1] - 1;
    const double coefficient = (tmp1 - tmp0) / (distance + 1.0);
    for (int j = e0 + 1 + lane; j <= s1 - 1; j += 32) best[j] = tmp0 + coefficient * (j - e0);
  }
}

// SmoothF0Contour: thread s filters voiced section s of the 300-frame padded contour; work rows: x[n], tmp[n] per section
__global__ void k_hv_smooth(const double* __restrict__ best, int nf, int max_sections, double* __restrict__ work, int* __restrict__ iwork,
                            double* __restrict__ basic) {
  const int lag = 300, n = nf + 2 * lag;
  __shared__ int s_nb;
  int* bl = iwork;
  for (int i = threadIdx.x; i < nf; i += blockDim.x) basic[i] = 0.0;
  if (threadIdx.x == 0) {
    int nb = 0, prev = 0;
    for (int i = 1; i < n; ++i) {
      const int k = i - lag;
      const int cur = (i == n - 1) ? 0 : ((k >= 0 && k < nf && best[k] > 0) ? 1 : 0);
      if (cur - prev != 0) { if (nb < 2 * max_sections) bl[nb] = i - nb % 2; nb++; }
      prev = cur;
    }
    s_nb = nb < 2 * max_sections ? nb : 2 * max_sections;
  }
  __syncthreads();
  const int ns = s_nb / 2;
  const double b0 = 0.0078202080334971724, b1 = 0.015640416066994345, a0 = 1.7347257688092754, a1 = -0.76600660094326412;
  for (int s = threadIdx.x; s < ns; s += blockDim.x) {
    const int st = bl[s * 2], ed = bl[s * 2 + 1];
    double* tmp = work + (size_t)s * n;
    const double xs = best[st - lag], xe = best[ed - lag];
    double w0 = 0.0, w1 = 0.0;
    for (int i = 0; i < n; ++i) {
      const double xv = i < st ? xs : (i > ed ? xe : best[i - lag]);
      const double wt = xv + a0 * w0 + a1 * w1;
      tmp[n - i - 1] = b0 * wt + b1 * w0 + b0 * w1;
      w1 = w0; w0 = wt;
    }
    w0 = w1 = 0.0;
    for (int i = 0; i < n; ++i) {
      const double wt = tmp[i] + a0 * w0 + a1 * w1;
      const double yv = b0 * wt + b1 * w0 + b0 * w1;
      const int pos = n - i - 1;
      if (pos >= st && pos <= ed) basic[pos - lag] = yv;
      w1 = w0; w0 = wt;
    }
  }
}

__global__ void k_hv_subsample(const double* __restrict__ basic, int nf1, double frame_period, int f0_length, double* __restrict__ f0) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= f0_length) return;
  const double t = i * frame_period / 1000.0;
  f0[i] = basic[imin(nf1 - 1, matlab_round(t * 1000.0))];
}

// ---- host side -----------------------------------------------------------------------------------------------------------------
void harvest_plan_free(HarvestPlan* p) {
  if (!p) return;
  if (p->fwd) cufftDestroy(p->fwd);
  if (p->inv) cufftDestroy(p->inv);
  void* ptrs[] = {p->d_t1, p->d_t2, p->d_y, p->d_Y, p->d_F, p->d_Z, p->d_filtered, p->d_flh, p->d_boundary, p->d_edges, p->d_loc, p->d_itv,
                  p->d_counts, p->d_raw, p->d_cand, p->d_score, p->d_tmpc, p->d_nc, p->d_best, p->d_basic, p->d_work, p->d_iwork};
  for (void* q : ptrs) if (q) cudaFree(q);
  delete p;
}

int harvest_plan_create(Engine* e, int n, int fs, double frame_period, double f0_floor, double f0_ceil, HarvestPlan** out) {
  HarvestPlan* p = new HarvestPlan();
  p->n = n; p->fs = fs; p->frame_period = frame_period; p->f0_floor = f0_floor; p->f0_ceil = f0_ceil;
  p->ratio = matlab_round(fs / 8000.0);
  RYK_CHECK(p->ratio >= 1 && p->ratio <= 12, "Harvest: sampling rate outside the decimation table (8 kHz .. 96 kHz)");
  const double lo = f0_floor * 0.9, hi = f0_ceil * 1.1;
  p->channels = 1 + (int)(log(hi / lo) / kLog2 * 40.0);
  p->actual_fs = (double)fs / p->ratio;
  std::vector<double> boundary(p->channels);
  std::vector<int> flh(p->channels);
  for (int i = 0; i < p->channels; ++i) {
    boundary[i] = lo * pow(2.0, (i + 1) / 40.0);
    flh[i] = matlab_round(p->actual_fs / boundary[i] * 2.0);
  }
  p->y_length = (int)ceil((double)n / p->ratio);
  p->fft_size = suitable_fft_size(p->y_length + 5 + 2 * (int)(2.0 * p->actual_fs / boundary[0]));
  p->nf1 = (int)(1000.0 * n / fs / 1.0) + 1;
  p->f0_length = (int)(1000.0 * n / fs / frame_period) + 1;
  p->max_cand = matlab_round(p->channels / 10.0) * 7;
  p->lag = (int)(ceil(140.0 / p->ratio) * p->ratio);
  p->n_pad = n + 2 * p->lag + 18;
  p->max_sections = p->nf1 / 7 + 2;
  { const int half = (int)(1.5 * p->actual_fs / f0_floor + 1.0);
    RYK_CHECK((1 << (2 + (int)(log(half * 2.0 + 1.0) / kLog2))) <= kTwiddleN, "Harvest: refinement window exceeds the twiddle table"); }
  const int nbins = p->fft_size / 2 + 1;
  const size_t ev = (size_t)p->channels * 4 * p->y_length, nsm = (size_t)(p->nf1 + 600);
  RYK_CUDA(cudaMalloc(&p->d_t1, sizeof(double) * p->n_pad));
  RYK_CUDA(cudaMalloc(&p->d_t2, sizeof(double) * p->n_pad));
  RYK_CUDA(cudaMalloc(&p->d_y, sizeof(double) * p->fft_size));
  RYK_CUDA(cudaMalloc(&p->d_Y, sizeof(cufftDoubleComplex) * nbins));
  RYK_CUDA(cudaMalloc(&p->d_F, sizeof(cufftDoubleComplex) * nbins * p->channels));
  RYK_CUDA(cudaMalloc(&p->d_Z, sizeof(cufftDoubleComplex) * nbins * p->channels));
  RYK_CUDA(cudaMalloc(&p->d_filtered, sizeof(double) * (size_t)p->fft_size * p->channels));
  RYK_CUDA(cudaMalloc(&p->d_flh, sizeof(int) * p->channels));
  RYK_CUDA(cudaMalloc(&p->d_boundary, sizeof(double) * p->channels));
  RYK_CUDA(cudaMalloc(&p->d_edges, sizeof(int) * ev));
  RYK_CUDA(cudaMalloc(&p->d_loc, sizeof(double) * ev));
  RYK_CUDA(cudaMalloc(&p->d_itv, sizeof(double) * ev));
  RYK_CUDA(cudaMalloc(&p->d_counts, sizeof(int) * p->channels * 4));
  RYK_CUDA(cudaMalloc(&p->d_raw, sizeof(double) * (size_t)p->channels * p->nf1));
  RYK_CUDA(cudaMalloc(&p->d_cand, sizeof(double) * (size_t)p->nf1 * p->max_cand));
  RYK_CUDA(cudaMalloc(&p->d_score, sizeof(double) * (size_t)p->nf1 * p->max_cand));
  RYK_CUDA(cudaMalloc(&p->d_tmpc, sizeof(double) * (size_t)p->nf1 * p->max_cand));
  RYK_CUDA(cudaMalloc(&p->d_nc, sizeof(int)));
  RYK_CUDA(cudaMalloc(&p->d_best, sizeof(double) * p->nf1));
  RYK_CUDA(cudaMalloc(&p->d_basic, sizeof(double) * p->nf1));
  const size_t work = std::max((size_t)(2 + p->max_sections) * p->nf1, (size_t)p->max_sections * nsm);
  RYK_CUDA(cudaMalloc(&p->d_work, sizeof(double) * work));
  RYK_CUDA(cudaMalloc(&p->d_iwork, sizeof(int) * (p->nf1 + 600 + 8 * p->max_sections + 16)));
  RYK_CUDA(cudaMemcpyAsync(p->d_flh, flh.data(), sizeof(int) * p->channels, cudaMemcpyHostToDevice, e->stream));
  RYK_CUDA(cudaMemcpyAsync(p->d_boundary, boundary.data(), sizeof(double) * p->channels, cudaMemcpyHostToDevice, e->stream));
  if (cufft_ok(cufftPlan1d(&p->fwd, p->fft_size, CUFFT_D2Z, 1), "plan D2Z")) return -1;
  if (cufft_ok(cufftPlan1d(&p->inv, p->fft_size, CUFFT_Z2D, p->channels), "plan Z2D")) return -1;
  cufftHandle filt = 0;
  if (cufft_ok(cufftPlan1d(&filt, p->fft_size, CUFFT_D2Z, p->channels), "plan D2Z filters")) return -1;
  if (cufft_ok(cufftSetStream(filt, e->stream), "set stream")) return -1;
  k_hv_design_filters<<<p->channels, 256, 0, e->stream>>>(p->d_filtered, p->fft_size, p->d_flh, p->d_boundary, p->actual_fs);
  if (cufft_ok(cufftExecD2Z(filt, p->d_filtered, p->d_F), "exec filters")) return -1;
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  RYK_CUDA(cudaGetLastError());
  cufftDestroy(filt);
  *out = p;
  return 0;
}

// Harvest: x (device float32, p->n samples) -> d_f0 (double, p->f0_length frames at frame_period).  Stream-ordered, no host sync.
int harvest_run(Engine* e, HarvestPlan* p, const float* d_x, double* d_f0, cudaStream_t st) {
  const int nbins = p->fft_size / 2 + 1;
  if (cufft_ok(cufftSetStream(p->fwd, st), "set stream")) return -1;
  if (cufft_ok(cufftSetStream(p->inv, st), "set stream")) return -1;
  k_hv_decimate<<<1, 512, 0, st>>>(d_x, p->n, p->ratio, p->lag, p->y_length, p->fft_size, p->d_t1, p->d_t2, p->d_y);
  if (cufft_ok(cufftExecD2Z(p->fwd, p->d_y, p->d_Y), "exec D2Z")) return -1;
  k_band_mul<<<dim3((nbins + 255) / 256, p->channels), 256, 0, st>>>(p->d_Y, p->d_F, p->d_Z, nbins);
  if (cufft_ok(cufftExecZ2D(p->inv, p->d_Z, p->d_filtered), "exec Z2D")) return -1;
  k_dio_zero_cross<<<dim3(4, p->channels), 1024, 0, st>>>(p->d_filtered, p->fft_size, p->y_length, p->d_flh, 1, 1, p->actual_fs, p->d_edges,
                                                        p->d_loc, p->d_itv, p->d_counts);
  k_hv_raw_candidates<<<dim3((p->nf1 + 127) / 128, p->channels), 128, 0, st>>>(p->d_loc, p->d_itv, p->d_counts, p->y_length, p->nf1, p->f0_floor,
                                                                              p->f0_ceil, p->d_boundary, p->d_raw);
  RYK_CUDA(cudaMemsetAsync(p->d_nc, 0, sizeof(int), st));
  k_hv_detect<<<(p->nf1 + 63) / 64, 64, 0, st>>>(p->d_raw, p->channels, p->nf1, p->max_cand, p->d_cand, p->d_score, p->d_nc);
  k_hv_overlap<<<(p->nf1 + 63) / 64, 64, 0, st>>>(p->d_cand, p->nf1, p->max_cand, p->d_nc);
  k_hv_refine<<<dim3((p->max_cand + 3) / 4, p->nf1), 128, 0, st>>>(p->d_y, p->y_length, p->actual_fs, p->nf1, p->max_cand, p->d_nc, p->f0_floor,
                                                                  p->f0_ceil, p->d_cand, p->d_score, e->d_twiddle);
  RYK_CUDA(cudaMemcpyAsync(p->d_tmpc, p->d_cand, sizeof(double) * (size_t)p->nf1 * p->max_cand, cudaMemcpyDeviceToDevice, st));
  k_hv_remove<<<dim3((p->max_cand + 63) / 64, p->nf1), 64, 0, st>>>(p->d_tmpc, p->nf1, p->max_cand, p->d_nc, p->d_cand, p->d_score);
  k_hv_fix_contour<<<1, 32, 0, st>>>(p->d_cand, p->d_score, p->nf1, p->max_cand, p->d_nc, p->max_sections, p->d_work, p->d_iwork, p->d_best);
  k_hv_smooth<<<1, 64, 0, st>>>(p->d_best, p->nf1, p->max_sections, p->d_work, p->d_iwork, p->d_basic);
  k_hv_subsample<<<(p->f0_length + 127) / 128, 128, 0, st>>>(p->d_basic, p->nf1, p->frame_period, p->f0_length, d_f0);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

int harvest_plan_frames(HarvestPlan* p) { return p->f0_length; }

// Intermediate arrays for the stage-by-stage parity test (host buffers sized by the caller from the plan's geometry; any may be null).
int harvest_plan_debug_copy(HarvestPlan* p, int* info, double* y, double* raw, double* cand, double* score, double* best, double* basic,
                            cudaStream_t st) {
  int nc = 0;
  RYK_CUDA(cudaMemcpyAsync(&nc, p->d_nc, sizeof(int), cudaMemcpyDeviceToHost, st));
  if (y) RYK_CUDA(cudaMemcpyAsync(y, p->d_y, sizeof(double) * p->y_length, cudaMemcpyDeviceToHost, st));
  if (raw) RYK_CUDA(cudaMemcpyAsync(raw, p->d_raw, sizeof(double) * (size_t)p->channels * p->nf1, cudaMemcpyDeviceToHost, st));
  if (cand) RYK_CUDA(cudaMemcpyAsync(cand, p->d_cand, sizeof(double) * (size_t)p->nf1 * p->max_cand, cudaMemcpyDeviceToHost, st));
  if (score) RYK_CUDA(cudaMemcpyAsync(score, p->d_score, sizeof(double) * (size_t)p->nf1 * p->max_cand, cudaMemcpyDeviceToHost, st));
  if (best) RYK_CUDA(cudaMemcpyAsync(best, p->d_best, sizeof(double) * p->nf1, cudaMemcpyDeviceToHost, st));
  if (basic) RYK_CUDA(cudaMemcpyAsync(basic, p->d_basic, sizeof(double) * p->nf1, cudaMemcpyDeviceToHost, st));
  RYK_CUDA(cudaStreamSynchronize(st));
  if (info) { info[0] = p->channels; info[1] = p->nf1; info[2] = p->y_length; info[3] = p->fft_size; info[4] = p->max_cand; info[5] = p->ratio; info[6] = nc * 7; }
  return 0;
}

}  // namespace ryk
