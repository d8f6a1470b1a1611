// features.cu -- the small feature-domain kernels between the big stages (SURVEY rows a9-a13):
//   * SPTK mel-cepstrum conversions as precomputed linear maps (E):  mc = G log(sp),  log(sp) = H mc
//     (freqt is a linear time-invariant recursion, so sp2mc / mc2sp collapse to one small matrix each;
//      the matrices are built on the host with the same recursion SPTK runs)
//   * librosa-style silence gate: centred frame mean-square -> dB vs the loudest frame -> mask -> compaction (F)
//   * stage-1 prologue/epilogue: gather effective frames, normalise, 'minimum' pad; denormalise, scatter into
//     the silent template, log-f0 linear conversion (G)
//   * stage-2 prologue/epilogue: 'minimum' pad + log + drop Nyquist bin; edge-pad + exp + unpad (a13)
#include <math.h>
#include <vector>

#include "engine.h"
#include "features.h"

namespace ryk {

// ------------------------------------------------------------------------------------ SPTK matrices (host)
static void freqt_host(const double* c1, int m1, double* c2, int m2, double a) {
  double b = 1 - a * a;
  std::vector<double> d(m2 + 1, 0.0), g(m2 + 1, 0.0);
  for (int i = -m1; i <= 0; i++) {
    if (0 <= m2) { d[0] = g[0]; g[0] = c1[-i] + a * d[0]; }
    if (1 <= m2) { d[1] = g[1]; g[1] = b * d[0] + a * d[1]; }
    for (int j = 2; j <= m2; j++) { d[j] = g[j]; g[j] = d[j - 1] + a * (d[j] - g[j - 1]); }
  }
  for (int j = 0; j <= m2; ++j) c2[j] = g[j];
}

int sptk_prepare(Engine* e, int order, double alpha, int fft_size, SptkMats* out) {
  const auto key = std::make_tuple(order, alpha, fft_size);
  auto it = e->sptk.find(key);
  if (it != e->sptk.end()) { *out = it->second; return 0; }
  const int nb = fft_size / 2 + 1, N = fft_size;
  // G: mc = freqt(irfft(logsp) with c[0] /= 2, order, alpha); column k = response to the unit log-spectrum e_k
  std::vector<double> G((size_t)(order + 1) * nb), H((size_t)nb * (order + 1));
  std::vector<double> c(N), mc(order + 1);
  for (int k = 0; k < nb; ++k) {
    double wk = (k == 0 || k == N / 2) ? 1.0 : 2.0;
    for (int n = 0; n < N; ++n) c[n] = wk * cos(2.0 * kPi * (double)k * (double)n / N) / N;
    c[0] /= 2.0;
    freqt_host(c.data(), N - 1, mc.data(), order, alpha);
    for (int j = 0; j <= order; ++j) G[(size_t)j * nb + k] = mc[j];
  }
  // H: logsp = real(rfft(sym(freqt(mc, N/2, -alpha) with c[0] *= 2))); column j = response to unit mc e_j
  std::vector<double> ej(order + 1), cc(nb);
  for (int j = 0; j <= order; ++j) {
    for (int i = 0; i <= order; ++i) ej[i] = i == j ? 1.0 : 0.0;
    freqt_host(ej.data(), order, cc.data(), N / 2, -alpha);
    cc[0] *= 2.0;
    for (int k = 0; k < nb; ++k) {
      double s = cc[0];
      for (int i = 1; i < N / 2; ++i) s += 2.0 * cc[i] * cos(2.0 * kPi * (double)i * (double)k / N);
      s += cc[N / 2] * cos(kPi * (double)k);
      H[(size_t)k * (order + 1) + j] = s;
    }
  }
  SptkMats m;
  cudaError_t err = cudaMalloc(&m.d_G, G.size() * sizeof(double));
  if (err == cudaSuccess) err = cudaMalloc(&m.d_H, H.size() * sizeof(double));
  if (err == cudaSuccess) err = cudaMemcpy(m.d_G, G.data(), G.size() * sizeof(double), cudaMemcpyHostToDevice);
  if (err == cudaSuccess) err = cudaMemcpy(m.d_H, H.data(), H.size() * sizeof(double), cudaMemcpyHostToDevice);
  if (err != cudaSuccess) {          // the entry was never handed out: nothing else holds these addresses
    cudaFree(m.d_G);
    cudaFree(m.d_H);
    RYK_CUDA(err);
  }
  e->sptk[key] = m;
  *out = m;
  return 0;
}

// sp = exp(H mc) + add  (voice_changer.py:38-39); float32 mc in (pysptk casts to f32), FP64 math.
__global__ void k_mc2sp(const float* __restrict__ mc, int T, int order, int nb, const double* __restrict__ H, double add,
                        float* __restrict__ sp32, double* __restrict__ sp64) {
  int t = blockIdx.y;
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T || k >= nb) return;
  double s = 0.0;
  for (int j = 0; j <= order; ++j) s += H[(size_t)k * (order + 1) + j] * (double)mc[(size_t)t * (order + 1) + j];
  double v = exp(s) + add;
  if (sp32) sp32[(size_t)t * nb + k] = (float)v;
  if (sp64) sp64[(size_t)t * nb + k] = v;
}

int mc2sp_run(Engine* e, const double* d_H, const float* d_mc, int T, int order, int fft_size, double add, float* d_sp32, double* d_sp64,
              cudaStream_t st) {
  if (T <= 0) return 0;
  int nb = fft_size / 2 + 1;
  k_mc2sp<<<dim3((nb + 127) / 128, T), 128, 0, st>>>(d_mc, T, order, nb, d_H, add, d_sp32, d_sp64);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------ silence gate
// mse[f] = mean over frame_length samples of x^2, frame centred at f*hop, reflect padding (librosa.feature.rms, center=True)
__global__ void k_frame_mse(const float* __restrict__ x, int n, int frame_length, int hop, int n_frames, double* __restrict__ mse) {
  __shared__ double scratch[32];
  int f = blockIdx.x;
  if (f >= n_frames) return;
  int pad = frame_length / 2;
  double acc = 0.0;
  for (int j = threadIdx.x; j < frame_length; j += blockDim.x) {
    int idx = f * hop + j - pad;
    if (idx < 0) idx = -idx;
    if (idx >= n) idx = 2 * (n - 1) - idx;
    if (idx < 0) idx = 0;
    if (idx >= n) idx = n - 1;
    double v = n > 0 ? (double)x[idx] : 0.0;
    acc += v * v;
  }
  double s = block_sum(acc, scratch);
  if (threadIdx.x == 0) mse[f] = s / frame_length;
}

// single CTA: reference power = max mse; mask; ordered compaction of effective frame ids.
// threshold_db < 0 means "no gate" (every frame effective).  count[0] = T_eff, count[1] = padded length (T_eff + 128 - T_eff % 128, 0 if empty)
__global__ void __launch_bounds__(1024) k_gate(const double* __restrict__ mse, int n_frames, double threshold_db,
                                              uint8_t* __restrict__ mask, int* __restrict__ index, int* __restrict__ count) {
  __shared__ double smax[32];
  __shared__ int wsum[32];
  __shared__ int total;
  double m = 0.0;
  for (int i = threadIdx.x; i < n_frames; i += blockDim.x) m = fmax(m, mse[i]);
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) smax[w] = m;
  __syncthreads();
  if (w == 0) {
    double v = lane < (blockDim.x >> 5) ? smax[lane] : 0.0;
    for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (lane == 0) smax[0] = v;
  }
  __syncthreads();
  const double ref_db = 10.0 * log10(fmax(1e-10, smax[0]));
  int per = (n_frames + blockDim.x - 1) / blockDim.x;
  int lo = threadIdx.x * per, hi = min(lo + per, n_frames);
  int cnt = 0;
  for (int i = lo; i < hi; ++i) {
    bool eff = threshold_db < 0 ? true : (10.0 * log10(fmax(1e-10, mse[i])) - ref_db > -threshold_db);
    mask[i] = eff ? 1 : 0;
    cnt += eff ? 1 : 0;
  }
  int inc = cnt;
  for (int o = 1; o < 32; o <<= 1) { int v = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += v; }
  if (lane == 31) wsum[w] = inc;
  __syncthreads();
  if (w == 0) {
    int v = wsum[lane], iv = v;
    for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, iv, o); if (lane >= o) iv += u; }
    wsum[lane] = iv - v;
    if (lane == 31) total = iv;
  }
  __syncthreads();
  int pos = wsum[w] + inc - cnt;
  for (int i = lo; i < hi; ++i) if (mask[i]) index[pos++] = i;
  if (threadIdx.x == 0) { count[0] = total; count[1] = total > 0 ? total + (128 - total % 128) : 0; }
}

int gate_mask_run(Engine* e, const float* d_wave, int n, int frame_length, int hop, double threshold_db, int n_frames,
                  double* d_mse, uint8_t* d_mask, int* d_index, int* d_count, cudaStream_t st) {
  if (n_frames <= 0) return 0;
  k_frame_mse<<<n_frames, 256, 0, st>>>(d_wave, n, frame_length, hop, n_frames, d_mse);
  k_gate<<<1, 1024, 0, st>>>(d_mse, n_frames, threshold_db, d_mask, d_index, d_count);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------ stage-1 prologue / epilogue
// x[t][c] = (mc[index[t]][c] - mean[c]) / std[c] for t < T_eff; rows T_eff..Tp-1 = per-channel minimum over t < T_eff.
// single CTA, C channels (<= 32). Tp is read from count[1]; index == nullptr means identity (T_eff = count[0]).
__global__ void __launch_bounds__(256) k_stage1_prologue(const float* __restrict__ mc, const int* __restrict__ index, const int* __restrict__ count,
                                                        int C, const float* __restrict__ mean, const float* __restrict__ std_,
                                                        float* __restrict__ x, int Tp_capacity) {
  __shared__ float cmin[32];
  const int T = count[0], Tp = min(count[1], Tp_capacity);
  if (threadIdx.x < 32) cmin[threadIdx.x] = INFINITY;
  __syncthreads();
  // normalise + gather
  for (int i = threadIdx.x; i < T * C; i += blockDim.x) {
    int t = i / C, c = i % C;
    int src = index ? index[t] : t;
    x[i] = __fdiv_rn(__fsub_rn(mc[(size_t)src * C + c], mean[c]), std_[c]);
  }
  __syncthreads();
  if (threadIdx.x < C) {
    float m = INFINITY;
    for (int t = 0; t < T; ++t) m = fminf(m, x[(size_t)t * C + threadIdx.x]);
    cmin[threadIdx.x] = m;
  }
  __syncthreads();
  for (int i = T * C + threadIdx.x; i < Tp * C; i += blockDim.x) x[i] = cmin[i % C];
}

// scatter converted rows back + silent template + f0 conversion (yukarin AcousticConverter.convert / combine_silent)
__global__ void k_stage1_epilogue(const float* __restrict__ y /*[Tp][C] network output*/, const int* __restrict__ index,
                                  const uint8_t* __restrict__ mask, const int* __restrict__ count, int T, int C,
                                  const float* __restrict__ mean, const float* __restrict__ std_,
                                  const float* __restrict__ f0_in, const float* __restrict__ ap_in, const uint8_t* __restrict__ voiced_in,
                                  int nb, F0Map voice_map, const F0Map* __restrict__ session_map, float silent_mc0,
                                  float* __restrict__ mc_out, float* __restrict__ f0_out, float* __restrict__ ap_out,
                                  uint8_t* __restrict__ voiced_out, double* __restrict__ formant_out) {
  int t = blockIdx.x;
  // the step's formant ratio goes with its hand-off slot: the stage-2 epilogue of this step reads it there, on another stream, after
  // the host may already have staged the block of a later step (DESIGN.md §4a)
  if (formant_out && t == 0 && threadIdx.x == 0) *formant_out = session_map->formant;
  if (t >= T) return;
  const bool eff = mask[t] != 0;
  // rank of t among effective frames = position in index[] (binary search; index is ascending)
  int rank = -1;
  if (eff) {
    int lo = 0, hi = count[0];
    while (lo < hi) { int mid = (lo + hi) >> 1; if (index[mid] < t) lo = mid + 1; else hi = mid; }
    rank = lo;
  }
  for (int c = threadIdx.x; c < C; c += blockDim.x)
    mc_out[(size_t)t * C + c] = eff ? __fadd_rn(__fmul_rn(y[(size_t)rank * C + c], std_[c]), mean[c]) : (c == 0 ? silent_mc0 : 0.f);
  for (int k = threadIdx.x; k < nb; k += blockDim.x) ap_out[(size_t)t * nb + k] = eff ? ap_in[(size_t)t * nb + k] : 0.f;
  if (threadIdx.x == 0) {
    bool v = eff && voiced_in[t] != 0;
    float f = 0.f;
    if (v) {
      float fi = f0_in[t];
      // a session's map lives in device memory (it changes between steps without a new capture); the per-op calls pass the voice's
      double mu_i = voice_map.mu_in, sd_i = voice_map.sd_in, mu_t = voice_map.mu_tgt, sd_t = voice_map.sd_tgt;
      int has_f0_stats = voice_map.has_stats;
      if (session_map) {
        mu_i = session_map->mu_in; sd_i = session_map->sd_in; mu_t = session_map->mu_tgt; sd_t = session_map->sd_tgt;
        has_f0_stats = session_map->has_stats;
      }
      if (has_f0_stats) {
        // F0Converter: exp((ln f0 - mu_i) / sd_i * sd_t + mu_t); DECIDE: evaluated in float64, rounded to float32
        f = (float)exp((log((double)fi) - mu_i) / sd_i * sd_t + mu_t);
      } else f = fi;
    }
    f0_out[t] = f;
    voiced_out[t] = v ? 1 : 0;
  }
}

// ------------------------------------------------------------------------------------ stage-2 prologue / epilogue
// x[t][k] = log(sp_pad[t][k]) for k < nb-1, where rows t >= T repeat the per-bin minimum over t < T
// ('minimum' padding of become_yukarin's convert).  Pass 1: per-bin minimum (one thread per bin strip, coalesced
// across bins); pass 2: one thread per output element.
__global__ void k_sr_colmin(const float* __restrict__ sp, int T, int nb, int rows_per_block, float* __restrict__ partial) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= nb - 1) return;
  int t0 = blockIdx.y * rows_per_block, t1 = min(T, t0 + rows_per_block);
  float m = INFINITY;
  for (int t = t0; t < t1; ++t) m = fminf(m, sp[(size_t)t * nb + k]);
  partial[(size_t)blockIdx.y * (nb - 1) + k] = m;
}
__global__ void k_sr_prologue(const float* __restrict__ sp, const float* __restrict__ partial, int nparts, int T, int Tp, int nb,
                              float* __restrict__ x) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  int t = blockIdx.y;
  if (k >= nb - 1 || t >= Tp) return;
  float v;
  if (t < T) v = sp[(size_t)t * nb + k];
  else { v = INFINITY; for (int q = 0; q < nparts; ++q) v = fminf(v, partial[(size_t)q * (nb - 1) + k]); }
  x[(size_t)t * (nb - 1) + k] = logf(v);
}

// sp_out[t][k] = exp(L[k]) with the edge-padded log row L[j] = y[t][min(j, nb - 2)].  Formant ratio r != 1 (DECIDE F1): sp'(f) = sp(f / r),
// i.e. bin k reads L at x = k / r, linearly interpolated in FP64 and rounded to FP32 before expf (numpy.interp(k / r, arange(nb), L)),
// and held at L[nb - 1] from x >= nb - 1 on.  r == 1 keeps the plain expression, so an unwarped envelope is bitwise what it was.
__global__ void k_sr_epilogue(const float* __restrict__ y, int T, int nb, int t0, double formant, const double* __restrict__ d_formant,
                              float* __restrict__ sp_out) {
  int t = t0 + blockIdx.y;
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T || k >= nb) return;
  const float* row = y + (size_t)t * (nb - 1);
  const double r = d_formant ? *d_formant : formant;
  float v;
  if (r == 1.0) {
    v = row[k < nb - 1 ? k : nb - 2];
  } else {
    const double x = (double)k / r;
    if (x >= (double)(nb - 1)) {
      v = row[nb - 2];
    } else {
      const int i = (int)x;                        // x >= 0: floor
      const double w = x - (double)i;
      v = (float)((1.0 - w) * (double)row[min(i, nb - 2)] + w * (double)row[min(i + 1, nb - 2)]);
    }
  }
  sp_out[(size_t)t * nb + k] = expf(v);
}

int stage1_prologue_run(const Voice* v, const float* d_mc, const int* d_index, const int* d_count, int C, float* d_x, int Tp_capacity, cudaStream_t st) {
  k_stage1_prologue<<<1, 256, 0, st>>>(d_mc, d_index, d_count, C, v->d_s1_in_mean, v->d_s1_in_std, d_x, Tp_capacity);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

F0Map voice_f0_map(const Voice* v) {
  F0Map m = {};
  m.mu_in = v->f0_in_mean; m.sd_in = v->f0_in_std; m.mu_tgt = v->f0_tgt_mean; m.sd_tgt = v->f0_tgt_std;
  m.has_stats = v->has_f0_stats ? 1 : 0;
  return m;
}

int stage1_epilogue_run(const Voice* v, const float* d_y, const int* d_index, const uint8_t* d_mask, const int* d_count, int T, int C,
                        const float* d_f0_in, const float* d_ap_in, const uint8_t* d_voiced_in, int nb, float silent_mc0,
                        float* d_mc_out, float* d_f0_out, float* d_ap_out, uint8_t* d_voiced_out, const F0Map* d_map, cudaStream_t st,
                        double* d_formant_out) {
  if (T <= 0) return 0;
  RYK_CHECK(d_map || !d_formant_out, "the formant ratio comes from a session's map");
  k_stage1_epilogue<<<T, 128, 0, st>>>(d_y, d_index, d_mask, d_count, T, C, v->d_s1_out_mean, v->d_s1_out_std, d_f0_in, d_ap_in,
                                       d_voiced_in, nb, voice_f0_map(v), d_map, silent_mc0, d_mc_out, d_f0_out, d_ap_out, d_voiced_out,
                                       d_formant_out);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------ speaker statistics of ln f0
// (count, mean, M2) of two disjoint sets -> of their union (Chan et al.): no sum of squares, so no cancellation at large counts
__device__ __forceinline__ void f0_stats_merge(long long& n, double& mean, double& m2, long long nb, double mean_b, double m2_b) {
  if (nb == 0) return;
  if (n == 0) { n = nb; mean = mean_b; m2 = m2_b; return; }
  const long long nn = n + nb;
  const double d = mean_b - mean;
  mean += d * ((double)nb / (double)nn);
  m2 += m2_b + d * d * ((double)n * (double)nb / (double)nn);
  n = nn;
}

// One CTA: the voiced frames of the chunk's n frames are folded into (count, mean, M2) of ln f0 in a fixed order -- thread i takes
// frames i, i + 256, ... one by one, then a pairwise tree over the 256 partial triples -- and thread 0 merges the chunk into the
// running triple.  No atomics: the result depends on the frames alone.  Follow mode: once min_voiced frames are counted the measured
// mean and max(sqrt(M2 / count), sd_floor) become the input side of the session's f0 map, which the stage-1 epilogue of this step reads
// next on the same stream.
constexpr int kF0MeasureThreads = 256;
__global__ void __launch_bounds__(kF0MeasureThreads) k_f0_measure(const float* __restrict__ f0, const uint8_t* __restrict__ voiced, int n,
                                                                 F0Stats* __restrict__ stats, F0Map* __restrict__ map) {
  __shared__ long long s_n[kF0MeasureThreads];
  __shared__ double s_mean[kF0MeasureThreads], s_m2[kF0MeasureThreads];
  const int tid = threadIdx.x;
  long long cn = 0; double mean = 0.0, m2 = 0.0;
#pragma unroll 1                   // a chunk is rarely longer than one pass; unrolled, the FP64 log and division bodies spill
  for (int i = tid; i < n; i += kF0MeasureThreads) {
    const float f = f0[i];
    if (voiced[i] != 0 && f > 0.f) {
      const double x = log((double)f);
      const double d = x - mean;
      ++cn;
      mean += d / (double)cn;
      m2 += d * (x - mean);
    }
  }
  s_n[tid] = cn; s_mean[tid] = mean; s_m2[tid] = m2;
  __syncthreads();
  for (int s = kF0MeasureThreads / 2; s > 0; s >>= 1) {
    if (tid < s) {
      f0_stats_merge(cn, mean, m2, s_n[tid + s], s_mean[tid + s], s_m2[tid + s]);
      s_n[tid] = cn; s_mean[tid] = mean; s_m2[tid] = m2;
    }
    __syncthreads();
  }
  if (tid == 0) {
    long long rn = stats->n; double rmean = stats->mean, rm2 = stats->m2;
    f0_stats_merge(rn, rmean, rm2, cn, mean, m2);
    stats->n = rn; stats->mean = rmean; stats->m2 = rm2;
    if (map->follow && rn >= (long long)map->min_voiced) {
      map->mu_in = rmean;
      map->sd_in = fmax(sqrt(rm2 / (double)rn), map->sd_floor);
    }
  }
}

int f0_measure_run(const float* d_f0, const uint8_t* d_voiced, int n, F0Stats* d_stats, F0Map* d_map, cudaStream_t st) {
  k_f0_measure<<<1, kF0MeasureThreads, 0, st>>>(d_f0, d_voiced, n, d_stats, d_map);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

int sr_prologue_run(Engine* e, const float* d_sp, int T, int Tp, int nb, float* d_x, cudaStream_t st, float* d_colmin) {
  const int rows_per_block = 32, nparts = (T + rows_per_block - 1) / rows_per_block;
  RYK_CHECK((size_t)nparts * (nb - 1) * sizeof(float) <= sizeof(float) * kColminFloats, "window too long for the column-minimum scratch");
  if (!d_colmin) d_colmin = e->d_colmin;     // per-op API: the engine's scratch (calls are serialised on the engine stream)
  k_sr_colmin<<<dim3((nb - 1 + 127) / 128, nparts), 128, 0, st>>>(d_sp, T, nb, rows_per_block, d_colmin);
  k_sr_prologue<<<dim3((nb - 1 + 127) / 128, Tp), 128, 0, st>>>(d_sp, d_colmin, nparts, T, Tp, nb, d_x);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

int sr_epilogue_run(Engine* e, const float* d_y, int T, int nb, float* d_sp_out, cudaStream_t st, int t0, int t1, double formant,
                    const double* d_formant) {
  if (t1 < 0) t1 = T;
  RYK_CHECK(0 <= t0 && t0 <= t1 && t1 <= T, "stage-2 epilogue rows out of range");
  if (t1 == t0) return 0;
  k_sr_epilogue<<<dim3((nb + 127) / 128, t1 - t0), 128, 0, st>>>(d_y, T, nb, t0, formant, d_formant, d_sp_out);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------ polyphase resampler
// SURVEY 8(f) rank 3 (check.py:80 librosa.load(..., sr=input_rate)): scipy.signal.resample_poly's upfirdn step on the device.
//   y[i] = sum over j of x[j] * h[(i + n_pre_remove) * down - j * up - n_pre_pad] = sum over j of x[j] * h[half_len + i * down - j * up],
//   0 <= tap index < n_taps, x zero outside [0, in_end)
// One thread per output sample, FP64 accumulation over the ~n_taps / up taps that hit an input sample (ascending j).  i and j are
// global indices of the whole signal, so the whole-signal call and the two streaming sides of a session sum the same terms in the
// same order: streamed output is bitwise the whole-signal output.
//   whole:      x = the whole signal (x_len samples), outputs 0 .. n_out-1.
//   stream in:  a fixed chunk of `chunk` samples per step; x = the history window ending at the newest sample (x_len samples, slid by
//               the caller).  Outputs out_end - delay .. + n_out - 1 of the resampled signal; those with a negative index are the
//               leading zeros of the delay.
//   stream out: *n_new new samples per step in x_new; x = the x_len samples before them (the kept history).  Emits the outputs not
//               yet emitted whose filter support ends inside the samples received so far (at most n_out of them), writes their count
//               to *n_out_dev and the history for the next step to hist_next.
// Streaming positions are read from *st and the next step's written to *st_next (double-buffered by the caller), so no host value
// changes from step to step and the launch can sit in a captured graph.
template <typename Tin, typename Tout>
__global__ void __launch_bounds__(256) k_resample_poly(PolyArgs<Tin, Tout> a) {
  const int half_len = (a.n_taps - 1) / 2;
  long long in_end, x_first, new_first, out_first;
  int n_out = a.n_out;
  if (a.mode == kPolyWhole) {
    in_end = a.x_len; x_first = 0; new_first = in_end; out_first = 0;
  } else {
    const ResampleState s = *a.st;
    if (a.mode == kPolyStreamIn) {
      in_end = s.in_end + a.chunk; x_first = in_end - a.x_len; new_first = in_end; out_first = s.out_end - a.delay;
    } else {
      const int n_new = *a.n_new > 0 ? *a.n_new : 0;
      in_end = s.in_end + n_new; x_first = s.in_end - a.x_len; new_first = s.in_end; out_first = s.out_end;
      // outputs 0 .. m-1 have their whole support in [0, in_end): half_len + i * down - j * up <= n_taps - 1 for j = in_end - 1
      const long long num = in_end * a.up - 1 - half_len;
      const long long m = (num >= 0 ? num / a.down : -((-num + a.down - 1) / a.down)) + 1;
      const long long avail = m - s.out_end;
      n_out = avail <= 0 ? 0 : (avail < n_out ? (int)avail : n_out);
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {
      a.st_next->in_end = in_end;
      a.st_next->out_end = s.out_end + n_out;
      if (a.n_out_dev) *a.n_out_dev = n_out;
    }
  }
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  auto sample = [&](long long j) -> Tin { return j < new_first ? a.x[j - x_first] : a.x_new[j - new_first]; };
  if (t < n_out) {
    const long long i = out_first + t;
    double acc = 0.0;
    if (i >= 0) {
      const long long c = i * a.down + half_len;                       // tap index of input sample 0
      // tap = c - j * up in [0, n_taps)  <=>  (c - n_taps + 1) / up <= j <= c / up
      long long jlo = c - (a.n_taps - 1);
      jlo = jlo <= 0 ? 0 : (jlo + a.up - 1) / a.up;
      long long jhi = c / a.up;
      if (jlo < x_first) jlo = x_first;
      if (jhi > in_end - 1) jhi = in_end - 1;
      for (long long j = jlo; j <= jhi; ++j) acc += (double)sample(j) * a.h[c - j * a.up];
    }
    a.y[t] = (Tout)acc;
  }
  if (a.hist_next && t < a.x_len) {
    const long long j = in_end - a.x_len + t;
    a.hist_next[t] = j < 0 ? (Tin)0 : sample(j);
  }
}

template <typename Tin, typename Tout>
static int resample_launch(Engine* e, const PolyArgs<Tin, Tout>& a, cudaStream_t st) {
  const int threads = a.hist_next && a.x_len > a.n_out ? a.x_len : a.n_out;
  if (threads <= 0) return 0;
  k_resample_poly<Tin, Tout><<<(threads + 255) / 256, 256, 0, st>>>(a);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

int resample_poly_run(Engine* e, const float* d_x, int n, int up, int down, const double* d_h, int n_taps, float* d_y, int n_out, cudaStream_t st) {
  PolyArgs<float, float> a = {};
  a.mode = kPolyWhole; a.h = d_h; a.n_taps = n_taps; a.up = up; a.down = down;
  a.x = d_x; a.x_len = n; a.y = d_y; a.n_out = n_out;
  return resample_launch(e, a, st);
}

int resample_stream_in_run(Engine* e, const float* d_window, int window, int chunk, int delay, int up, int down, const double* d_h, int n_taps,
                           const ResampleState* d_st, ResampleState* d_st_next, float* d_y, int n_out, cudaStream_t st) {
  PolyArgs<float, float> a = {};
  a.mode = kPolyStreamIn; a.h = d_h; a.n_taps = n_taps; a.up = up; a.down = down;
  a.x = d_window; a.x_len = window; a.chunk = chunk; a.delay = delay; a.y = d_y; a.n_out = n_out; a.st = d_st; a.st_next = d_st_next;
  return resample_launch(e, a, st);
}

int resample_stream_out_run(Engine* e, const double* d_hist, double* d_hist_next, int hist, const double* d_new, const int* d_n_new, int up,
                            int down, const double* d_h, int n_taps, const ResampleState* d_st, ResampleState* d_st_next, double* d_y,
                            int max_out, int* d_n_out, cudaStream_t st) {
  PolyArgs<double, double> a = {};
  a.mode = kPolyStreamOut; a.h = d_h; a.n_taps = n_taps; a.up = up; a.down = down;
  a.x = d_hist; a.x_len = hist; a.hist_next = d_hist_next; a.x_new = d_new; a.n_new = d_n_new;
  a.y = d_y; a.n_out = max_out; a.n_out_dev = d_n_out; a.st = d_st; a.st_next = d_st_next;
  return resample_launch(e, a, st);
}

}  // namespace ryk
