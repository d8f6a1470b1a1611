// crepe.cu -- the CREPE f0 front-end on the H100 (SURVEY 8(f) rank 4; realtime_voice_conversion/yukarin_wrapper/
// acoustic_feature_wrapper.py:65-80: crepe.predict(x, fs, viterbi=True, model_capacity='full', step_size=frame_period) followed by
// crepe.predict_voicing).  Input is the 16 kHz signal (the caller resamples with ryk_resample_poly); output is the per-frame
// frequency, confidence and voicing state, plus the 360-bin activation.
//
//   frames (1024 samples, zero mean / unit std)  ->  im2col of the stride-4 k512 first layer  ->  six [conv -> ReLU -> BatchNorm ->
//   MaxPool 2] blocks  ->  Dense 360 + sigmoid  ->  Viterbi pitch path + local weighted average of cents  ->  2-state voicing Viterbi
//
// The reference computes CREPE in FP32 (Keras) and decodes with a per-frame ARGMAX over 360 sigmoid outputs, which an FP16 (or plain
// TF32) tensor-core evaluation moves.  So the convolutions run either on the FP32 CUDA-core implicit-GEMM kernel (conv_direct.cu:
// ryk_crepe_predict, sessions in precision 0) or on the error-compensated 3xTF32 tensor-core kernel (crepe_tc.cu: sessions in
// precision 1), which is at least as accurate.  'same' padding is materialised: every block
// writes its pooled output into the zero-framed input buffer of the next one, so all convolutions run with padding 0.  The Viterbi
// decoders use log-probability tables computed by the host mirror (realtime_yukarin_b200/crepe.py) -- the sums are then bit-identical
// to the CPU restatement and so are the arg-max decisions (hmmlearn semantics: first maximum wins).
//
// Two callers share the network (crepe_network):
//   ryk_crepe_predict   host 16 kHz signal in, host arrays out; uses the model's own workspace, grown on demand.
//   CrepePlan           the session's analysis stage (f0 method 2): a caller-owned workspace sized for one window length, so the
//                       forward (resample to 16 kHz -> network -> decoders -> voicing rule) allocates nothing, copies nothing to the
//                       host and never synchronises, and a CUDA graph can capture it.  Its f0 (0 where unvoiced) is what
//                       spectral_analysis_run reads in place of DIO/StoneMask.  While a plan exists the model refuses to change.
#include <math.h>

#include <vector>

#include "../../include/ryk.h"
#include "conv.h"
#include "crepe_tc.h"
#include "engine.h"

namespace ryk {

constexpr int kCrepeBins = 360;
static const int kCrepeFilters[6] = {32, 4, 4, 4, 8, 16};
static const int kCrepeWidths[6] = {512, 64, 64, 64, 64, 64};
static const int kCrepeStrides[6] = {4, 1, 1, 1, 1, 1};

// Buffers of one forward over F frames of n16 samples at 16 kHz.
struct CrepeWork {
  int F = 0, n16 = 0;
  float* d_audio = nullptr;
  float* d_im2col = nullptr; float* d_conv[6] = {}; float* d_in[6] = {};   // d_in[l]: zero-framed input of block l (l >= 1)
  float* d_flat = nullptr; float* d_logit = nullptr; float* d_act = nullptr;
  float* d_conf = nullptr; int* d_obs = nullptr;
  double* d_lattice = nullptr; int* d_path = nullptr; double* d_f0 = nullptr; int* d_voicing = nullptr; double* d_vlat = nullptr;
  bool tc = false;                 // convolutions on the 3xTF32 tensor-core kernel (crepe_tc.cu) instead of conv_direct
  float* d_tc_ws = nullptr;        // its split-K workspace (largest layer)
};

// Polyphase filter that brings an input rate to the model's 16 kHz (wave_io.resample_filter(up, down)).
struct CrepeResampler { int fs = 0, up = 0, down = 0, n_taps = 0; double* d_taps = nullptr; };

struct CrepeModel {
  int mult = 32;
  int cin[6], cout[6];
  float* d_w[6] = {};        // [tap][cin][cout]  (layer 0: [1][512][cout] -- a 1x1 conv over the im2col rows)
  float* d_bias[6] = {};
  float* d_ones = nullptr;   // scale = 1 for the conv epilogue (ReLU(acc + bias))
  float* d_bn_a[6] = {};     // gamma / sqrt(var + eps)
  float* d_bn_c[6] = {};     // beta - mean * a
  float* d_dense_w = nullptr;   // [64 m][360]
  float* d_dense_b = nullptr;
  double* d_log_trans = nullptr;   // [360][360]
  double* d_cents = nullptr;       // [360] crepe's cents_mapping (np.linspace(0, 7180, 360) + 1997.379...)
  double h_log_start = 0, h_log_emit[2] = {0, 0};
  bool tables = false;
  bool loaded[7] = {};
  std::vector<CrepeResampler> resamplers;
  CrepeWork work;            // workspace of ryk_crepe_predict (grown on demand)
  int plans = 0;             // live CrepePlans: captured session graphs point at the weights, so the model may not change under them
};

// A caller-owned forward for a fixed input length n at rate fs: fixed buffers, so it can be captured in a CUDA graph.
struct CrepePlan {
  CrepeWork w;
  int n = 0, hop16 = 0, up = 0, down = 0, n_taps = 0;
  const double* d_taps = nullptr;
  double* d_f0 = nullptr;    // [F] f0 after the voicing rule (0 where unvoiced)
};

static CrepeModel* g_crepe = nullptr;     // one model per process (one engine per process / GPU)

static void same_padding(int n_in, int k, int stride, int* n_out, int* left, int* right) {
  *n_out = (n_in + stride - 1) / stride;
  int total = (*n_out - 1) * stride + k - n_in;
  if (total < 0) total = 0;
  *left = total / 2; *right = total - total / 2;
}

// frames + normalisation + im2col of block 0: A[f][o][k] = xn_f[4 o + k - left] (0 outside the frame), o < 256, k < 512
__global__ void __launch_bounds__(256) k_crepe_frames(const float* __restrict__ audio, int n, int hop, int left, float* __restrict__ im2col) {
  __shared__ float fr[1024];
  __shared__ double scratch[40];
  const int f = blockIdx.x;
  // np.pad(audio, 512): frame f covers padded samples [f hop, f hop + 1024) = audio[f hop - 512 ..]
  double s = 0.0;
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) {
    const int src = f * hop + i - 512;
    const float v = (src >= 0 && src < n) ? audio[src] : 0.f;
    fr[i] = v; s += v;
  }
  const double mean = block_sum(s, scratch) / 1024.0;
  double q = 0.0;
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) { const double d = (double)((float)(fr[i] - (float)mean)); q += d * d; }
  // numpy: frames -= mean (float32); std of the centred float32 frame (population), clipped at 1e-8
  double var = block_sum(q, scratch) / 1024.0;
  double m2 = 0.0;
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) m2 += (double)((float)(fr[i] - (float)mean));
  const double mean2 = block_sum(m2, scratch) / 1024.0;      // np.std subtracts the (tiny) mean of the centred frame again
  var -= mean2 * mean2;
  const float sd = fmaxf((float)sqrt(var > 0.0 ? var : 0.0), 1e-8f);
  __syncthreads();
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) fr[i] = (float)(fr[i] - (float)mean) / sd;
  __syncthreads();
  float* dst = im2col + (size_t)f * 256 * 512;
  for (int i = threadIdx.x; i < 256 * 512; i += blockDim.x) {
    const int o = i >> 9, k = i & 511, src = 4 * o + k - left;
    dst[i] = (src >= 0 && src < 1024) ? fr[src] : 0.f;
  }
}

// BatchNorm affine then MaxPool(2) of x [F][W][C] into the interior of the next block's zero-framed input [F][W / 2 + pad_l + pad_r][C]
__global__ void k_crepe_bn_pool(const float* __restrict__ x, int F, int W, int C, const float* __restrict__ a, const float* __restrict__ c,
                                int pad_l, int pad_r, float* __restrict__ y) {
  const int Wo = W / 2, Wp = Wo + pad_l + pad_r;
  const size_t total = (size_t)F * Wp * C;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % C); const size_t r = i / C;
    const int wp = (int)(r % Wp), f = (int)(r / Wp), w = wp - pad_l;
    float v = 0.f;
    if (w >= 0 && w < Wo) {
      const float s = a[ch], t = c[ch];
      const float v0 = x[((size_t)f * W + 2 * w) * C + ch] * s + t, v1 = x[((size_t)f * W + 2 * w + 1) * C + ch] * s + t;
      v = fmaxf(v0, v1);
    }
    y[i] = v;
  }
}

// sigmoid, confidence (max) and observation (first arg-max) per frame
__global__ void __launch_bounds__(128) k_crepe_sigmoid(const float* __restrict__ logit, float* __restrict__ act, float* __restrict__ conf,
                                                      int* __restrict__ obs) {
  __shared__ float sv[128]; __shared__ int si[128];
  const int f = blockIdx.x;
  float best = -1.f; int bi = 0;
  for (int i = threadIdx.x; i < kCrepeBins; i += blockDim.x) {
    const float v = 1.f / (1.f + expf(-logit[(size_t)f * kCrepeBins + i]));
    act[(size_t)f * kCrepeBins + i] = v;
    if (v > best) { best = v; bi = i; }
  }
  sv[threadIdx.x] = best; si[threadIdx.x] = bi;
  __syncthreads();
  for (int o = 64; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      const float ov = sv[threadIdx.x + o]; const int oi = si[threadIdx.x + o];
      if (ov > sv[threadIdx.x] || (ov == sv[threadIdx.x] && oi < si[threadIdx.x])) { sv[threadIdx.x] = ov; si[threadIdx.x] = oi; }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) { conf[f] = sv[0]; obs[f] = si[0]; }
}

// first arg-max of v[0..n) over the CTA (n <= 384 = blockDim.x); all threads get the index
__device__ inline int crepe_argmax(double v, int i, int n, double* sval, int* sidx) {
  sval[threadIdx.x] = i < n ? v : -INFINITY; sidx[threadIdx.x] = i < n ? i : 0x7fffffff;
  __syncthreads();
  for (int o = 256; o > 0; o >>= 1) {
    if (threadIdx.x < o && threadIdx.x + o < blockDim.x) {
      const double ov = sval[threadIdx.x + o]; const int oi = sidx[threadIdx.x + o];
      if (ov > sval[threadIdx.x] || (ov == sval[threadIdx.x] && oi < sidx[threadIdx.x])) { sval[threadIdx.x] = ov; sidx[threadIdx.x] = oi; }
    }
    __syncthreads();
  }
  const int r = sidx[0];
  __syncthreads();
  return r;
}

// hmmlearn _viterbi over the 360 pitch bins (one CTA of 384 threads: thread j owns state j), local average of cents around the path,
// f0 = 10 * 2^(cents / 1200); then the 2-state Gaussian voicing HMM on the confidence (thread 0) and the reference's voicing rule.
__global__ void __launch_bounds__(384) k_crepe_decode(const float* __restrict__ act, const float* __restrict__ conf, const int* __restrict__ obs,
                                                     int F, const double* __restrict__ log_trans, const double* __restrict__ cents_map,
                                                     double log_start, double log_emit_self,
                                                     double log_emit_other, double* __restrict__ lattice, int* __restrict__ path,
                                                     double* __restrict__ vlat, double* __restrict__ f0, int* __restrict__ voicing) {
  __shared__ double sval[384]; __shared__ int sidx[384];
  __shared__ double prev[kCrepeBins];
  const int j = threadIdx.x;
  if (F <= 0) return;
  if (j < kCrepeBins) { const double v = log_start + (j == obs[0] ? log_emit_self : log_emit_other); lattice[j] = v; prev[j] = v; }
  __syncthreads();
  for (int t = 1; t < F; ++t) {
    double best = -INFINITY;
    if (j < kCrepeBins) {
      // np.max(lattice[t-1][:, None] + log_trans, axis=0)[j]: transitions are -inf outside |i - j| < 12
      const int lo = j - 11 < 0 ? 0 : j - 11, hi = j + 11 > kCrepeBins - 1 ? kCrepeBins - 1 : j + 11;
      for (int i = lo; i <= hi; ++i) { const double v = prev[i] + log_trans[(size_t)i * kCrepeBins + j]; if (v > best) best = v; }
      best += (j == obs[t] ? log_emit_self : log_emit_other);
      lattice[(size_t)t * kCrepeBins + j] = best;
    }
    __syncthreads();
    if (j < kCrepeBins) prev[j] = best;
    __syncthreads();
  }
  int where = crepe_argmax(j < kCrepeBins ? lattice[(size_t)(F - 1) * kCrepeBins + j] : 0.0, j, kCrepeBins, sval, sidx);
  if (j == 0) path[F - 1] = where;
  for (int t = F - 2; t >= 0; --t) {
    const double v = j < kCrepeBins ? lattice[(size_t)t * kCrepeBins + j] + log_trans[(size_t)j * kCrepeBins + where] : 0.0;
    where = crepe_argmax(v, j, kCrepeBins, sval, sidx);
    if (j == 0) path[t] = where;
  }
  __syncthreads();
  // to_local_average_cents around the path, frequency
  for (int t = j; t < F; t += blockDim.x) {
    const int center = path[t];
    const int start = center - 4 < 0 ? 0 : center - 4, end = center + 5 > kCrepeBins ? kCrepeBins : center + 5;
    // np.sum(salience * cents_mapping[start:end]) / np.sum(salience) with numpy's dtypes and summation order: the products are float64,
    // the weight sum stays float32; n < 8 elements are added left to right, otherwise eight accumulators are combined pairwise and the
    // remainder added (numpy's pairwise_sum for n <= 128).
    const int n = end - start;
    double p[9]; float s32[9];
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      const bool in = i < n;
      const float s = in ? act[(size_t)t * kCrepeBins + start + i] : 0.f;
      s32[i] = s; p[i] = in ? (double)s * cents_map[start + i] : 0.0;
    }
    double ps; float ws;
    if (n < 8) {
      ps = 0.0; ws = 0.f;
      for (int i = 0; i < n; ++i) { ps += p[i]; ws += s32[i]; }
    } else {
      ps = ((p[0] + p[1]) + (p[2] + p[3])) + ((p[4] + p[5]) + (p[6] + p[7]));
      ws = ((s32[0] + s32[1]) + (s32[2] + s32[3])) + ((s32[4] + s32[5]) + (s32[6] + s32[7]));
      for (int i = 8; i < n; ++i) { ps += p[i]; ws += s32[i]; }
    }
    const double cents = ps / (double)ws;
    double fr = 10.0 * exp2(cents / 1200.0);
    if (isnan(fr)) fr = 0.0;
    f0[t] = fr;
  }
  __syncthreads();
  // predict_voicing: 2-state Gaussian HMM (means 0 / 1, variance 0.25, start 0.5, self transition 0.99), Viterbi, first maximum wins
  if (j == 0) {
    const double ls = log(0.5), l_stay = log(0.99), l_move = log(0.01), cst = log(2.0 * kPi) + log(0.25);
    double p0 = 0, p1 = 0;
    for (int t = 0; t < F; ++t) {
      const double c = (double)conf[t];
      const double e0 = -0.5 * (cst + (c - 0.0) * (c - 0.0) / 0.25), e1 = -0.5 * (cst + (c - 1.0) * (c - 1.0) / 0.25);
      double n0, n1;
      if (t == 0) { n0 = ls + e0; n1 = ls + e1; }
      else {
        const double a0 = p0 + l_stay, a1 = p1 + l_move;        // into state 0
        const double b0 = p0 + l_move, b1 = p1 + l_stay;        // into state 1
        n0 = (a1 > a0 ? a1 : a0) + e0; n1 = (b1 > b0 ? b1 : b0) + e1;
      }
      vlat[2 * t] = n0; vlat[2 * t + 1] = n1; p0 = n0; p1 = n1;
    }
    int w = vlat[2 * (F - 1) + 1] > vlat[2 * (F - 1)] ? 1 : 0;
    voicing[F - 1] = w;
    for (int t = F - 2; t >= 0; --t) {
      const double v0 = vlat[2 * t] + (w == 0 ? l_stay : l_move), v1 = vlat[2 * t + 1] + (w == 1 ? l_stay : l_move);
      w = v1 > v0 ? 1 : 0;
      voicing[t] = w;
    }
  }
}

// the reference's rule (acoustic_feature_wrapper.py:78-79): voiced = (predict_voicing == 1) | (confidence > 0.1); f0[~voiced] = 0.
// numpy compares the float32 confidence with the Python scalar in float32.
__global__ void k_crepe_voiced(const double* __restrict__ f0, const float* __restrict__ conf, const int* __restrict__ voicing, int F,
                               double* __restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < F) out[t] = (voicing[t] == 1 || conf[t] > 0.1f) ? f0[t] : 0.0;
}

// ---- host side -----------------------------------------------------------------------------------------------------------------
static void work_free(CrepeWork& w) {
  for (int l = 0; l < 6; ++l) { cudaFree(w.d_conv[l]); cudaFree(w.d_in[l]); }
  void* ptrs[] = {w.d_audio, w.d_im2col, w.d_flat, w.d_logit, w.d_act, w.d_conf, w.d_obs, w.d_lattice, w.d_path, w.d_f0, w.d_voicing, w.d_vlat,
                  w.d_tc_ws};
  for (void* p : ptrs) cudaFree(p);
  w = CrepeWork();
}

static void crepe_free(CrepeModel* m) {
  if (!m) return;
  for (int l = 0; l < 6; ++l) { cudaFree(m->d_w[l]); cudaFree(m->d_bias[l]); cudaFree(m->d_bn_a[l]); cudaFree(m->d_bn_c[l]); }
  void* ptrs[] = {m->d_ones, m->d_dense_w, m->d_dense_b, m->d_log_trans, m->d_cents};
  for (void* p : ptrs) cudaFree(p);
  for (CrepeResampler& r : m->resamplers) cudaFree(r.d_taps);
  work_free(m->work);
  delete m;
}

static int crepe_check_unused(const CrepeModel* m) {
  RYK_CHECK(m == nullptr || m->plans == 0, "the CREPE model is in use by a live session (f0 method 2): destroy those sessions before changing it");
  return 0;
}

int crepe_create(Engine* e, int capacity_multiplier) {
  RYK_CHECK(capacity_multiplier == 4 || capacity_multiplier == 8 || capacity_multiplier == 16 || capacity_multiplier == 24 || capacity_multiplier == 32,
            "CREPE capacity multiplier must be 4 (tiny), 8, 16, 24 or 32 (full)");
  if (crepe_check_unused(g_crepe)) return -1;
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  crepe_free(g_crepe);
  CrepeModel* m = new CrepeModel();
  m->mult = capacity_multiplier;
  for (int l = 0; l < 6; ++l) { m->cout[l] = kCrepeFilters[l] * m->mult; m->cin[l] = l == 0 ? 1 : m->cout[l - 1]; }
  std::vector<float> ones(1024, 1.f);
  RYK_CUDA(cudaMalloc(&m->d_ones, sizeof(float) * 1024));
  RYK_CUDA(cudaMemcpy(m->d_ones, ones.data(), sizeof(float) * 1024, cudaMemcpyHostToDevice));
  g_crepe = m;
  return 0;
}

void crepe_destroy() { crepe_free(g_crepe); g_crepe = nullptr; }

// W: (cout, cin, k) as in the restatement's npz; BatchNorm statistics of the block (eps 1e-3)
int crepe_set_conv(Engine* e, int layer, const float* W, const float* bias, const float* gamma, const float* beta, const float* mean, const float* var) {
  CrepeModel* m = g_crepe;
  RYK_CHECK(m != nullptr && layer >= 0 && layer < 6, "create the CREPE model first; layers are 0..5");
  if (crepe_check_unused(m)) return -1;
  const int cin = m->cin[layer], cout = m->cout[layer], k = kCrepeWidths[layer];
  const size_t nw = (size_t)cout * cin * k;
  float* d_tmp = nullptr;
  RYK_CUDA(cudaMalloc(&d_tmp, sizeof(float) * nw));
  RYK_CUDA(cudaMemcpyAsync(d_tmp, W, sizeof(float) * nw, cudaMemcpyHostToDevice, e->stream));
  if (!m->d_w[layer]) RYK_CUDA(cudaMalloc(&m->d_w[layer], sizeof(float) * nw));
  // conv weights (cout, cin, 1, k) -> [tap][cin][cout]; for layer 0 (cin = 1) this is [512][1][cout] = the [K = 512][cout] matrix of the im2col GEMM
  if (pack_weights_direct(d_tmp, 0, cin, cout, 1, k, m->d_w[layer], e->stream)) return -1;
  std::vector<float> a(cout), c(cout);
  for (int i = 0; i < cout; ++i) {
    const double ai = (double)gamma[i] / sqrt((double)var[i] + 1e-3);
    a[i] = (float)ai; c[i] = (float)((double)beta[i] - (double)mean[i] * (double)a[i]);
  }
  if (!m->d_bias[layer]) { RYK_CUDA(cudaMalloc(&m->d_bias[layer], sizeof(float) * cout)); RYK_CUDA(cudaMalloc(&m->d_bn_a[layer], sizeof(float) * cout)); RYK_CUDA(cudaMalloc(&m->d_bn_c[layer], sizeof(float) * cout)); }
  RYK_CUDA(cudaMemcpyAsync(m->d_bias[layer], bias, sizeof(float) * cout, cudaMemcpyHostToDevice, e->stream));
  RYK_CUDA(cudaMemcpyAsync(m->d_bn_a[layer], a.data(), sizeof(float) * cout, cudaMemcpyHostToDevice, e->stream));
  RYK_CUDA(cudaMemcpyAsync(m->d_bn_c[layer], c.data(), sizeof(float) * cout, cudaMemcpyHostToDevice, e->stream));
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  RYK_CUDA(cudaFree(d_tmp));
  m->loaded[layer] = true;
  return 0;
}

// W: (360, 64 m) row-major (Keras kernel transposed), bias (360)
int crepe_set_dense(Engine* e, const float* W, const float* bias) {
  CrepeModel* m = g_crepe;
  RYK_CHECK(m != nullptr, "create the CREPE model first");
  if (crepe_check_unused(m)) return -1;
  const int nin = 4 * m->cout[5];
  float* d_tmp = nullptr;
  RYK_CUDA(cudaMalloc(&d_tmp, sizeof(float) * nin * kCrepeBins));
  RYK_CUDA(cudaMemcpyAsync(d_tmp, W, sizeof(float) * nin * kCrepeBins, cudaMemcpyHostToDevice, e->stream));
  if (!m->d_dense_w) { RYK_CUDA(cudaMalloc(&m->d_dense_w, sizeof(float) * nin * kCrepeBins)); RYK_CUDA(cudaMalloc(&m->d_dense_b, sizeof(float) * kCrepeBins)); }
  if (pack_weights_direct(d_tmp, 0, nin, kCrepeBins, 1, 1, m->d_dense_w, e->stream)) return -1;      // (cout, cin, 1, 1) -> [cin][cout]
  RYK_CUDA(cudaMemcpyAsync(m->d_dense_b, bias, sizeof(float) * kCrepeBins, cudaMemcpyHostToDevice, e->stream));
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  RYK_CUDA(cudaFree(d_tmp));
  m->loaded[6] = true;
  return 0;
}

int crepe_set_tables(Engine* e, const double* log_trans, const double* cents_mapping, double log_start, double log_emit_self, double log_emit_other) {
  CrepeModel* m = g_crepe;
  RYK_CHECK(m != nullptr, "create the CREPE model first");
  if (crepe_check_unused(m)) return -1;
  if (!m->d_log_trans) RYK_CUDA(cudaMalloc(&m->d_log_trans, sizeof(double) * kCrepeBins * kCrepeBins));
  RYK_CUDA(cudaMemcpy(m->d_log_trans, log_trans, sizeof(double) * kCrepeBins * kCrepeBins, cudaMemcpyHostToDevice));
  if (!m->d_cents) RYK_CUDA(cudaMalloc(&m->d_cents, sizeof(double) * kCrepeBins));
  RYK_CUDA(cudaMemcpy(m->d_cents, cents_mapping, sizeof(double) * kCrepeBins, cudaMemcpyHostToDevice));
  m->h_log_start = log_start; m->h_log_emit[0] = log_emit_self; m->h_log_emit[1] = log_emit_other;
  m->tables = true;
  return 0;
}

int crepe_num_frames(int n16, double step_ms) {
  const int hop = (int)(16000 * step_ms / 1000);
  return hop > 0 ? 1 + (int)((n16 + 1024 - 1024) / hop) : 0;
}

static int work_alloc(const CrepeModel* m, CrepeWork& w, int F, int n16, bool tc) {
  RYK_CUDA(cudaMalloc(&w.d_audio, sizeof(float) * n16));
  RYK_CUDA(cudaMalloc(&w.d_im2col, sizeof(float) * (size_t)F * 256 * 512));
  int W = 256;                                           // output length of block 0 before pooling
  for (int l = 0; l < 6; ++l) {
    RYK_CUDA(cudaMalloc(&w.d_conv[l], sizeof(float) * (size_t)F * W * m->cout[l]));
    const int Wo = W / 2;
    if (l < 5) {
      int n_out, left, right; same_padding(Wo, kCrepeWidths[l + 1], kCrepeStrides[l + 1], &n_out, &left, &right);
      RYK_CUDA(cudaMalloc(&w.d_in[l + 1], sizeof(float) * (size_t)F * (Wo + left + right) * m->cout[l]));
      W = n_out;
    }
  }
  RYK_CUDA(cudaMalloc(&w.d_flat, sizeof(float) * (size_t)F * 4 * m->cout[5]));
  RYK_CUDA(cudaMalloc(&w.d_logit, sizeof(float) * (size_t)F * kCrepeBins));
  RYK_CUDA(cudaMalloc(&w.d_act, sizeof(float) * (size_t)F * kCrepeBins));
  RYK_CUDA(cudaMalloc(&w.d_conf, sizeof(float) * F));
  RYK_CUDA(cudaMalloc(&w.d_obs, sizeof(int) * F));
  RYK_CUDA(cudaMalloc(&w.d_lattice, sizeof(double) * (size_t)F * kCrepeBins));
  RYK_CUDA(cudaMalloc(&w.d_path, sizeof(int) * F));
  RYK_CUDA(cudaMalloc(&w.d_f0, sizeof(double) * F));
  RYK_CUDA(cudaMalloc(&w.d_voicing, sizeof(int) * F));
  RYK_CUDA(cudaMalloc(&w.d_vlat, sizeof(double) * 2 * F));
  if (tc) {
    size_t ws = crepe_tc_ws_floats(F * 256, 512, m->cout[0]);
    int Wl = 128;
    for (int l = 1; l < 6; ++l) {
      const size_t need = crepe_tc_ws_floats(F * Wl, kCrepeWidths[l] * m->cin[l], m->cout[l]);
      if (need > ws) ws = need;
      Wl /= 2;
    }
    if (ws) RYK_CUDA(cudaMalloc(&w.d_tc_ws, sizeof(float) * ws));
  }
  w.F = F; w.n16 = n16; w.tc = tc;
  return 0;
}

// conv layer l over x = [F][Win][Cin] (layer 0: the im2col rows, Win = 256, Cin = 512, KW = 1) -> ReLU(conv + bias) [F][Wout][Cout],
// stride 1, no padding (the buffers are already zero-framed)
static int crepe_conv(Engine* e, CrepeModel* m, const CrepeWork& w, int l, const float* x, int F, int Win, int Cin, int KW, int Wout, float* y,
                      cudaStream_t st) {
  if (w.tc) {
    CrepeGemm g;
    g.x = x; g.M = F * Wout; g.W = Wout; g.fstride = (long long)Win * Cin; g.wstep = Cin; g.K = KW * Cin; g.N = m->cout[l];
    g.w = m->d_w[l]; g.bias = m->d_bias[l]; g.y = y;
    return crepe_tc_run(g, w.d_tc_ws, st);
  }
  ConvLayer L;
  L.transposed = 0; L.B = F; L.Hin = 1; L.Win = Win; L.Hout = 1; L.Wout = Wout; L.C0 = Cin; L.C1 = 0; L.Cout = m->cout[l];
  L.KH = 1; L.KW = KW; L.SH = 1; L.SW = 1; L.PH = 0; L.PW = 0; L.act = ACT_RELU;
  L.in0 = x; L.in_dtype = DT_F32; L.out = y; L.out_dtype = DT_F32;
  L.wt.w[0] = m->d_w[l]; L.wt.scale[0] = m->d_ones; L.wt.shift[0] = m->d_bias[l];
  return conv_direct_run(L, st);
}

static bool crepe_complete(const CrepeModel* m) {
  if (m == nullptr || !m->tables) return false;
  for (bool b : m->loaded) if (!b) return false;
  return true;
}

// frames -> network -> sigmoid -> decoders over the n16 samples in w.d_audio (F frames at hop samples); stream-ordered only
static int crepe_network(Engine* e, CrepeModel* m, CrepeWork& w, int n16, int hop, int F, cudaStream_t st) {
  int n_out, left, right;
  same_padding(1024, 512, 4, &n_out, &left, &right);                 // 256 outputs, 254 + 254
  k_crepe_frames<<<F, 256, 0, st>>>(w.d_audio, n16, hop, left, w.d_im2col);
  // block 0: 1x1 conv over the im2col rows ([F][256][512] x [512][cout])
  if (crepe_conv(e, m, w, 0, w.d_im2col, F, 256, 512, 1, 256, w.d_conv[0], st)) return -1;
  int W = 256;
  for (int l = 0; l < 6; ++l) {
    const int Wo = W / 2;
    if (l < 5) {
      int nl, pl, pr; same_padding(Wo, kCrepeWidths[l + 1], kCrepeStrides[l + 1], &nl, &pl, &pr);
      k_crepe_bn_pool<<<296, 256, 0, st>>>(w.d_conv[l], F, W, m->cout[l], m->d_bn_a[l], m->d_bn_c[l], pl, pr, w.d_in[l + 1]);
      if (crepe_conv(e, m, w, l + 1, w.d_in[l + 1], F, Wo + pl + pr, m->cout[l], kCrepeWidths[l + 1], nl, w.d_conv[l + 1], st)) return -1;
      W = nl;
    } else {
      k_crepe_bn_pool<<<296, 256, 0, st>>>(w.d_conv[l], F, W, m->cout[l], m->d_bn_a[l], m->d_bn_c[l], 0, 0, w.d_flat);   // [F][4][C] = time-major flatten
    }
  }
  {                                                                   // Dense(360): 1x1 conv over [F][1][64 m]
    ConvLayer L;
    L.transposed = 0; L.B = F; L.Hin = 1; L.Win = 1; L.Hout = 1; L.Wout = 1; L.C0 = 4 * m->cout[5]; L.C1 = 0; L.Cout = kCrepeBins;
    L.KH = 1; L.KW = 1; L.SH = 1; L.SW = 1; L.PH = 0; L.PW = 0; L.act = ACT_NONE;
    L.in0 = w.d_flat; L.in_dtype = DT_F32; L.out = w.d_logit; L.out_dtype = DT_F32;
    L.wt.w[0] = m->d_dense_w; L.wt.scale[0] = m->d_ones; L.wt.shift[0] = m->d_dense_b;
    if (conv_direct_run(L, st)) return -1;
  }
  k_crepe_sigmoid<<<F, 128, 0, st>>>(w.d_logit, w.d_act, w.d_conf, w.d_obs);
  k_crepe_decode<<<1, 384, 0, st>>>(w.d_act, w.d_conf, w.d_obs, F, m->d_log_trans, m->d_cents, m->h_log_start, m->h_log_emit[0], m->h_log_emit[1],
                                   w.d_lattice, w.d_path, w.d_vlat, w.d_f0, w.d_voicing);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

// audio16k: host float32, n samples at 16 kHz.  Outputs (host, any may be null): f0 / confidence [F], voicing [F] (HMM state), activation [F][360].
int crepe_predict(Engine* e, const float* audio16k, int n, double step_ms, double* f0, float* confidence, int* voicing, float* activation,
                  int* path_out) {
  CrepeModel* m = g_crepe;
  RYK_CHECK(m != nullptr && m->tables, "CREPE model / decoder tables not loaded");
  RYK_CHECK(crepe_complete(m), "CREPE model is missing a layer");
  RYK_CHECK(m->cout[0] <= 1024, "scale vector too short");
  const int hop = (int)(16000 * step_ms / 1000);
  RYK_CHECK(hop > 0 && n > 0, "bad step size or empty signal");
  const int F = crepe_num_frames(n, step_ms);
  cudaStream_t st = e->stream;
  CrepeWork& w = m->work;
  if (F > w.F || n > w.n16) {
    const int F_cap = F > w.F ? F : w.F, n_cap = n > w.n16 ? n : w.n16;
    RYK_CUDA(cudaStreamSynchronize(st));
    work_free(w);
    if (work_alloc(m, w, F_cap, n_cap, false)) { work_free(w); return -1; }
  }
  RYK_CUDA(cudaMemcpyAsync(w.d_audio, audio16k, sizeof(float) * n, cudaMemcpyHostToDevice, st));
  if (crepe_network(e, m, w, n, hop, F, st)) return -1;
  if (f0) RYK_CUDA(cudaMemcpyAsync(f0, w.d_f0, sizeof(double) * F, cudaMemcpyDeviceToHost, st));
  if (confidence) RYK_CUDA(cudaMemcpyAsync(confidence, w.d_conf, sizeof(float) * F, cudaMemcpyDeviceToHost, st));
  if (voicing) RYK_CUDA(cudaMemcpyAsync(voicing, w.d_voicing, sizeof(int) * F, cudaMemcpyDeviceToHost, st));
  if (activation) RYK_CUDA(cudaMemcpyAsync(activation, w.d_act, sizeof(float) * (size_t)F * kCrepeBins, cudaMemcpyDeviceToHost, st));
  if (path_out) RYK_CUDA(cudaMemcpyAsync(path_out, w.d_path, sizeof(int) * F, cudaMemcpyDeviceToHost, st));
  RYK_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// taps: the (odd-length) resample_poly filter for fs -> 16 kHz, up / down = 16000 / fs reduced
int crepe_set_resampler(Engine* e, int fs, int up, int down, const double* taps, int n_taps) {
  CrepeModel* m = g_crepe;
  RYK_CHECK(m != nullptr, "create the CREPE model first");
  if (crepe_check_unused(m)) return -1;
  RYK_CHECK(fs > 0 && up > 0 && down > 0 && (long long)fs * up == 16000LL * down, "up / down must map fs to 16 kHz");
  RYK_CHECK(taps != nullptr && n_taps > 0 && (n_taps & 1), "the resampler filter must have an odd number of taps");
  CrepeResampler* r = nullptr;
  for (CrepeResampler& x : m->resamplers) if (x.fs == fs) r = &x;
  if (!r) { m->resamplers.emplace_back(); r = &m->resamplers.back(); r->fs = fs; }
  if (r->d_taps && r->n_taps != n_taps) { RYK_CUDA(cudaFree(r->d_taps)); r->d_taps = nullptr; }
  if (!r->d_taps) RYK_CUDA(cudaMalloc(&r->d_taps, sizeof(double) * n_taps));
  RYK_CUDA(cudaMemcpy(r->d_taps, taps, sizeof(double) * n_taps, cudaMemcpyHostToDevice));
  r->up = up; r->down = down; r->n_taps = n_taps;
  return 0;
}

void crepe_plan_free(CrepePlan* p) {
  if (!p) return;
  work_free(p->w);
  cudaFree(p->d_f0);
  if (g_crepe) g_crepe->plans--;
  delete p;
}

// A forward for n samples at fs, analysed with frame_period: the frames must coincide with WORLD's n / hop + 1.
// Precision mode 1 runs the convolutions on the 3xTF32 tensor-core kernel, mode 0 on conv_direct (the FP32 bisect mode).
const char* crepe_plan_refusal(int fs) {
  if (!crepe_complete(g_crepe)) return "f0 method 2 (CREPE) needs a complete CREPE model and decoder tables: load one first (RYK_CREPE_MODEL)";
  for (const CrepeResampler& x : g_crepe->resamplers) if (x.fs == fs) return nullptr;
  return "f0 method 2 (CREPE): no resampler taps to 16 kHz for this sampling rate (ryk_crepe_set_resampler)";
}

int crepe_plan_create(Engine* e, int n, int fs, double frame_period, CrepePlan** out) {
  if (const char* refusal = crepe_plan_refusal(fs)) { set_error(refusal); return -2; }
  CrepeModel* m = g_crepe;
  const CrepeResampler* r = nullptr;
  for (const CrepeResampler& x : m->resamplers) if (x.fs == fs) r = &x;
  const int hop = (int)(fs * frame_period / 1000.0), hop16 = (int)(16000 * frame_period / 1000);
  const int n16 = ryk_resample_length(n, r->up, r->down);
  RYK_CHECK(hop > 0 && hop16 > 0 && n > 0, "bad frame period or empty window");
  const int F = crepe_num_frames(n16, frame_period);
  RYK_CHECK(F == n / hop + 1, "f0 method 2 (CREPE): the CREPE frame count of the analysis window differs from WORLD's n / hop + 1");
  CrepePlan* p = new CrepePlan();
  m->plans++;
  p->n = n; p->hop16 = hop16; p->up = r->up; p->down = r->down; p->n_taps = r->n_taps; p->d_taps = r->d_taps;
  if (work_alloc(m, p->w, F, n16, e->precision == 1) || cudaMalloc(&p->d_f0, sizeof(double) * F) != cudaSuccess) {
    crepe_plan_free(p);
    RYK_CHECK(false, "f0 method 2 (CREPE): out of device memory for the analysis plan");
  }
  *out = p;
  return 0;
}

// resample d_x (n samples at fs) to 16 kHz, run the network and decoders and apply the voicing rule into crepe_plan_f0(p).
// No allocation, host copy or synchronisation: the sequence can be captured in a CUDA graph.
int crepe_plan_run(Engine* e, CrepePlan* p, const float* d_x, cudaStream_t st) {
  CrepeModel* m = g_crepe;
  CrepeWork& w = p->w;
  if (resample_poly_run(e, d_x, p->n, p->up, p->down, p->d_taps, p->n_taps, w.d_audio, w.n16, st)) return -1;
  if (crepe_network(e, m, w, w.n16, p->hop16, w.F, st)) return -1;
  k_crepe_voiced<<<(w.F + 127) / 128, 128, 0, st>>>(w.d_f0, w.d_conf, w.d_voicing, w.F, p->d_f0);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

const double* crepe_plan_f0(const CrepePlan* p) { return p->d_f0; }

// ---- test entry points ---------------------------------------------------------------------------------------------------------
// One CREPE-shaped conv layer in isolation: x [F][Win][Cin], W (Cout, Cin, k), stride 1, no padding -> y = ReLU(conv + bias)
// [F][Win - k + 1][Cout].  Layer 1 is given as its im2col form (Win = 256, Cin = 512, k = 1).  backend 0: conv_direct, 1: crepe_tc.
int crepe_test_conv(Engine* e, int backend, int F, int Win, int Cin, int Cout, int k, const float* x, const float* W, const float* bias, float* y) {
  RYK_CHECK((backend == 0 || backend == 1) && F > 0 && Cin > 0 && Cout > 0 && k > 0 && Win >= k, "bad CREPE test-conv arguments");
  const int Wout = Win - k + 1;
  const size_t nx = (size_t)F * Win * Cin, nw = (size_t)Cout * Cin * k, ny = (size_t)F * Wout * Cout;
  const size_t nws = backend ? crepe_tc_ws_floats(F * Wout, k * Cin, Cout) : 0;
  cudaStream_t st = e->stream;
  std::vector<void*> frees;
  auto A = [&](size_t bytes) -> float* { void* p = nullptr; if (cudaMalloc(&p, bytes ? bytes : 16) != cudaSuccess) return nullptr; frees.push_back(p); return (float*)p; };
  float *d_x = A(nx * 4), *d_wraw = A(nw * 4), *d_w = A(nw * 4), *d_b = A(Cout * 4), *d_ones = A(Cout * 4), *d_y = A(ny * 4), *d_ws = A(nws * 4);
  int rc = -1;
  if (d_x && d_wraw && d_w && d_b && d_ones && d_y && d_ws) {
    std::vector<float> ones(Cout, 1.f);
    cudaMemcpyAsync(d_x, x, nx * 4, cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(d_wraw, W, nw * 4, cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(d_b, bias, Cout * 4, cudaMemcpyHostToDevice, st);
    cudaMemcpyAsync(d_ones, ones.data(), Cout * 4, cudaMemcpyHostToDevice, st);
    rc = pack_weights_direct(d_wraw, 0, Cin, Cout, 1, k, d_w, st);
    if (!rc && backend) {
      CrepeGemm g;
      g.x = d_x; g.M = F * Wout; g.W = Wout; g.fstride = (long long)Win * Cin; g.wstep = Cin; g.K = k * Cin; g.N = Cout;
      g.w = d_w; g.bias = d_b; g.y = d_y;
      rc = crepe_tc_run(g, d_ws, st);
    } else if (!rc) {
      ConvLayer L;
      L.transposed = 0; L.B = F; L.Hin = 1; L.Win = Win; L.Hout = 1; L.Wout = Wout; L.C0 = Cin; L.C1 = 0; L.Cout = Cout;
      L.KH = 1; L.KW = k; L.SH = 1; L.SW = 1; L.PH = 0; L.PW = 0; L.act = ACT_RELU;
      L.in0 = d_x; L.in_dtype = DT_F32; L.out = d_y; L.out_dtype = DT_F32; L.wt.w[0] = d_w; L.wt.scale[0] = d_ones; L.wt.shift[0] = d_b;
      rc = conv_direct_run(L, st);
    }
    if (!rc && (cudaMemcpyAsync(y, d_y, ny * 4, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)) {
      rc = -1;
      set_error("CREPE test conv failed on the device");
    }
  } else {
    set_error("cudaMalloc failed in the CREPE test conv");
  }
  cudaStreamSynchronize(st);
  for (void* p : frees) cudaFree(p);
  return rc;
}

// The network and decoders on a host 16 kHz signal with an explicit conv backend (0: conv_direct, 1: crepe_tc), on a workspace of its
// own.  activation [F][360], path / voicing [F] (any may be null).  repeat > 0: that many further network runs are timed with CUDA
// events and *ms_per_run receives their mean device time.
int crepe_test_network(Engine* e, int backend, const float* audio16k, int n, double step_ms, float* activation, int* path, int* voicing,
                       int repeat, float* ms_per_run) {
  CrepeModel* m = g_crepe;
  RYK_CHECK(crepe_complete(m), "CREPE model / decoder tables not loaded");
  RYK_CHECK(backend == 0 || backend == 1, "backend must be 0 (conv_direct) or 1 (3xTF32 tensor cores)");
  const int hop = (int)(16000 * step_ms / 1000);
  RYK_CHECK(hop > 0 && n > 0, "bad step size or empty signal");
  const int F = crepe_num_frames(n, step_ms);
  cudaStream_t st = e->stream;
  CrepeWork w;
  int rc = work_alloc(m, w, F, n, backend == 1);
  cudaEvent_t ev[2] = {nullptr, nullptr};
  if (!rc) rc = cudaMemcpyAsync(w.d_audio, audio16k, sizeof(float) * n, cudaMemcpyHostToDevice, st) == cudaSuccess ? 0 : -1;
  if (!rc) rc = crepe_network(e, m, w, n, hop, F, st);
  if (!rc && activation) rc = cudaMemcpyAsync(activation, w.d_act, sizeof(float) * (size_t)F * kCrepeBins, cudaMemcpyDeviceToHost, st) == cudaSuccess ? 0 : -1;
  if (!rc && path) rc = cudaMemcpyAsync(path, w.d_path, sizeof(int) * F, cudaMemcpyDeviceToHost, st) == cudaSuccess ? 0 : -1;
  if (!rc && voicing) rc = cudaMemcpyAsync(voicing, w.d_voicing, sizeof(int) * F, cudaMemcpyDeviceToHost, st) == cudaSuccess ? 0 : -1;
  if (!rc && repeat > 0 && ms_per_run) {
    rc = (cudaEventCreate(&ev[0]) == cudaSuccess && cudaEventCreate(&ev[1]) == cudaSuccess && cudaEventRecord(ev[0], st) == cudaSuccess) ? 0 : -1;
    for (int i = 0; i < repeat && !rc; ++i) rc = crepe_network(e, m, w, n, hop, F, st);
    float ms = 0.f;
    if (!rc) rc = (cudaEventRecord(ev[1], st) == cudaSuccess && cudaEventSynchronize(ev[1]) == cudaSuccess &&
                   cudaEventElapsedTime(&ms, ev[0], ev[1]) == cudaSuccess) ? 0 : -1;
    if (!rc) *ms_per_run = ms / repeat;
  }
  if (cudaStreamSynchronize(st) != cudaSuccess && !rc) rc = -1;
  for (cudaEvent_t x : ev) if (x) cudaEventDestroy(x);
  work_free(w);
  if (rc) set_error("CREPE test network failed");
  return rc;
}

}  // namespace ryk
