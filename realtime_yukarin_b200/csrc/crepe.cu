// crepe.cu -- the CREPE f0 front-end on the H100 (SURVEY 8(f) rank 4; realtime_voice_conversion/yukarin_wrapper/
// acoustic_feature_wrapper.py:65-80: crepe.predict(x, fs, viterbi=True, model_capacity='full', step_size=frame_period) followed by
// crepe.predict_voicing).  Input is the 16 kHz signal (the caller resamples with ryk_resample_poly); output is the per-frame
// frequency, confidence and voicing state, plus the 360-bin activation.
//
//   frames (1024 samples, zero mean / unit std)  ->  im2col of the stride-4 k512 first layer  ->  six [conv -> ReLU -> BatchNorm ->
//   MaxPool 2] blocks  ->  Dense 360 + sigmoid  ->  Viterbi pitch path + local weighted average of cents  ->  2-state voicing Viterbi
//
// The convolutions run on the FP32 CUDA-core implicit-GEMM kernel (conv_direct.cu): the reference computes CREPE in FP32 (Keras), the
// decoding is a per-frame ARGMAX over 360 sigmoid outputs, and an FP16 tensor-core evaluation moves those maxima; this mode is outside
// the benchmarked path (BASELINE config 2 uses WORLD f0), so reference precision is kept.  'same' padding is materialised: every block
// writes its pooled output into the zero-framed input buffer of the next one, so all convolutions run with padding 0.  The Viterbi
// decoders use log-probability tables computed by the host mirror (realtime_yukarin_b200/crepe.py) -- the sums are then bit-identical
// to the CPU restatement and so are the arg-max decisions (hmmlearn semantics: first maximum wins).
#include <math.h>

#include <vector>

#include "conv.h"
#include "engine.h"

namespace ryk {

constexpr int kCrepeBins = 360;
static const int kCrepeFilters[6] = {32, 4, 4, 4, 8, 16};
static const int kCrepeWidths[6] = {512, 64, 64, 64, 64, 64};
static const int kCrepeStrides[6] = {4, 1, 1, 1, 1, 1};

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
  // workspace of the last plan (grown on demand)
  int cap_frames = 0;
  float *d_audio = nullptr; int cap_audio = 0;
  float* d_im2col = nullptr; float* d_conv[6] = {}; float* d_in[6] = {};   // d_in[l]: zero-framed input of block l (l >= 1)
  float* d_flat = nullptr; float* d_logit = nullptr; float* d_act = nullptr;
  float* d_conf = nullptr; int* d_obs = nullptr;
  double* d_lattice = nullptr; int* d_path = nullptr; double* d_f0 = nullptr; int* d_voicing = nullptr; double* d_vlat = nullptr;
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

// ---- host side -----------------------------------------------------------------------------------------------------------------
static void crepe_free(CrepeModel* m) {
  if (!m) return;
  for (int l = 0; l < 6; ++l) { cudaFree(m->d_w[l]); cudaFree(m->d_bias[l]); cudaFree(m->d_bn_a[l]); cudaFree(m->d_bn_c[l]); cudaFree(m->d_conv[l]); cudaFree(m->d_in[l]); }
  void* ptrs[] = {m->d_ones, m->d_dense_w, m->d_dense_b, m->d_log_trans, m->d_cents, m->d_audio, m->d_im2col, m->d_flat, m->d_logit, m->d_act, m->d_conf, m->d_obs,
                  m->d_lattice, m->d_path, m->d_f0, m->d_voicing, m->d_vlat};
  for (void* p : ptrs) cudaFree(p);
  delete m;
}

int crepe_create(Engine* e, int capacity_multiplier) {
  RYK_CHECK(capacity_multiplier == 4 || capacity_multiplier == 8 || capacity_multiplier == 16 || capacity_multiplier == 24 || capacity_multiplier == 32,
            "CREPE capacity multiplier must be 4 (tiny), 8, 16, 24 or 32 (full)");
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

static int crepe_reserve(CrepeModel* m, int F, int n) {
  if (n > m->cap_audio) { cudaFree(m->d_audio); RYK_CUDA(cudaMalloc(&m->d_audio, sizeof(float) * n)); m->cap_audio = n; }
  if (F <= m->cap_frames) return 0;
  cudaFree(m->d_im2col); cudaFree(m->d_flat); cudaFree(m->d_logit); cudaFree(m->d_act); cudaFree(m->d_conf); cudaFree(m->d_obs);
  cudaFree(m->d_lattice); cudaFree(m->d_path); cudaFree(m->d_f0); cudaFree(m->d_voicing); cudaFree(m->d_vlat);
  for (int l = 0; l < 6; ++l) { cudaFree(m->d_conv[l]); cudaFree(m->d_in[l]); m->d_conv[l] = m->d_in[l] = nullptr; }
  RYK_CUDA(cudaMalloc(&m->d_im2col, sizeof(float) * (size_t)F * 256 * 512));
  int W = 256;                                           // output length of block 0 before pooling
  for (int l = 0; l < 6; ++l) {
    RYK_CUDA(cudaMalloc(&m->d_conv[l], sizeof(float) * (size_t)F * W * m->cout[l]));
    const int Wo = W / 2;
    if (l < 5) {
      int n_out, left, right; same_padding(Wo, kCrepeWidths[l + 1], kCrepeStrides[l + 1], &n_out, &left, &right);
      RYK_CUDA(cudaMalloc(&m->d_in[l + 1], sizeof(float) * (size_t)F * (Wo + left + right) * m->cout[l]));
      W = n_out;
    }
  }
  RYK_CUDA(cudaMalloc(&m->d_flat, sizeof(float) * (size_t)F * 4 * m->cout[5]));
  RYK_CUDA(cudaMalloc(&m->d_logit, sizeof(float) * (size_t)F * kCrepeBins));
  RYK_CUDA(cudaMalloc(&m->d_act, sizeof(float) * (size_t)F * kCrepeBins));
  RYK_CUDA(cudaMalloc(&m->d_conf, sizeof(float) * F));
  RYK_CUDA(cudaMalloc(&m->d_obs, sizeof(int) * F));
  RYK_CUDA(cudaMalloc(&m->d_lattice, sizeof(double) * (size_t)F * kCrepeBins));
  RYK_CUDA(cudaMalloc(&m->d_path, sizeof(int) * F));
  RYK_CUDA(cudaMalloc(&m->d_f0, sizeof(double) * F));
  RYK_CUDA(cudaMalloc(&m->d_voicing, sizeof(int) * F));
  RYK_CUDA(cudaMalloc(&m->d_vlat, sizeof(double) * 2 * F));
  m->cap_frames = F;
  return 0;
}

static int crepe_conv(Engine* e, CrepeModel* m, int l, const float* d_in, int F, int Win, int Cin, int KW, int SW, int Wout, float* d_out, cudaStream_t st) {
  ConvLayer L;
  L.transposed = 0; L.B = F; L.Hin = 1; L.Win = Win; L.Hout = 1; L.Wout = Wout; L.C0 = Cin; L.C1 = 0; L.Cout = m->cout[l];
  L.KH = 1; L.KW = KW; L.SH = 1; L.SW = SW; L.PH = 0; L.PW = 0; L.act = ACT_RELU;
  L.in0 = d_in; L.in_dtype = DT_F32; L.out = d_out; L.out_dtype = DT_F32;
  L.w_direct = m->d_w[l]; L.scale = m->d_ones; L.shift = m->d_bias[l];
  e->launches += 1;
  return conv_direct_run(L, st);
}

// audio16k: host float32, n samples at 16 kHz.  Outputs (host, any may be null): f0 / confidence [F], voicing [F] (HMM state), activation [F][360].
int crepe_predict(Engine* e, const float* audio16k, int n, double step_ms, double* f0, float* confidence, int* voicing, float* activation,
                  int* path_out) {
  CrepeModel* m = g_crepe;
  RYK_CHECK(m != nullptr && m->tables, "CREPE model / decoder tables not loaded");
  for (int i = 0; i < 7; ++i) RYK_CHECK(m->loaded[i], "CREPE model is missing a layer");
  RYK_CHECK(m->cout[0] <= 1024, "scale vector too short");
  const int hop = (int)(16000 * step_ms / 1000);
  RYK_CHECK(hop > 0 && n > 0, "bad step size or empty signal");
  const int F = crepe_num_frames(n, step_ms);
  cudaStream_t st = e->stream;
  if (crepe_reserve(m, F, n)) return -1;
  RYK_CUDA(cudaMemcpyAsync(m->d_audio, audio16k, sizeof(float) * n, cudaMemcpyHostToDevice, st));
  int n_out, left, right;
  same_padding(1024, 512, 4, &n_out, &left, &right);                 // 256 outputs, 254 + 254
  k_crepe_frames<<<F, 256, 0, st>>>(m->d_audio, n, hop, left, m->d_im2col);
  // block 0: 1x1 conv over the im2col rows ([F][256][512] x [512][cout])
  {
    ConvLayer L;
    L.transposed = 0; L.B = F; L.Hin = 1; L.Win = 256; L.Hout = 1; L.Wout = 256; L.C0 = 512; L.C1 = 0; L.Cout = m->cout[0];
    L.KH = 1; L.KW = 1; L.SH = 1; L.SW = 1; L.PH = 0; L.PW = 0; L.act = ACT_RELU;
    L.in0 = m->d_im2col; L.in_dtype = DT_F32; L.out = m->d_conv[0]; L.out_dtype = DT_F32;
    L.w_direct = m->d_w[0]; L.scale = m->d_ones; L.shift = m->d_bias[0];
    if (conv_direct_run(L, st)) return -1;
  }
  int W = 256;
  for (int l = 0; l < 6; ++l) {
    const int Wo = W / 2;
    if (l < 5) {
      int nl, pl, pr; same_padding(Wo, kCrepeWidths[l + 1], kCrepeStrides[l + 1], &nl, &pl, &pr);
      k_crepe_bn_pool<<<296, 256, 0, st>>>(m->d_conv[l], F, W, m->cout[l], m->d_bn_a[l], m->d_bn_c[l], pl, pr, m->d_in[l + 1]);
      if (crepe_conv(e, m, l + 1, m->d_in[l + 1], F, Wo + pl + pr, m->cout[l], kCrepeWidths[l + 1], 1, nl, m->d_conv[l + 1], st)) return -1;
      W = nl;
    } else {
      k_crepe_bn_pool<<<296, 256, 0, st>>>(m->d_conv[l], F, W, m->cout[l], m->d_bn_a[l], m->d_bn_c[l], 0, 0, m->d_flat);   // [F][4][C] = time-major flatten
    }
  }
  {                                                                   // Dense(360): 1x1 conv over [F][1][64 m]
    ConvLayer L;
    L.transposed = 0; L.B = F; L.Hin = 1; L.Win = 1; L.Hout = 1; L.Wout = 1; L.C0 = 4 * m->cout[5]; L.C1 = 0; L.Cout = kCrepeBins;
    L.KH = 1; L.KW = 1; L.SH = 1; L.SW = 1; L.PH = 0; L.PW = 0; L.act = ACT_NONE;
    L.in0 = m->d_flat; L.in_dtype = DT_F32; L.out = m->d_logit; L.out_dtype = DT_F32;
    L.w_direct = m->d_dense_w; L.scale = m->d_ones; L.shift = m->d_dense_b;
    if (conv_direct_run(L, st)) return -1;
  }
  k_crepe_sigmoid<<<F, 128, 0, st>>>(m->d_logit, m->d_act, m->d_conf, m->d_obs);
  k_crepe_decode<<<1, 384, 0, st>>>(m->d_act, m->d_conf, m->d_obs, F, m->d_log_trans, m->d_cents, m->h_log_start, m->h_log_emit[0], m->h_log_emit[1],
                                   m->d_lattice, m->d_path, m->d_vlat, m->d_f0, m->d_voicing);
  RYK_CUDA(cudaGetLastError());
  e->launches += 12;
  if (f0) RYK_CUDA(cudaMemcpyAsync(f0, m->d_f0, sizeof(double) * F, cudaMemcpyDeviceToHost, st));
  if (confidence) RYK_CUDA(cudaMemcpyAsync(confidence, m->d_conf, sizeof(float) * F, cudaMemcpyDeviceToHost, st));
  if (voicing) RYK_CUDA(cudaMemcpyAsync(voicing, m->d_voicing, sizeof(int) * F, cudaMemcpyDeviceToHost, st));
  if (activation) RYK_CUDA(cudaMemcpyAsync(activation, m->d_act, sizeof(float) * (size_t)F * kCrepeBins, cudaMemcpyDeviceToHost, st));
  if (path_out) RYK_CUDA(cudaMemcpyAsync(path_out, m->d_path, sizeof(int) * F, cudaMemcpyDeviceToHost, st));
  RYK_CUDA(cudaStreamSynchronize(st));
  return 0;
}

}  // namespace ryk
