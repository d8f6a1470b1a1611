// conv_direct.cu -- FP32 CUDA-core implicit-GEMM convolution / transposed convolution over NHWC
// activations with fused folded-BN scale/shift + LeakyReLU/ReLU epilogue and skip-concat by pointer.
//
// Role on the hot path (SURVEY rows a10 / a13, components H and I):
//   * every layer of the stage-1 1-D U-Net (0.55 GFLOP, latency bound, M <= 192 pixels per layer);
//   * the first (Cin = 1) and last (Cout = 1) 3x3 layers of the stage-2 2-D U-Net, whose GEMM shape
//     has nothing for a tensor core to chew on;
//   * all layers when the engine runs in FP32 "bisect" precision (the numerics reference for the
//     wgmma path in conv_tc.cu).
// Tiling: 64 output pixels x 64 output channels per CTA, 16-channel K steps through shared memory,
// 4x4 register micro-tiles (classic SGEMM shape).  Transposed convs are evaluated per output-parity
// class so that every pixel of a tile shares the same set of contributing taps.
#include "conv.h"

namespace ryk {

template <typename T> __device__ inline float ld_act(const T* p);
template <> __device__ inline float ld_act<float>(const float* p) { return *p; }
template <> __device__ inline float ld_act<__half>(const __half* p) { return __half2float(*p); }
template <typename T> __device__ inline void st_act(T* p, float v);
template <> __device__ inline void st_act<float>(float* p, float v) { *p = v; }
template <> __device__ inline void st_act<__half>(__half* p, float v) { *p = __float2half_rn(v); }

struct DirectParams {
  int transposed, B, Hin, Win, Hout, Wout, C0, C1, Cout, KH, KW, SH, SW, PH, PW, act;
  int classH, classW;            // transposed: SH, SW ; else 1, 1
  int Hc, Wc;                    // class-local output grid
  const void* in0; const void* in1; void* out;
  const float* w; const float* scale; const float* shift;
};

template <typename TIn, typename TOut>
__global__ void __launch_bounds__(256) k_conv_direct(DirectParams p) {
  constexpr int BM = 64, BN = 64, BK = 16;
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  __shared__ int pix_b[BM], pix_y[BM], pix_x[BM];
  const int Cin = p.C0 + p.C1;
  const int cls = blockIdx.z;
  const int py = cls / p.classW, px = cls % p.classW;
  const int npix = p.B * p.Hc * p.Wc;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int tid = threadIdx.x, ty = tid >> 4, tx = tid & 15;
  if (tid < BM) {
    int q = m0 + tid;
    if (q < npix) {
      int b = q / (p.Hc * p.Wc);
      int r = q - b * p.Hc * p.Wc;
      int my = r / p.Wc, mx = r - my * p.Wc;
      pix_b[tid] = b; pix_y[tid] = my * p.classH + py; pix_x[tid] = mx * p.classW + px;
    } else {
      pix_b[tid] = -1; pix_y[tid] = 0; pix_x[tid] = 0;
    }
  }
  __syncthreads();
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int a_pix = tid >> 2, a_c4 = (tid & 3) * 4;     // A loader: pixel, first of 4 channels
  const int b_k = tid >> 4, b_n4 = (tid & 15) * 4;      // B loader
  const TIn* in0 = (const TIn*)p.in0;
  const TIn* in1 = (const TIn*)p.in1;

  for (int ky = 0; ky < p.KH; ++ky) {
    if (p.transposed && ((py + p.PH - ky) % p.SH + p.SH) % p.SH != 0) continue;
    for (int kx = 0; kx < p.KW; ++kx) {
      if (p.transposed && ((px + p.PW - kx) % p.SW + p.SW) % p.SW != 0) continue;
      // input coordinate of this thread's A pixel for this tap
      long long abase = -1;
      {
        int b = pix_b[a_pix];
        if (b >= 0) {
          int iy, ix;
          if (!p.transposed) { iy = pix_y[a_pix] * p.SH - p.PH + ky; ix = pix_x[a_pix] * p.SW - p.PW + kx; }
          else { iy = (pix_y[a_pix] + p.PH - ky) / p.SH; ix = (pix_x[a_pix] + p.PW - kx) / p.SW; }
          if (iy >= 0 && iy < p.Hin && ix >= 0 && ix < p.Win) abase = ((long long)(b * p.Hin + iy) * p.Win + ix);
        }
      }
      const float* wtap = p.w + (size_t)(ky * p.KW + kx) * Cin * p.Cout;
      for (int c0 = 0; c0 < Cin; c0 += BK) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          int c = c0 + a_c4 + j;
          float v = 0.f;
          if (abase >= 0 && c < Cin) {
            if (c < p.C0) v = ld_act<TIn>(in0 + abase * p.C0 + c);
            else v = ld_act<TIn>(in1 + abase * p.C1 + (c - p.C0));
          }
          As[a_c4 + j][a_pix] = v;
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          int c = c0 + b_k, n = n0 + b_n4 + j;
          Bs[b_k][b_n4 + j] = (c < Cin && n < p.Cout) ? wtap[(size_t)c * p.Cout + n] : 0.f;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
          float a[4], b[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) a[i] = As[k][ty * 4 + i];
#pragma unroll
          for (int j = 0; j < 4; ++j) b[j] = Bs[k][tx * 4 + j];
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
      }
    }
  }
  TOut* out = (TOut*)p.out;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    int pl = ty * 4 + i;
    int b = pix_b[pl];
    if (b < 0) continue;
    size_t obase = ((size_t)(b * p.Hout + pix_y[pl]) * p.Wout + pix_x[pl]) * p.Cout;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int n = n0 + tx * 4 + j;
      if (n >= p.Cout) continue;
      float v = acc[i][j] * p.scale[n] + p.shift[n];
      if (p.act == ACT_LEAKY) v = v > 0.f ? v : 0.2f * v;
      else if (p.act == ACT_RELU) v = v > 0.f ? v : 0.f;
      st_act<TOut>(out + obase + n, v);
    }
  }
}

static int conv_direct_generic(const ConvLayer& L, cudaStream_t st) {
  DirectParams p;
  p.transposed = L.transposed; p.B = L.B; p.Hin = L.Hin; p.Win = L.Win; p.Hout = L.Hout; p.Wout = L.Wout;
  p.C0 = L.C0; p.C1 = L.C1; p.Cout = L.Cout; p.KH = L.KH; p.KW = L.KW; p.SH = L.SH; p.SW = L.SW; p.PH = L.PH; p.PW = L.PW;
  p.act = L.act;
  p.classH = L.transposed ? L.SH : 1; p.classW = L.transposed ? L.SW : 1;
  RYK_CHECK(L.Hout % p.classH == 0 && L.Wout % p.classW == 0, "transposed conv output must be a multiple of the stride");
  p.Hc = L.Hout / p.classH; p.Wc = L.Wout / p.classW;
  p.in0 = L.in0; p.in1 = L.in1; p.out = L.out; p.w = L.wt.w[0]; p.scale = L.wt.scale[0]; p.shift = L.wt.shift[0];
  RYK_CHECK(p.w && p.scale && p.shift && L.in0 && L.out, "direct conv layer is missing a device pointer");
  int npix = L.B * p.Hc * p.Wc;
  dim3 grid((npix + 63) / 64, (L.Cout + 63) / 64, p.classH * p.classW);
  if (L.in_dtype == DT_F32 && L.out_dtype == DT_F32) k_conv_direct<float, float><<<grid, 256, 0, st>>>(p);
  else if (L.in_dtype == DT_F32 && L.out_dtype == DT_F16) k_conv_direct<float, __half><<<grid, 256, 0, st>>>(p);
  else if (L.in_dtype == DT_F16 && L.out_dtype == DT_F16) k_conv_direct<__half, __half><<<grid, 256, 0, st>>>(p);
  else k_conv_direct<__half, float><<<grid, 256, 0, st>>>(p);
  RYK_CUDA(cudaGetLastError());
  return 0;
}


// ---- stage-2 edge layers -----------------------------------------------------------------------
// The first (Cin = 1) and last (Cout = 1) 3x3 layers of the 2-D U-Net are pure bandwidth problems
// (25 MB written / 50 MB read at 384x512); the generic 64x64 tile above would waste 16-64x of its math on
// them, so they get dedicated kernels: coalesced 16-byte accesses, weights in shared memory.

// Cin = 1, fp32 input -> Cout (multiple of 8, <= 64) channels.  Block = 32 pixels (x) x Cout/8 channel groups, walking
// kRows rows of the image with a 3-row register window: every input value is loaded once per thread column, every
// store is a full 16-byte piece of a 128-byte pixel (4 pixels per warp instruction), no integer divisions.
// Weights [9][1][Cout] of batch item b's voice.  The row blocks [skip_b0, skip_b0 + skip_nb) (a padded tail; ConvLayer::skip_y0) are
// not launched.
template <typename TOut>
__global__ void __launch_bounds__(256) k_conv3x3_cin1(const float* __restrict__ in, const __grid_constant__ LayerWeights wt, int act,
                                                     int B, int H, int W, int Cout, int skip_b0, int skip_nb, TOut* __restrict__ out) {
  constexpr int kRows = kCin1Rows;
  const int groups = Cout >> 3;                   // blockDim.x = 32 * groups  (<= 256)
  const int g = threadIdx.x % groups, xl = threadIdx.x / groups;
  const int x = blockIdx.x * 32 + xl;
  const int y0 = (blockIdx.y + (blockIdx.y >= skip_b0 ? skip_nb : 0)) * kRows;
  const int b = blockIdx.z;
  const int voice = item_voice(wt, b);
  const float* __restrict__ w = wt.w[voice];
  const float* __restrict__ scale = wt.scale[voice];
  const float* __restrict__ shift = wt.shift[voice];
  float wr[9][8], sc[8], sh[8];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int j = 0; j < 8; ++j) wr[t][j] = __ldg(w + t * Cout + g * 8 + j);
#pragma unroll
  for (int j = 0; j < 8; ++j) { sc[j] = __ldg(scale + g * 8 + j); sh[j] = __ldg(shift + g * 8 + j); }
  if (x >= W) return;
  const float* base = in + (size_t)b * H * W;
  auto ld = [&](int yy, int xx) -> float { return (yy >= 0 && yy < H && xx >= 0 && xx < W) ? __ldg(base + (size_t)yy * W + xx) : 0.f; };
  float r0[3], r1[3], r2[3];
#pragma unroll
  for (int d = 0; d < 3; ++d) { r0[d] = ld(y0 - 1, x + d - 1); r1[d] = ld(y0, x + d - 1); }
  for (int yy = 0; yy < kRows; ++yy) {
    const int y = y0 + yy;
    if (y >= H) break;
#pragma unroll
    for (int d = 0; d < 3; ++d) r2[d] = ld(y + 1, x + d - 1);
    float o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float a = 0.f;
#pragma unroll
      for (int d = 0; d < 3; ++d) { a = fmaf(r0[d], wr[d][j], a); a = fmaf(r1[d], wr[3 + d][j], a); a = fmaf(r2[d], wr[6 + d][j], a); }
      a = a * sc[j] + sh[j];
      if (act == ACT_LEAKY) a = a > 0.f ? a : 0.2f * a; else if (act == ACT_RELU) a = fmaxf(a, 0.f);
      o[j] = a;
    }
    TOut* dst = out + (((size_t)b * H + y) * W + x) * Cout + g * 8;
    if constexpr (sizeof(TOut) == 2) {
      __half2 h0 = __floats2half2_rn(o[0], o[1]), h1 = __floats2half2_rn(o[2], o[3]), h2 = __floats2half2_rn(o[4], o[5]), h3 = __floats2half2_rn(o[6], o[7]);
      *reinterpret_cast<uint4*>(dst) = make_uint4(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1),
                                                  *reinterpret_cast<uint32_t*>(&h2), *reinterpret_cast<uint32_t*>(&h3));
    } else {
      *reinterpret_cast<float4*>(dst) = make_float4(o[0], o[1], o[2], o[3]);
      *reinterpret_cast<float4*>(dst + 4) = make_float4(o[4], o[5], o[6], o[7]);
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) { r0[d] = r1[d]; r1[d] = r2[d]; }
  }
}

// Cout = 1 from two fp16 sources of 64 channels each (skip concat) -> fp32.  One warp = 8 consecutive pixels of a row:
// lanes 0-15 own 4 channels each of source 0, lanes 16-31 of source 1; the 3 x 10 input pixels are loaded once
// (30 independent 8-byte loads in flight per lane) and feed all 8 outputs, which are then reduced across the warp.
// Computes output rows y0 .. y0 + gridDim.y - 1, with the weights [9][128][1] and scalar scale / shift of batch item b's voice.
__global__ void __launch_bounds__(256) k_conv3x3_cout1_h(const __half* __restrict__ in0, const __half* __restrict__ in1,
                                                        const __grid_constant__ LayerWeights weights, int act,
                                                        int B, int H, int W, int y0, float* __restrict__ out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int x0 = (blockIdx.x * 8 + warp) * 8;          // 8 warps x 8 pixels = 64 pixels of a row per block
  const int y = y0 + blockIdx.y, b = blockIdx.z;
  const int voice = item_voice(weights, b);
  const float* __restrict__ w = weights.w[voice];
  const float scale = weights.host_scale[voice], shift = weights.host_shift[voice];
  if (x0 >= W) return;
  const __half* src = lane < 16 ? in0 : in1;
  const int c = (lane & 15) * 4;
  float wt[9][4];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int j = 0; j < 4; ++j) wt[t][j] = __ldg(w + t * 128 + (lane < 16 ? 0 : 64) + c + j);
  float acc[8];
#pragma unroll
  for (int q = 0; q < 8; ++q) acc[q] = 0.f;
#pragma unroll
  for (int dy = 0; dy < 3; ++dy) {
    const int iy = y + dy - 1;
    if (iy < 0 || iy >= H) continue;
    uint2 raw[10];
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      const int ix = x0 + i - 1;
      raw[i] = (ix >= 0 && ix < W) ? __ldg(reinterpret_cast<const uint2*>(src + (((size_t)b * H + iy) * W + ix) * 64 + c)) : make_uint2(0u, 0u);
    }
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      const float2 f01 = __half22float2(*reinterpret_cast<__half2*>(&raw[i].x)), f23 = __half22float2(*reinterpret_cast<__half2*>(&raw[i].y));
#pragma unroll
      for (int dx = 0; dx < 3; ++dx) {
        const int q = i - dx;                    // output pixel fed by input column i through tap dx
        if (q < 0 || q >= 8) continue;
        const float* wv = wt[dy * 3 + dx];
        acc[q] = fmaf(f01.x, wv[0], acc[q]); acc[q] = fmaf(f01.y, wv[1], acc[q]);
        acc[q] = fmaf(f23.x, wv[2], acc[q]); acc[q] = fmaf(f23.y, wv[3], acc[q]);
      }
    }
  }
  // warp reduction of 8 values: fold pairs so that lane l ends up owning pixel (l & 7)
#pragma unroll
  for (int q = 0; q < 8; ++q) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[q] += __shfl_xor_sync(0xffffffffu, acc[q], o);
  }
  if (lane < 8) {
    float a = acc[0];
#pragma unroll
    for (int q = 1; q < 8; ++q) a = lane == q ? acc[q] : a;
    const int x = x0 + lane;
    if (x < W) {
      a = a * scale + shift;
      if (act == ACT_LEAKY) a = a > 0.f ? a : 0.2f * a; else if (act == ACT_RELU) a = fmaxf(a, 0.f);
      out[((size_t)b * H + y) * W + x] = a;
    }
  }
}

// Last layer of the stage-1 1-D U-Net: k3 s1 p1 over two fp16 sources of 64 channels -> Cout <= 16 channels, fp32.
// One warp per output position: lane l owns channels 4l..4l+3 of the concatenated 128 (lanes 0-15 source 0, 16-31
// source 1), 3 taps x 4 channels x Cout FMAs, warp-shuffle reduction per output channel.  (The generic 64x64x16 tile
// kernel put this layer on 6 CTAs: 39 us for 0.3 MFLOP.)
__global__ void __launch_bounds__(256) k_conv1d_k3_small(const __half* __restrict__ in0, const __half* __restrict__ in1,
                                                        const float* __restrict__ w /*[3][128][Cout]*/, const float* __restrict__ scale,
                                                        const float* __restrict__ shift, int act, int B, int W, int Cout, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int pos = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (pos >= B * W) return;
  const int b = pos / W, x = pos - b * W;
  const __half* src = lane < 16 ? in0 : in1;
  const int c = (lane & 15) * 4, cg = lane * 4;       // channel inside the source / inside the concatenation
  float xin[3][4];
#pragma unroll
  for (int t = 0; t < 3; ++t) {
    const int ix = x + t - 1;
    uint2 raw = make_uint2(0u, 0u);
    if (ix >= 0 && ix < W) raw = __ldg(reinterpret_cast<const uint2*>(src + ((size_t)b * W + ix) * 64 + c));
    const float2 f01 = __half22float2(*reinterpret_cast<__half2*>(&raw.x)), f23 = __half22float2(*reinterpret_cast<__half2*>(&raw.y));
    xin[t][0] = f01.x; xin[t][1] = f01.y; xin[t][2] = f23.x; xin[t][3] = f23.y;
  }
  float mine = 0.f;
  for (int co = 0; co < Cout; ++co) {
    float a = 0.f;
#pragma unroll
    for (int t = 0; t < 3; ++t)
#pragma unroll
      for (int j = 0; j < 4; ++j) a = fmaf(xin[t][j], __ldg(w + ((size_t)t * 128 + cg + j) * Cout + co), a);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == co) mine = a;
  }
  if (lane < Cout) {
    float a = mine * __ldg(scale + lane) + __ldg(shift + lane);
    if (act == ACT_LEAKY) a = a > 0.f ? a : 0.2f * a; else if (act == ACT_RELU) a = fmaxf(a, 0.f);
    out[(size_t)pos * Cout + lane] = a;
  }
}

__global__ void k_read2(const float* a, const float* b, float* out) { out[0] = a[0]; out[1] = b[0]; }

// the last stage-2 layer in FP16 plans (k_conv3x3_cout1_h), the one CUDA-core kernel that computes a row band
bool conv_direct_band_supported(const ConvLayer& L) {
  return !L.transposed && L.KH == 3 && L.KW == 3 && L.SH == 1 && L.SW == 1 && L.PH == 1 && L.PW == 1 && L.Cout == 1 && L.C0 == 64 &&
         L.C1 == 64 && L.in_dtype == DT_F16 && L.out_dtype == DT_F32 && L.host_scale_valid;
}

bool conv_direct_cin1(const ConvLayer& L) {
  return !L.transposed && L.KH == 3 && L.KW == 3 && L.SH == 1 && L.SW == 1 && L.PH == 1 && L.PW == 1 && L.C0 == 1 && L.C1 == 0 &&
         L.in_dtype == DT_F32 && L.Cout % 8 == 0 && L.Cout <= 64;
}

bool conv_direct_per_item_weights(const ConvLayer& L) { return conv_direct_cin1(L) || conv_direct_band_supported(L); }

int conv_direct_run(const ConvLayer& L, cudaStream_t st) {
  const bool cout1_h = conv_direct_band_supported(L);
  const bool cin1 = conv_direct_cin1(L);
  RYK_CHECK(L.n_voices == 1 || cout1_h || cin1, "of the CUDA-core kernels only the stage-2 edge layers take weights per batch item");
  RYK_CHECK(cout1_h || (L.band_y0 == 0 && L.band_y1 == 0), "of the CUDA-core kernels only the Cout = 1 3x3 kernel computes a row band");
  RYK_CHECK(cin1 || L.skip_y1 == 0, "of the CUDA-core kernels only the Cin = 1 3x3 kernel skips a padded tail");
  // dedicated kernels for the stage-2 edge layers
  if (!L.transposed && L.KH == 3 && L.KW == 3 && L.SH == 1 && L.SW == 1 && L.PH == 1 && L.PW == 1) {
    if (cin1) {
      RYK_CHECK(L.skip_y0 % kCin1Rows == 0 && L.skip_y1 % kCin1Rows == 0 && L.skip_y0 <= L.skip_y1 && L.skip_y1 <= L.Hout,
                "skipped rows are not whole row blocks of the first layer");
      const int skip_b0 = L.skip_y0 / kCin1Rows, skip_nb = (L.skip_y1 - L.skip_y0) / kCin1Rows;
      dim3 grid((L.Win + 31) / 32, (L.Hin + kCin1Rows - 1) / kCin1Rows - skip_nb, L.B);
      int threads = 32 * (L.Cout / 8);
      if (L.out_dtype == DT_F16)
        k_conv3x3_cin1<__half><<<grid, threads, 0, st>>>((const float*)L.in0, L.wt, L.act, L.B, L.Hin, L.Win, L.Cout, skip_b0, skip_nb, (__half*)L.out);
      else
        k_conv3x3_cin1<float><<<grid, threads, 0, st>>>((const float*)L.in0, L.wt, L.act, L.B, L.Hin, L.Win, L.Cout, skip_b0, skip_nb, (float*)L.out);
      RYK_CUDA(cudaGetLastError());
      return 0;
    }
    if (cout1_h) {
      dim3 blocks((L.Win + 63) / 64, layer_band_end(L) - L.band_y0, L.B);       // the layer's row band
      k_conv3x3_cout1_h<<<blocks, 256, 0, st>>>((const __half*)L.in0, (const __half*)L.in1, L.wt, L.act,
                                                L.B, L.Hin, L.Win, L.band_y0, (float*)L.out);
      RYK_CUDA(cudaGetLastError());
      return 0;
    }
  }
  if (!L.transposed && L.KH == 1 && L.KW == 3 && L.SW == 1 && L.PW == 1 && L.Hin == 1 && L.C0 == 64 && L.C1 == 64 && L.Cout <= 16 &&
      L.in_dtype == DT_F16 && L.out_dtype == DT_F32) {
    const int npos = L.B * L.Win;
    k_conv1d_k3_small<<<(npos + 7) / 8, 256, 0, st>>>((const __half*)L.in0, (const __half*)L.in1, L.wt.w[0], L.wt.scale[0], L.wt.shift[0], L.act, L.B, L.Win, L.Cout,
                                                     (float*)L.out);
    RYK_CUDA(cudaGetLastError());
    return 0;
  }
  return conv_direct_generic(L, st);
}

// ---- weight repacking ------------------------------------------------------------------------
__global__ void k_pack_direct(const float* __restrict__ w, int transposed, int Cin, int Cout, int KH, int KW, float* __restrict__ out) {
  size_t total = (size_t)KH * KW * Cin * Cout;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    int n = i % Cout; size_t r = i / Cout;
    int c = r % Cin; r /= Cin;
    int kx = r % KW; int ky = r / KW;
    size_t src = transposed ? (((size_t)c * Cout + n) * KH + ky) * KW + kx : (((size_t)n * Cin + c) * KH + ky) * KW + kx;
    out[i] = w[src];
  }
}

int pack_weights_direct(const float* d_w, int transposed, int Cin, int Cout, int KH, int KW, float* d_out, cudaStream_t st) {
  k_pack_direct<<<256, 256, 0, st>>>(d_w, transposed, Cin, Cout, KH, KW, d_out);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

// tensor-core packing: fp16, K-major rows.
//   conv  : out[n][(ky*KW+kx)*Cin + c]                                    = W[n][c][ky][kx]
//   deconv: out[cls][n][(dy*(KW/SW)+dx)*Cin + c], cls = py*SW+px          = W[c][n][ky][kx]
//           with k = 3 - 2d - parity along a k4 s2 p1 dimension and k = 0 along a k1 s1 p0 dimension (1-D nets)
__global__ void k_pack_tc(const float* __restrict__ w, int transposed, int Cin, int Cout, int KH, int KW, int SH, int SW,
                          __half* __restrict__ out) {
  size_t total = (size_t)KH * KW * Cin * Cout;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    if (!transposed) {
      size_t K = (size_t)KH * KW * Cin;
      int n = i / K; size_t k = i % K;
      int tap = k / Cin, c = k % Cin;
      int ky = tap / KW, kx = tap % KW;
      out[i] = __float2half_rn(w[(((size_t)n * Cin + c) * KH + ky) * KW + kx]);
    } else {
      int th = KH / SH, tw = KW / SW;
      size_t K = (size_t)th * tw * Cin;
      size_t per_cls = K * Cout;
      int cls = i / per_cls; size_t r = i % per_cls;
      int n = r / K; size_t k = r % K;
      int tap = k / Cin, c = k % Cin;
      int dy = tap / tw, dx = tap % tw, py = cls / SW, px = cls % SW;
      int ky = SH == 2 ? 3 - 2 * dy - py : 0, kx = SW == 2 ? 3 - 2 * dx - px : 0;
      out[i] = __float2half_rn(w[(((size_t)c * Cout + n) * KH + ky) * KW + kx]);
    }
  }
}

int pack_weights_tc(const float* d_w, int transposed, int Cin, int Cout, int KH, int KW, int SH, int SW, __half* d_out, cudaStream_t st) {
  k_pack_tc<<<512, 256, 0, st>>>(d_w, transposed, Cin, Cout, KH, KW, SH, SW, d_out);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace ryk
