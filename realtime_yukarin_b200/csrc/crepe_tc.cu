// crepe_tc.cu -- the CREPE convolutions (conv layers 1..6, every capacity, any frame count) on the H100's tensor cores with
// error-compensated 3xTF32, for sessions in precision mode 1.
//
// Why 3xTF32: the session decodes CREPE with a per-frame arg-max over 360 sigmoid outputs and a Viterbi path over them.  FP16 or
// plain TF32 operands (10-bit mantissa) move those maxima.  Each FP32 operand x is split into hi = tf32(x) and lo = tf32(x - hi);
// the product is accumulated as lo_a * hi_b + hi_a * lo_b + hi_a * hi_b in FP32, which keeps about FP32 accuracy (the dropped
// lo_a * lo_b term is ~2^-22 relative).
//
// Every layer is one implicit GEMM  y[m][n] = ReLU(bias[n] + sum_k A[m][k] B[k][n]):
//   layer 1 (k512, stride 4): A = the im2col rows k_crepe_frames writes, [F * 256][512];
//   layers 2..6 (k64, stride 1): output pixel m = (f, w) reads the zero-framed input [F][W + pad][Cin] at f * (W + pad) * Cin + w * Cin,
//   and its K = 64 * Cin operands (tap, channel) are contiguous there, so A[m][k] = x[f * fstride + w * Cin + k] with no gather;
//   B = the [tap][Cin][Cout] FP32 weights the model already holds (the same matrix conv_direct reads).
// CTA tile 64 x BN x 32 (BN = 64, 32 or 16, the largest that divides Cout; Cout is 16 at tiny capacity), 4 warps of 32 x BN/2, each
// issuing mma.sync.m16n8k8 TF32.  Operands stream through a two-stage cp.async ring in shared memory (out-of-range rows zero-filled).
// The hi / lo split is made in registers as each fragment is loaded from shared memory: 2 cvt.rna.tf32 + 1 FADD per operand element
// per use, no extra memory traffic and no second copy of the weights or activations.  The cost is ALU work next to three MMAs per
// operand pair.
// The tensor cores' FP32 accumulation does not round like an FP32 add, and its error grows with the length of the sum (K is up to
// 65536 here): each 32-wide K tile is therefore summed into a fresh register tile on the tensor cores and added to the running
// accumulator with an ordinary FP32 add.
// Layers with few output tiles split K over up to 32 CTAs; each split writes its FP32 partial tile to a workspace and a second kernel
// adds the partials in split order, then bias and ReLU.  No atomics: results are bitwise reproducible.
#include <stdint.h>

#include "crepe_tc.h"

namespace ryk {

namespace {

constexpr int kBM = 64, kBK = 32, kThreads = 128, kNumSms = 132;
constexpr int kAStride = kBK + 4;      // floats per A row in shared memory (conflict-free fragment reads)

__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = to_tf32(x);
  lo = to_tf32(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma_tf32(float* c, const uint32_t* a, const uint32_t* b) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(s), "l"(gmem), "r"(valid ? 16 : 0));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }

template <int BN>
__global__ void __launch_bounds__(kThreads) k_crepe_tc(CrepeGemm g, int kit_per_split, float* __restrict__ ws) {
  constexpr int BS = BN + 8;                   // floats per B row in shared memory
  constexpr int NT = BN / 16;                  // n8 tiles per warp (warp tile 32 x BN/2)
  __shared__ __align__(16) float As[2][kBM * kAStride];
  __shared__ __align__(16) float Bs[2][kBK * BS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gq = lane >> 2, tq = lane & 3;
  const int wm0 = (warp >> 1) * 32, wn0 = (warp & 1) * (BN / 2);
  const int m0 = blockIdx.x * kBM, n0 = blockIdx.y * BN;
  const int kit_total = g.K / kBK;
  const int kit0 = blockIdx.z * kit_per_split;
  const int kit1 = min(kit_total, kit0 + kit_per_split);

  // per-thread A rows (4 float4 per thread) and B columns (BN / 16 float4 per thread), fixed over the K loop
  const float* a_src[4]; bool a_ok[4]; int a_dst[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int idx = tid + j * kThreads, row = idx >> 3, c4 = idx & 7, m = m0 + row;
    a_ok[j] = m < g.M;
    const int mm = a_ok[j] ? m : 0;
    a_src[j] = g.x + (long long)(mm / g.W) * g.fstride + (long long)(mm % g.W) * g.wstep + c4 * 4;
    a_dst[j] = row * kAStride + c4 * 4;
  }
  auto load_stage = [&](int stage, int kit) {
    const int k0 = kit * kBK;
#pragma unroll
    for (int j = 0; j < 4; ++j) cp_async16(&As[stage][a_dst[j]], a_src[j] + k0, a_ok[j]);      // rows past M read row 0, zero-filled
#pragma unroll
    for (int j = 0; j < BN / 16; ++j) {
      const int idx = tid + j * kThreads, kr = idx / (BN / 4), c4 = idx % (BN / 4), n = n0 + c4 * 4;
      const bool ok = n < g.N;
      cp_async16(&Bs[stage][kr * BS + c4 * 4], g.w + (long long)(k0 + kr) * g.N + (ok ? n : 0), ok);
    }
    cp_async_commit();
  };

  float acc[2][NT][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int r = 0; r < 4; ++r) acc[i][j][r] = 0.f;

  if (kit0 < kit1) load_stage(0, kit0);
  for (int kit = kit0; kit < kit1; ++kit) {
    const int st = (kit - kit0) & 1;
    if (kit + 1 < kit1) { load_stage(st ^ 1, kit + 1); cp_async_wait<1>(); }
    else cp_async_wait<0>();
    __syncthreads();
    const float* as = As[st];
    const float* bs = Bs[st];
    float part[2][NT][4];                      // this K tile's sum on the tensor cores, added to acc with FP32 FADDs below
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int r = 0; r < 4; ++r) part[i][j][r] = 0.f;
#pragma unroll
    for (int kk = 0; kk < kBK; kk += 8) {
      uint32_t ah[2][4], al[2][4];
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float* p = as + (wm0 + i * 16 + gq) * kAStride + kk + tq;
        split_tf32(p[0], ah[i][0], al[i][0]);
        split_tf32(p[8 * kAStride], ah[i][1], al[i][1]);
        split_tf32(p[4], ah[i][2], al[i][2]);
        split_tf32(p[8 * kAStride + 4], ah[i][3], al[i][3]);
      }
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        const float* q = bs + (kk + tq) * BS + wn0 + j * 8 + gq;
        uint32_t bh[2], bl[2];
        split_tf32(q[0], bh[0], bl[0]);
        split_tf32(q[4 * BS], bh[1], bl[1]);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          mma_tf32(part[i][j], al[i], bh);
          mma_tf32(part[i][j], ah[i], bl);
          mma_tf32(part[i][j], ah[i], bh);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j < NT; ++j)
#pragma unroll
        for (int r = 0; r < 4; ++r) acc[i][j][r] += part[i][j][r];
    __syncthreads();
  }

  // epilogue: c0 (g, 2t), c1 (g, 2t + 1), c2 (g + 8, 2t), c3 (g + 8, 2t + 1)
  const bool direct = gridDim.z == 1;
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      const int n = n0 + wn0 + j * 8 + 2 * tq;
      if (n >= g.N) continue;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = m0 + wm0 + i * 16 + gq + 8 * h;
        if (m >= g.M) continue;
        const float v0 = acc[i][j][2 * h], v1 = acc[i][j][2 * h + 1];
        if (direct) {
          float2 o = make_float2(fmaxf(v0 + g.bias[n], 0.f), fmaxf(v1 + g.bias[n + 1], 0.f));
          *reinterpret_cast<float2*>(g.y + (long long)m * g.N + n) = o;
        } else {
          *reinterpret_cast<float2*>(ws + ((long long)blockIdx.z * g.M + m) * g.N + n) = make_float2(v0, v1);
        }
      }
    }
}

// y = ReLU(bias + sum of the S partials in split order)
__global__ void k_crepe_tc_reduce(const float* __restrict__ ws, int S, long long MN, int N, const float* __restrict__ bias, float* __restrict__ y) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < MN; i += (long long)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int z = 0; z < S; ++z) s += ws[z * MN + i];
    y[i] = fmaxf(s + bias[i % N], 0.f);
  }
}

int pick_bn(int N) { return N % 64 == 0 ? 64 : N % 32 == 0 ? 32 : 16; }

// split-K factor and K iterations per split: about 4 CTAs per SM, at least 8 K iterations (256 K) per split, at most 32 splits
void plan_split(int M, int K, int N, int* S, int* kit_per_split) {
  const int tiles = ((M + kBM - 1) / kBM) * ((N + pick_bn(N) - 1) / pick_bn(N));
  const int kit = K / kBK;
  int s = (4 * kNumSms + tiles - 1) / tiles;
  if (s > kit / 8) s = kit / 8;
  if (s > 32) s = 32;
  if (s < 1) s = 1;
  const int per = (kit + s - 1) / s;
  *kit_per_split = per;
  *S = (kit + per - 1) / per;
}

}  // namespace

size_t crepe_tc_ws_floats(int M, int K, int N) {
  int S, per;
  plan_split(M, K, N, &S, &per);
  return S > 1 ? (size_t)S * M * N : 0;
}

int crepe_tc_run(const CrepeGemm& g, float* ws, cudaStream_t st) {
  RYK_CHECK(g.M > 0 && g.N % 16 == 0 && g.K % kBK == 0 && g.wstep % 4 == 0 && g.fstride % 4 == 0,
            "CREPE tensor-core conv: Cout must be a multiple of 16, K of 32 and the row offsets of 4 floats");
  int S, per;
  plan_split(g.M, g.K, g.N, &S, &per);
  RYK_CHECK(S == 1 || ws != nullptr, "CREPE tensor-core conv: split-K workspace missing");
  const int bn = pick_bn(g.N);
  const dim3 grid((g.M + kBM - 1) / kBM, (g.N + bn - 1) / bn, S);
  if (bn == 64) k_crepe_tc<64><<<grid, kThreads, 0, st>>>(g, per, ws);
  else if (bn == 32) k_crepe_tc<32><<<grid, kThreads, 0, st>>>(g, per, ws);
  else k_crepe_tc<16><<<grid, kThreads, 0, st>>>(g, per, ws);
  if (S > 1) {
    const long long MN = (long long)g.M * g.N;
    int blocks = (int)((MN + 255) / 256); if (blocks > 4 * kNumSms) blocks = 4 * kNumSms;
    k_crepe_tc_reduce<<<blocks, 256, 0, st>>>(ws, S, MN, g.N, g.bias, g.y);
  }
  RYK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace ryk
