// s1_fused.cu -- the whole stage-1 1-D U-Net (yukarin acoustic-feature converter, SURVEY a10: realtime_voice_conversion/
// yukarin_wrapper/voice_changer.py:36 -> AcousticConverter.convert_from_feature) as ONE kernel launch.
//
// Round 1/2 ran it as 16 layer launches + 14 split-K reduces (~200 us of launch latency for 0.55 GFLOP, 27 MB of FP16 weights).
// Here one thread-block CLUSTER walks the 16 layers:
//   * the cluster barrier (barrier.cluster, hardware, release / acquire) is the only inter-layer synchronisation -- a cluster is
//     co-scheduled by the hardware, so there is no software grid barrier that could dead-lock on a full GPU, and the kernel occupies
//     only `cluster size` SMs next to the stage-2 tensor-core kernels of the neighbouring chunks;
//   * each k4 layer is a skinny GEMM out[m][n] = sum_k A[m][k] W[n][k] (s1_map.h) on mma.sync m16n8k16 (FP16 in, FP32 accumulate:
//     same operand precision as the wgmma path it replaces; M is 3..320 rows, far below a 128-row tile);
//   * weights are pre-packed in B-fragment order, so a warp streams its share with coalesced 16-byte loads straight into the mma
//     operands, every weight byte exactly once per M slab; the blocks a CTA will need three layers later are requested into L2 with
//     cp.async.bulk.prefetch.L2, which keeps HBM busy across the layer barriers;
//   * a CTA stages the input rows of its M slab in shared memory once per layer (skip concatenation happens here) and reads A
//     fragments with ldmatrix; warps split the slab's m-tiles and, for the deep layers with 1-2 m-tiles, the K range (partial
//     accumulators are reduced through shared memory in a fixed order: deterministic);
//   * the k3 edge layers (9 -> 64 and 128 -> 9 channels) run on the CUDA cores inside the same kernel.
// Activations between layers live in the plan's HBM buffers (<= 48 KB each, L2 resident), exactly where the layered path keeps them.
#include <stdlib.h>

#include <vector>

#include "conv.h"
#include "engine.h"
#include "s1_map.h"
#include "tc_ptx.cuh"
#include "unet.h"

namespace ryk {

struct S1LayerP {
  const __half* in0; const __half* in1; __half* out;
  const uint4* w;                       // fragment-packed weights (s1_w_dst)
  const float* scale; const float* shift;
  int transposed, Win, C0, C1, Cout, act;
  int lgCin;                             // Cin = C0 + C1 is a power of two
  S1Cut cut;                             // s1_cut(geometry, cluster size), computed on the host
};
struct S1Params {
  S1LayerP L[14];
  // first layer: conv k3 s1 p1 on the FP32 input, last layer: conv k3 s1 p1 to the FP32 output
  const float* x; const float* w0; const float* sc0; const float* sh0; __half* enc0; int in_ch, base, act0;
  const __half* yin0; const __half* yin1; const float* w15; const float* sc15; const float* sh15; float* y; int yc0, yc1, out_ch, act15;
  int W;
};

__device__ __forceinline__ uint32_t cluster_size() { uint32_t r; asm volatile("mov.u32 %0, %%cluster_nctaid.x;" : "=r"(r)); return r; }
__device__ __forceinline__ void l2_prefetch_bulk(const void* p, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
__device__ __forceinline__ void cluster_arrive() { asm volatile("barrier.cluster.arrive.release;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.acquire;" ::: "memory"); }
__device__ __forceinline__ uint4 ldcg_u4(const void* p) { return __ldcg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&a)[4], uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];" : "=r"(a[0]), "=r"(a[1]), "=r"(a[2]), "=r"(a[3]) : "r"(addr));
}
__device__ __forceinline__ void mma_16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3]) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ float apply_act(float v, int act) {
  if (act == ACT_LEAKY) return v > 0.f ? v : 0.2f * v;
  if (act == ACT_RELU) return fmaxf(v, 0.f);
  return v;
}

// Ask L2 for the weight blocks this CTA will read in layer L (one bulk prefetch per task, issued by one thread each).
__device__ __forceinline__ void s1_prefetch_layer(const S1LayerP& L, int rank, int nc) {
  const S1Geom g{L.transposed, L.Win, L.C0 + L.C1, L.Cout};
  const S1Cut c = L.cut;
  const int np = rank / c.MS, ntasks = s1_tasks(g);
  const uint32_t bytes = (uint32_t)s1_task_halfs(g) * 2;
  const int task = np + (int)threadIdx.x * c.NP;
  if (task < ntasks) l2_prefetch_bulk(reinterpret_cast<const char*>(L.w) + (size_t)task * bytes, bytes);
}

// two k-tile pairs (kp, kp + 1) x two 8-column tiles of B fragments of one lane
struct S1BChunk { uint4 v[2][2]; };
__device__ __forceinline__ void s1_load_b(S1BChunk& b, const uint4* __restrict__ wt, int kp, int lane) {
#pragma unroll
  for (int q = 0; q < 2; ++q)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) b.v[q][nt] = __ldg(wt + ((size_t)(kp + q) * 2 + nt) * 32 + lane);
}

// acc[tile][nt][4] += A(rows of the two m-tiles, k-tile pairs kp, kp + 1) x B chunk
__device__ __forceinline__ void s1_mma_chunk(float (&acc)[2][2][4], const S1BChunk& b, int kp, const S1Geom& g, int lgCin, int cls, int RS, int px0,
                                             int mA, int mB, int kofs, uint32_t act_addr) {
#pragma unroll
  for (int q = 0; q < 2; ++q) {
#pragma unroll
    for (int kt = 0; kt < 2; ++kt) {
      const int k0 = (kp + q) * 32 + kt * 16;
      const int j = k0 >> lgCin, ch = (k0 & (g.Cin - 1)) + kofs;
      const int rowA = s1_in_px(g, cls, mA, j) - px0, rowB = s1_in_px(g, cls, mB, j) - px0;
      uint32_t aA[4], aB[4];
      ldmatrix_x4(aA, act_addr + (uint32_t)(rowA * RS + ch) * 2u);
      ldmatrix_x4(aB, act_addr + (uint32_t)(rowB * RS + ch) * 2u);
      const uint32_t b00 = kt ? b.v[q][0].z : b.v[q][0].x, b01 = kt ? b.v[q][0].w : b.v[q][0].y;
      const uint32_t b10 = kt ? b.v[q][1].z : b.v[q][1].x, b11 = kt ? b.v[q][1].w : b.v[q][1].y;
      mma_16816(acc[0][0], aA, b00, b01);
      mma_16816(acc[0][1], aA, b10, b11);
      mma_16816(acc[1][0], aB, b00, b01);
      mma_16816(acc[1][1], aB, b10, b11);
    }
  }
}

// this warp's first weight chunk of an upcoming (layer, task, pass): loaded ahead so that its latency hides behind the reduction /
// epilogue of the current task or behind the cluster barrier and the staging of the next layer
struct S1Carry { S1BChunk b; bool valid; };

__device__ __forceinline__ void s1_first_of_layer(const S1LayerP& L, int rank, int nc, int warp, int lane, S1Carry& carry) {
  const S1Geom g{L.transposed, L.Win, L.C0 + L.C1, L.Cout};
  const S1Cut c = L.cut;
  const int M = s1_M(g), KP = s1_K(g) / 32;
  const int mslab = rank % c.MS, np = rank / c.MS;
  const int m0 = mslab * c.slab, m1 = min(M, m0 + c.slab);
  carry.valid = false;
  if (m0 >= M || np >= s1_tasks(g)) return;
  const int mg = warp / c.ks, kpart = warp - mg * c.ks;
  const int mt_slab = (m1 - m0 + 15) / 16;
  if (!(warp < c.ms * c.ks && mg < mt_slab)) return;
  const uint4* wt = L.w + (size_t)np * (s1_task_halfs(g) / 8);
  s1_load_b(carry.b, wt, kpart * (KP / c.ks), lane);
  carry.valid = true;
}

__device__ __forceinline__ void s1_layer(const S1LayerP& L, int rank, int nc, __half* act, float* partial, S1Carry& carry) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const S1Geom g{L.transposed, L.Win, L.C0 + L.C1, L.Cout};
  const S1Cut c = L.cut;
  const int M = s1_M(g), K = s1_K(g), KP = K / 32, NG = g.Cout / 16;
  const int mslab = rank % c.MS, np = rank / c.MS;
  const int m0 = mslab * c.slab, m1 = min(M, m0 + c.slab);
  if (m0 >= M) { carry.valid = false; return; }          // CTA-uniform: this slab is empty
  const int px0 = s1_px0(g, m0), RS = c.RS;
  // ---- stage the slab's input rows (zero rows = padding), concatenating the skip tensor; four 16-byte loads in flight per thread ----
  {
    const int nrows = s1_rows_for(g, m1 - m0), lgv = L.lgCin - 3, nv = nrows << lgv;          // Cin / 8 16-byte vectors per row
    for (int i0 = tid; i0 < nv; i0 += 4 * kS1Threads) {
      uint4 v[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * kS1Threads;
        v[u] = make_uint4(0u, 0u, 0u, 0u);
        if (i < nv) {
          const int r = i >> lgv, ch = (i - (r << lgv)) * 8, px = px0 + r;
          if (px >= 0 && px < L.Win)
            v[u] = ch < L.C0 ? ldcg_u4(L.in0 + (size_t)px * L.C0 + ch) : ldcg_u4(L.in1 + (size_t)px * L.C1 + (ch - L.C0));
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + u * kS1Threads;
        if (i < nv) { const int r = i >> lgv, ch = (i - (r << lgv)) * 8; *reinterpret_cast<uint4*>(act + (size_t)r * RS + ch) = v[u]; }
      }
    }
  }
  __syncthreads();
  const uint32_t act_addr = smem_u32(act);
  const int mg = warp / c.ks, kpart = warp - mg * c.ks;
  const bool active = warp < c.ms * c.ks;
  const int kp_per = KP / c.ks, kp_lo = kpart * kp_per, kp_hi = kp_lo + kp_per;
  const int rows = m1 - m0, mt_slab = (rows + 15) / 16;
  const int npass = (mt_slab + 2 * c.ms - 1) / (2 * c.ms);
  const int ntasks = s1_tasks(g);
  const size_t task_u4 = s1_task_halfs(g) / 8;
  const int lrow = s1_ldm_row(lane), kofs = s1_ldm_kofs(lane);
  for (int task = np; task < ntasks; task += c.NP) {
    const int cls = task / NG, ng = task - cls * NG;
    const uint4* __restrict__ wt = L.w + (size_t)task * task_u4;
    for (int p = 0; p < npass; ++p) {
      const int tA = mg + c.ms * (2 * p), tB = tA + c.ms;
      const bool work = active && tA < mt_slab;
      float acc[2][2][4];
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int nt = 0; nt < 2; ++nt)
#pragma unroll
          for (int r = 0; r < 4; ++r) acc[i][nt][r] = 0.f;
      if (work) {
        const int mA = m0 + min(tA * 16 + lrow, rows - 1), mB = m0 + min(tB * 16 + lrow, rows - 1);
        S1BChunk b0 = carry.b, b1;
        if (!carry.valid) s1_load_b(b0, wt, kp_lo, lane);
        for (int kp = kp_lo; kp < kp_hi; kp += 4) {
          const bool more = kp + 2 < kp_hi;
          if (more) s1_load_b(b1, wt, kp + 2, lane);
          s1_mma_chunk(acc, b0, kp, g, L.lgCin, cls, RS, px0, mA, mB, kofs, act_addr);
          if (more) {
            if (kp + 4 < kp_hi) s1_load_b(b0, wt, kp + 4, lane);
            s1_mma_chunk(acc, b1, kp + 2, g, L.lgCin, cls, RS, px0, mA, mB, kofs, act_addr);
          }
        }
      }
      // first chunk of this warp's next (task, pass) of the layer, requested before the reduction / epilogue below
      {
        int ntask = task, pn = p + 1;
        if (pn >= npass) { pn = 0; ntask = task + c.NP; }
        carry.valid = false;
        if (ntask < ntasks && active && mg + c.ms * (2 * pn) < mt_slab) {
          s1_load_b(carry.b, L.w + (size_t)ntask * task_u4, kp_lo, lane);
          carry.valid = true;
        }
      }
      if (c.ks > 1) {                                      // CTA-uniform: split-K partials reduced and stored by ALL threads
        if (work) {
#pragma unroll
          for (int i = 0; i < 2; ++i)
#pragma unroll
            for (int nt = 0; nt < 2; ++nt)
#pragma unroll
              for (int r = 0; r < 4; ++r) partial[((size_t)warp * 16 + (i * 2 + nt) * 4 + r) * 32 + lane] = acc[i][nt][r];
        }
        __syncthreads();
        for (int e = tid; e < c.ms * 256; e += kS1Threads) {
          const int mgp = e >> 8, idx2 = (e >> 5) & 7, ln = e & 31;       // idx2 = (i * 2 + nt) * 2 + rr
          const int i = idx2 >> 2, nt = (idx2 >> 1) & 1, rr = idx2 & 1;
          const int tile = mgp + c.ms * (2 * p + i);
          const int mrel = tile * 16 + s1_c_row(ln, rr * 2);
          if (mrel < rows) {
            const float* src = partial + ((size_t)(mgp * c.ks) * 16 + (i * 2 + nt) * 4 + rr * 2) * 32 + ln;
            float v0 = 0.f, v1 = 0.f;
#pragma unroll 4
            for (int kq = 0; kq < c.ks; ++kq) { v0 += src[(size_t)kq * 512]; v1 += src[(size_t)kq * 512 + 32]; }   // fixed order
            const int n = ng * 16 + nt * 8 + s1_c_col(ln, 0);
            const int opx = s1_out_px(g, cls, m0 + mrel);
            v0 = apply_act(fmaf(v0, __ldg(L.scale + n), __ldg(L.shift + n)), L.act);
            v1 = apply_act(fmaf(v1, __ldg(L.scale + n + 1), __ldg(L.shift + n + 1)), L.act);
            *reinterpret_cast<__half2*>(L.out + (size_t)opx * g.Cout + n) = __floats2half2_rn(v0, v1);
          }
        }
        __syncthreads();                                   // the partial buffer is rewritten by the next pass / task
      } else if (work) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int tile = i ? tB : tA;
#pragma unroll
          for (int nt = 0; nt < 2; ++nt) {
            const int n = ng * 16 + nt * 8 + s1_c_col(lane, 0);
            const float s0 = __ldg(L.scale + n), s1 = __ldg(L.scale + n + 1), h0 = __ldg(L.shift + n), h1 = __ldg(L.shift + n + 1);
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
              const int mrel = tile * 16 + s1_c_row(lane, rr * 2);
              if (mrel < rows) {
                const int opx = s1_out_px(g, cls, m0 + mrel);
                const float v0 = apply_act(fmaf(acc[i][nt][rr * 2], s0, h0), L.act), v1 = apply_act(fmaf(acc[i][nt][rr * 2 + 1], s1, h1), L.act);
                *reinterpret_cast<__half2*>(L.out + (size_t)opx * g.Cout + n) = __floats2half2_rn(v0, v1);
              }
            }
          }
        }
      }
    }
  }
  carry.valid = false;
}

__global__ void __launch_bounds__(kS1Threads, 1) k_s1_fused(const __grid_constant__ S1Params P) {
  extern __shared__ __align__(128) unsigned char s1_smem[];
  __half* act = reinterpret_cast<__half*>(s1_smem);
  float* partial = reinterpret_cast<float*>(s1_smem + kS1ActBytes);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rank = (int)cluster_rank(), nc = (int)cluster_size();
  for (int l = 0; l < 3; ++l) s1_prefetch_layer(P.L[l], rank, nc);
  // ---- layer 0: conv k3 s1 p1, in_ch -> base, FP32 input, LeakyReLU, FP16 output (input rows and weights staged in smem) ----
  {
    float* xs = reinterpret_cast<float*>(s1_smem);                 // [W][in_ch]
    float* ws = xs + P.W * P.in_ch;                                // [3][in_ch][base]
    for (int i = tid; i < P.W * P.in_ch; i += kS1Threads) xs[i] = P.x[i];
    for (int i = tid; i < 3 * P.in_ch * P.base; i += kS1Threads) ws[i] = __ldg(P.w0 + i);
    __syncthreads();
    const int total = P.W * P.base;
    for (int i = rank * kS1Threads + tid; i < total; i += nc * kS1Threads) {
      const int px = i / P.base, co = i - px * P.base;
      float a = 0.f;
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        const int ix = px + t - 1;
        if (ix < 0 || ix >= P.W) continue;
        for (int ci = 0; ci < P.in_ch; ++ci) a = fmaf(xs[ix * P.in_ch + ci], ws[(t * P.in_ch + ci) * P.base + co], a);
      }
      P.enc0[i] = __float2half_rn(apply_act(fmaf(a, __ldg(P.sc0 + co), __ldg(P.sh0 + co)), P.act0));
    }
  }
  S1Carry carry;
  carry.valid = false;
  cluster_arrive();
  s1_first_of_layer(P.L[0], rank, nc, warp, lane, carry);           // weights do not depend on the activations being exchanged
  cluster_wait();
  for (int l = 0; l < 14; ++l) {
    s1_layer(P.L[l], rank, nc, act, partial, carry);
    cluster_arrive();
    if (l + 3 < 14) s1_prefetch_layer(P.L[l + 3], rank, nc);
    if (l + 1 < 14) s1_first_of_layer(P.L[l + 1], rank, nc, warp, lane, carry);
    cluster_wait();
  }
  // ---- layer 15: conv k3 s1 p1 over the concatenation (yc0 + yc1 channels) -> out_ch, FP32 output; one warp per output pixel,
  //      weights staged in shared memory ----
  {
    const int Ct = P.yc0 + P.yc1;
    float* ws = reinterpret_cast<float*>(s1_smem);                 // [3][Ct][out_ch]
    for (int i = tid; i < 3 * Ct * P.out_ch; i += kS1Threads) ws[i] = __ldg(P.w15 + i);
    __syncthreads();
    for (int px = rank * kS1Warps + warp; px < P.W; px += nc * kS1Warps) {
      float a[16];
#pragma unroll
      for (int co = 0; co < 16; ++co) a[co] = 0.f;
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        const int ix = px + t - 1;
        if (ix < 0 || ix >= P.W) continue;
        for (int c = lane * 2; c < Ct; c += 64) {
          const __half2 hv = c < P.yc0 ? __ldcg(reinterpret_cast<const __half2*>(P.yin0 + (size_t)ix * P.yc0 + c))
                                       : __ldcg(reinterpret_cast<const __half2*>(P.yin1 + (size_t)ix * P.yc1 + (c - P.yc0)));
          const float2 xv = __half22float2(hv);
          const float* w = ws + (t * Ct + c) * P.out_ch;
#pragma unroll
          for (int co = 0; co < 16; ++co)
            if (co < P.out_ch) a[co] = fmaf(xv.y, w[P.out_ch + co], fmaf(xv.x, w[co], a[co]));
        }
      }
      float mine = 0.f;
#pragma unroll
      for (int co = 0; co < 16; ++co) {
        float v = a[co];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if (lane == co) mine = v;
      }
      if (lane < P.out_ch) P.y[(size_t)px * P.out_ch + lane] = apply_act(fmaf(mine, __ldg(P.sc15 + lane), __ldg(P.sh15 + lane)), P.act15);
    }
  }
}

// ---- host side -----------------------------------------------------------------------------------------------------------------
__global__ void k_s1_pack(const float* __restrict__ w, S1Geom g, __half* __restrict__ out) {
  const int K = s1_K(g);
  const size_t total = (size_t)s1_classes(g) * g.Cout * K;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % K); const size_t r = i / K;
    const int n = (int)(r % g.Cout), cls = (int)(r / g.Cout);
    out[s1_w_dst(g, cls, n, k)] = __float2half_rn(w[s1_w_src(g, cls, n, k)]);
  }
}

// Fragment-packed FP16 copy of a k4 layer of a 1-D net (d_w_chainer: the model file's layout, on the device).
int s1_pack_weights(const float* d_w_chainer, int transposed, int Cin, int Cout, __half* d_out, cudaStream_t st) {
  S1Geom g{transposed, 0, Cin, Cout};
  k_s1_pack<<<256, 256, 0, st>>>(d_w_chainer, g, d_out);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

static int g_s1_cluster = 0;     // 0: not initialised, -1: unavailable, else the cluster size

static bool pow2(int v) { return v > 0 && (v & (v - 1)) == 0; }

int s1_fused_init() {
  if (g_s1_cluster != 0) return 0;
  const int smem = kS1ActBytes + kS1PartialBytes;
  if (cudaFuncSetAttribute(k_s1_fused, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) { cudaGetLastError(); g_s1_cluster = -1; return 0; }
  int want = 16;
  if (cudaFuncSetAttribute(k_s1_fused, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) { cudaGetLastError(); want = 8; }
  for (; want >= 1; want /= 2) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(want); cfg.blockDim = dim3(kS1Threads); cfg.dynamicSmemBytes = smem;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = want; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    int n = 0;
    if (cudaOccupancyMaxActiveClusters(&n, k_s1_fused, &cfg) == cudaSuccess && n >= 1) { g_s1_cluster = want; return 0; }
    cudaGetLastError();
  }
  g_s1_cluster = -1;
  return 0;
}

// Can this plan run as the fused kernel?  (1-D net, FP16 plan, batch 1, fragment-packed weights present, channel counts the GEMM
// tiling assumes.)
bool s1_fused_eligible(const UNet* n, const UNetPlan* p) {
  if (g_s1_cluster <= 0 || !n || !p) return false;
  if (n->ndim != 1 || p->precision != 1 || p->B != 1 || p->H != 1 || p->W % 128 != 0) return false;
  if (n->base % 64 != 0 || !pow2(n->base / 64) || n->out_ch > 16 || n->layers.size() != 16) return false;
  for (int i = 1; i <= 14; ++i) {
    const UNetLayerW& L = n->layers[i];
    if (!L.d_w_frag || L.k != 4 || L.s != 2 || L.p != 1 || L.cin % 64 != 0 || L.cout % 16 != 0 || !pow2(L.cin / 64)) return false;
  }
  for (int i = 1; i <= 14; ++i) {                       // every layer's smallest M slab must fit the staging buffer
    const ConvLayer& L = p->layers[i];
    const S1Geom g{L.transposed, L.Win, L.C0 + L.C1, L.Cout};
    const S1Cut c = s1_cut(g, g_s1_cluster);
    const int M = s1_M(g);
    if ((size_t)s1_rows_for(g, c.slab < M ? c.slab : M) * c.RS * 2 > (size_t)kS1ActBytes) return false;
    if ((s1_K(g) / 32) % c.ks != 0 || ((s1_K(g) / 32) / c.ks) % 2 != 0 || c.MS * c.NP != g_s1_cluster) return false;
  }
  if ((size_t)(p->W * n->in_ch + 3 * n->in_ch * n->base) * 4 > (size_t)kS1ActBytes) return false;      // layer 0 stages its input and weights
  if ((size_t)3 * 2 * n->base * n->out_ch * 4 > (size_t)kS1ActBytes) return false;                       // layer 15 stages its weights
  return n->layers[0].k == 3 && n->layers[15].k == 3;
}

int s1_fused_run(Engine* e, const UNetPlan* p, cudaStream_t st) {
  RYK_CHECK(g_s1_cluster > 0 && p->fused, "fused stage-1 kernel not available for this plan");
  for (const ConvLayer& L : p->layers) RYK_CHECK(L.n_voices == 1, "the fused stage-1 kernel runs plans of one voice");
  S1Params P;
  for (int i = 1; i <= 14; ++i) {
    const ConvLayer& L = p->layers[i];
    S1LayerP& Q = P.L[i - 1];
    Q.in0 = (const __half*)L.in0; Q.in1 = (const __half*)L.in1; Q.out = (__half*)L.out;
    Q.w = (const uint4*)L.w_frag; Q.scale = L.wt.scale[0]; Q.shift = L.wt.shift[0];
    Q.transposed = L.transposed; Q.Win = L.Win; Q.C0 = L.C0; Q.C1 = L.C1; Q.Cout = L.Cout; Q.act = L.act;
    Q.lgCin = 0; while ((1 << Q.lgCin) < L.C0 + L.C1) ++Q.lgCin;
    Q.cut = s1_cut(S1Geom{L.transposed, L.Win, L.C0 + L.C1, L.Cout}, g_s1_cluster);
  }
  const ConvLayer& A = p->layers[0];
  P.x = (const float*)A.in0; P.w0 = A.wt.w[0]; P.sc0 = A.wt.scale[0]; P.sh0 = A.wt.shift[0]; P.enc0 = (__half*)A.out; P.in_ch = A.C0; P.base = A.Cout; P.act0 = A.act;
  const ConvLayer& Z = p->layers[15];
  P.yin0 = (const __half*)Z.in0; P.yin1 = (const __half*)Z.in1; P.w15 = Z.wt.w[0]; P.sc15 = Z.wt.scale[0]; P.sh15 = Z.wt.shift[0]; P.y = (float*)Z.out;
  P.yc0 = Z.C0; P.yc1 = Z.C1; P.out_ch = Z.Cout; P.act15 = Z.act;
  P.W = p->W;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(g_s1_cluster); cfg.blockDim = dim3(kS1Threads); cfg.dynamicSmemBytes = kS1ActBytes + kS1PartialBytes; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = g_s1_cluster; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  RYK_CUDA(cudaLaunchKernelEx(&cfg, k_s1_fused, P));
  return 0;
}

int s1_fused_cluster_size() { return g_s1_cluster; }

}  // namespace ryk
