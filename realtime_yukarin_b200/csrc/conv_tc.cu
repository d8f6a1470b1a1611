// conv_tc.cu -- Hopper (sm_90a) warpgroup-MMA implicit-GEMM convolution for the stage-2
// "Become-Yukarin" 2-D U-Net (SURVEY row a13, component I: > 99 % of the hot path's FLOPs).
//
//   D[pixels, Cout] = sum over taps t, channels c of  A_t[pixels, c] * W[t, c, Cout]
//
// * Operands are FP16, accumulation FP32 in registers (wgmma.mma_async m64nNk16, N = BLOCK_N).
// * A tiles (128 output pixels x 64 input channels of ONE tap) are fetched by TMA straight from the
//   NHWC activation tensor: a 4-D box (64 ch, tile_w, tile_h, 1) whose W/H traversal stride is the
//   conv stride (elementStrides = 2 for the k4 s2 p1 encoder convs) and whose out-of-bounds part is
//   zero-filled by the TMA unit -- that IS the zero padding; no im2col buffer ever exists.
//   Transposed convs (decoder) are run per output-parity class, each a dense 2x2-tap conv.
// * The U-Net skip concat is "by pointer": the K loop walks the channels of tensor 0, then tensor 1.
// * B tiles (BLOCK_N output channels x 64 K) come from a K-major packed weight matrix, also by TMA.
// * Both tiles land in the canonical 128-byte-swizzled K-major layout that wgmma smem descriptors
//   address; a ring of kStages stages is handed between the roles through mbarriers:
//     warp 8          : TMA producer   (waits empty[s], arms full[s] with expect_tx, issues 2 loads)
//     warpgroups 0, 1 : MMA + epilogue (wait full[s], 4 x wgmma on pixel rows 64 g .. 64 g + 63; release stage s once the
//                                       next stage's MMAs are issued; then folded BN scale/shift + LeakyReLU/ReLU,
//                                       FP16 staging in the idle stage buffers, TMA store)
// * Small-M bottleneck layers are weight-bandwidth bound: split-K over blockIdx.z spreads the weight
//   stream over all SMs; partial sums meet in an FP32 workspace and a reduce kernel applies the epilogue.
#include <cuda.h>
#include <cudaTypedefs.h>

#include "conv.h"
#include "tc_ptx.cuh"

namespace ryk {

struct TcParams {
  int transposed, B, Hout, Wout, Cout;
  int Hc, Wc;                    // class-local output grid (== Hout, Wout for convs)
  int tile_w, tile_h, tiles_w, tiles_h;  // tiles_h: tile rows of the band, which starts at tile row th0
  int th0;
  int skip_t0, skip_tn;          // tile rows [skip_t0, skip_t0 + skip_tn) are not launched (padded tail); the workspace omits them
  int run_y0, run_y1;            // rows [run_y0, run_y1) of source 0 repeat row run_y0: a box wholly inside them reads from run_y0
  int ws_y0;                     // output row of the band's first row: row 0 of the split-K workspace
  int chunks0, chunks1;          // 64-channel chunks of source 0 / 1
  int taps_w, ntaps;             // taps per class: conv KH*KW (taps_w = KW); deconv (KH/SH)*(KW/SW)
  int sh, sw, ph, pw;            // conv stride / padding per dimension (1-D nets: sh = 1, ph = 0)
  int classes_w;                 // deconv output-parity classes along W (SW); along H it is SH
  int ksplit, chunks_per_split;
  int act;
  LayerWeights wt;               // per-voice scale / shift and the voice of each batch item (weights: the per-voice tensor maps)
  float* ws;                     // split-K workspace [ksplit][pixels][Cout] or nullptr
  size_t out_pixels;             // B * Hout * Wout
};

template <int BLOCK_N>
__device__ __forceinline__ void wgmma_tile(float (&acc)[BLOCK_N / 2], uint64_t adesc, uint64_t bdesc) {
  if constexpr (BLOCK_N == 128) wgmma_m64n128(acc, adesc, bdesc);
  else wgmma_m64n64(acc, adesc, bdesc);
}

template <int BLOCK_N, int kStages, int kMinBlocks>
__global__ void __launch_bounds__(kTcThreads, kMinBlocks)
k_conv_tc(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
          const __grid_constant__ TcWeightMaps tmB, const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmW,
          const __grid_constant__ TcParams p) {
  static_assert(BLOCK_N == 64 || BLOCK_N == 128, "BLOCK_N");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  constexpr uint32_t kABytes = kBlockM * kBlockK * 2;
  constexpr uint32_t kBBytes = BLOCK_N * kBlockK * 2;
  static_assert((size_t)kBlockM * BLOCK_N * 4 <= (size_t)kStages * (kABytes + kBBytes), "epilogue staging must fit the stage buffers");
  // carve: 1024-aligned stage buffers first, barriers after
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * kABytes;
  uint64_t* full_bar = (uint64_t*)(smem_b + kStages * kBBytes);
  uint64_t* empty_bar = full_bar + kStages;
  // per-channel scale / shift of this CTA's BLOCK_N output channels, staged once: the epilogue reads them from shared memory
  float* s_scale = (float*)(((uintptr_t)(empty_bar + kStages) + 15) & ~(uintptr_t)15);
  float* s_shift = s_scale + BLOCK_N;

  const int warp = threadIdx.x >> 5;
  pdl_trigger();

  // tile coordinates
  int mt = blockIdx.x;
  const int tw = mt % p.tiles_w; mt /= p.tiles_w;
  int th = mt % p.tiles_h + p.th0; mt /= p.tiles_h;
  const bool past_skip = th >= p.skip_t0;
  th += past_skip ? p.skip_tn : 0;
  const int b = mt;
  const int n0 = blockIdx.y * BLOCK_N;
  const int cls = blockIdx.z / p.ksplit, split = blockIdx.z % p.ksplit;
  const int py = cls / p.classes_w, px = cls % p.classes_w;
  const int oy0 = th * p.tile_h, ox0 = tw * p.tile_w;       // class-local output origin of the tile
  const int chunks_per_tap = p.chunks0 + p.chunks1;
  const int total_chunks = p.ntaps * chunks_per_tap;
  const int kc_begin = split * p.chunks_per_split;
  const int kc_end = min(total_chunks, kc_begin + p.chunks_per_split);
  const int my_chunks = kc_end - kc_begin;
  const int voice = item_voice(p.wt, b);                     // this tile's batch item reads its voice's weights
  const CUtensorMap* tmBv = &tmB.m[voice];

  if (threadIdx.x == kTcConsumers) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA0) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(tmBv) : "memory");
    if (p.chunks1 > 0) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA1) : "memory");
    if (!p.ws) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmO) : "memory");
    else asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW) : "memory");
    for (int i = 0; i < kStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kTcConsumers / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (threadIdx.x < kTcConsumers && !p.ws) {
    const float* scale = p.wt.scale[voice]; const float* shift = p.wt.shift[voice];
    for (int i = threadIdx.x; i < BLOCK_N; i += kTcConsumers) { s_scale[i] = __ldg(scale + n0 + i); s_shift[i] = __ldg(shift + n0 + i); }
  }
  __syncthreads();
  pdl_wait();                      // the previous layer's outputs (our A operand) are complete from here on

  if (warp == kTcConsumers / 32) {
    // ===== TMA producer (warp-uniform loop, one elected lane issues: see elect_one() in tc_ptx.cuh) =====
    for (int i = 0; i < my_chunks; ++i) {
      const int s = i % kStages;
      const uint32_t ph = (i / kStages) & 1;
      mbar_wait(&empty_bar[s], ph ^ 1);
      const int kc = kc_begin + i;
      const int tap = kc / chunks_per_tap;
      const int cc = kc - tap * chunks_per_tap;
      const int ty = tap / p.taps_w, tx = tap - ty * p.taps_w;
      int ix, iy;
      if (!p.transposed) {
        ix = ox0 * p.sw + tx - p.pw; iy = oy0 * p.sh + ty - p.ph;
        if (iy >= p.run_y0 && iy + p.sh * (p.tile_h - 1) < p.run_y1) iy = p.run_y0;
      }
      else {   // k4 s2 p1 along a strided dimension: input = m + d - 1 + parity; k1 s1 p0 along the other: input = m
        ix = p.sw == 2 ? ox0 + tx - 1 + px : ox0;
        iy = p.sh == 2 ? oy0 + ty - 1 + py : oy0;
      }
      if (elect_one()) {
        mbar_expect_tx(&full_bar[s], kABytes + kBBytes);
        if (cc < p.chunks0) tma_load_4d(smem_a + s * kABytes, &tmA0, &full_bar[s], cc * kBlockK, ix, iy, b);
        else tma_load_4d(smem_a + s * kABytes, &tmA1, &full_bar[s], (cc - p.chunks0) * kBlockK, ix, iy, b);
        tma_load_2d(smem_b + s * kBBytes, tmBv, &full_bar[s], kc * kBlockK, cls * p.Cout + n0);
      }
    }
  } else if (warp < kTcConsumers / 32) {
    // ===== MMA: warpgroup g owns accumulator rows (tile pixels) 64 g .. 64 g + 63 =====
    const int g = threadIdx.x >> 7, wl = warp & 3, lane = threadIdx.x & 31;
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; ++i) acc[i] = 0.f;
    wgmma_fence_acc(acc);
    for (int i = 0; i < my_chunks; ++i) {
      const int s = i % kStages;
      mbar_wait(&full_bar[s], (i / kStages) & 1);
      const uint64_t adesc = make_sw128_desc(smem_u32(smem_a + s * kABytes + g * (64 * 128)));
      const uint64_t bdesc = make_sw128_desc(smem_u32(smem_b + s * kBBytes));
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBlockK / kMmaK; ++k) wgmma_tile<BLOCK_N>(acc, adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2));
      wgmma_commit();
      // at most this stage's MMAs still in flight: the previous stage has been read and goes back to the producer
      wgmma_wait<1>();
      wgmma_fence_acc(acc);
      if (i > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[(i - 1) % kStages]);
      }
    }
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    // both warpgroups' MMAs have finished reading the stage buffers before either overwrites them with its epilogue staging
    asm volatile("bar.sync 1, %0;" ::"n"(kTcConsumers) : "memory");
    const int rbase = g * 64 + wl * 16 + (lane >> 2);           // tile rows of registers i with ((i >> 1) & 1) == 0; +8 for the others
    const int cq = 2 * (lane & 3);
    // (out-of-range pixels of ragged tiles need no masking: both TMA stores below clip at the tensor-map bounds)
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; i += 2) {
      const int row = rbase + 8 * ((i >> 1) & 1);
      const int col = 8 * (i >> 2) + cq;
      const float a0 = acc[i], a1 = acc[i + 1];
      if (p.ws) {
        // split-K partial tile (raw FP32 sums) -> 128B-swizzled [128 pixels][32 channels] blocks, stored below by TMA into this
        // split's slice of the workspace; k_splitk_reduce sums the slices
        uint8_t* blk = smem + (col >> 5) * (kBlockM * 128) + row * 128;
        *reinterpret_cast<float2*>(blk + ((((col & 31) >> 2) ^ (row & 7)) << 4) + (col & 3) * 4) = make_float2(a0, a1);
      } else {
        // scale/shift/activation -> FP16 -> 128B-swizzled [128 pixels][64 channels] blocks; one TMA store per block writes full
        // 128-byte rows
        float v0 = fmaf(a0, s_scale[col], s_shift[col]);
        float v1 = fmaf(a1, s_scale[col + 1], s_shift[col + 1]);
        if (p.act == ACT_LEAKY) { v0 = v0 > 0.f ? v0 : 0.2f * v0; v1 = v1 > 0.f ? v1 : 0.2f * v1; }
        else if (p.act == ACT_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
        uint8_t* blk = smem + (col >> 6) * (kBlockM * 128) + row * 128;
        *reinterpret_cast<__half2*>(blk + ((((col & 63) >> 3) ^ (row & 7)) << 4) + (col & 7) * 2) = __floats2half2_rn(v0, v1);
      }
    }
    if (my_chunks > 0) {
      // generic-proxy smem writes -> visible to the async proxy; one thread hands the tile to the TMA unit
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      asm volatile("bar.sync 1, %0;" ::"n"(kTcConsumers) : "memory");
      if (threadIdx.x == 0) {
        const int xs = p.transposed ? ox0 * p.sw + px : ox0;
        const int ys = p.transposed ? oy0 * p.sh + py : oy0;
        if (!p.ws) {
#pragma unroll
          for (int jb = 0; jb < BLOCK_N / 64; ++jb)
            asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                         ::"l"(&tmO), "r"(smem_u32(smem + jb * (kBlockM * 128))), "r"(n0 + jb * 64), "r"(xs), "r"(ys), "r"(b) : "memory");
        } else {
#pragma unroll
          for (int jb = 0; jb < BLOCK_N / 32; ++jb)
            asm volatile("cp.async.bulk.tensor.5d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5, %6}], [%1];"
                         ::"l"(&tmW), "r"(smem_u32(smem + jb * (kBlockM * 128))), "r"(n0 + jb * 32), "r"(xs),
                         "r"(ys - p.ws_y0 - (past_skip ? p.skip_tn * p.tile_h : 0)), "r"(b), "r"(split) : "memory");
        }
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      }
    }
  }
}

// split-K reduce + epilogue: out = act((sum over splits of ws[s]) * scale + shift) as fp16, 4 channels per thread.
// The workspace holds the layer's row band: band4 float4s per batch item, written to out at out_off4 + b * out_stride4 (float4 units).
// Block = G warps x 32 lanes: lane = one float4 of the output (512 contiguous bytes per warp load), warp g sums the
// slices g, g + G, g + 2G, ... ; the G partial sums are combined through shared memory in a fixed order, so the result
// is deterministic (same summation tree every run) while G x more loads are in flight than with one thread per output.
__global__ void __launch_bounds__(256) k_splitk_reduce(const float* __restrict__ ws, size_t total4, size_t slice_elems, int ksplit, int Cout,
                                const __grid_constant__ LayerWeights wt, int act, __half* __restrict__ out,
                                size_t band4, size_t out_stride4, size_t out_off4, size_t gap_at4, size_t gap4) {
  __shared__ float4 part[8][32];
  pdl_trigger();
  pdl_wait();
  const int lane = threadIdx.x & 31, g = threadIdx.x >> 5, G = blockDim.x >> 5;
  const size_t i = (size_t)blockIdx.x * 32 + lane;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i < total4) {
    const float4* p = reinterpret_cast<const float4*>(ws) + i;
    const size_t stride4 = slice_elems / 4;
#pragma unroll 4
    for (int s = g; s < ksplit; s += G) {
      const float4 b = __ldg(p + (size_t)s * stride4);
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
  }
  part[g][lane] = a;
  __syncthreads();
  if (g != 0 || i >= total4) return;
  for (int k = 1; k < G; ++k) { const float4 b = part[k][lane]; a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }
  const size_t item = i / band4;
  const size_t r = i % band4, o = item * out_stride4 + out_off4 + r + (r >= gap_at4 ? gap4 : 0);
  const int n = (int)((o * 4) % Cout);
  const int voice = item_voice(wt, (int)item);
  const float* scale = wt.scale[voice]; const float* shift = wt.shift[voice];
  const float4 sc = __ldg(reinterpret_cast<const float4*>(scale + n)), sh = __ldg(reinterpret_cast<const float4*>(shift + n));
  float v[4] = {fmaf(a.x, sc.x, sh.x), fmaf(a.y, sc.y, sh.y), fmaf(a.z, sc.z, sh.z), fmaf(a.w, sc.w, sh.w)};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (act == ACT_LEAKY) v[j] = v[j] > 0.f ? v[j] : 0.2f * v[j]; else if (act == ACT_RELU) v[j] = fmaxf(v[j], 0.f);
  }
  __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
  reinterpret_cast<uint2*>(out)[o] = make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
}

// few splits, large outputs (c3 / c4 / d3): one thread per float4 of the output, grid-stride, all slices summed in order
__global__ void __launch_bounds__(256) k_splitk_reduce_few(const float* __restrict__ ws, size_t total4, size_t slice_elems, int ksplit, int Cout,
                                    const __grid_constant__ LayerWeights wt, int act, __half* __restrict__ out,
                                    size_t band4, size_t out_stride4, size_t out_off4, size_t gap_at4, size_t gap4) {
  const size_t stride4 = slice_elems / 4;
  pdl_trigger();
  pdl_wait();
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total4; i += (size_t)gridDim.x * blockDim.x) {
    const float4* p = reinterpret_cast<const float4*>(ws) + i;
    float4 a = __ldg(p);
#pragma unroll 4
    for (int s = 1; s < ksplit; ++s) {
      const float4 b = __ldg(p + (size_t)s * stride4);
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    const size_t item = i / band4;
    const size_t r = i % band4, o = item * out_stride4 + out_off4 + r + (r >= gap_at4 ? gap4 : 0);
    const int n = (int)((o * 4) % Cout);
    const int voice = item_voice(wt, (int)item);
    const float* scale = wt.scale[voice]; const float* shift = wt.shift[voice];
    const float4 sc = __ldg(reinterpret_cast<const float4*>(scale + n)), sh = __ldg(reinterpret_cast<const float4*>(shift + n));
    float v[4] = {fmaf(a.x, sc.x, sh.x), fmaf(a.y, sc.y, sh.y), fmaf(a.z, sc.z, sh.z), fmaf(a.w, sc.w, sh.w)};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (act == ACT_LEAKY) v[j] = v[j] > 0.f ? v[j] : 0.2f * v[j]; else if (act == ACT_RELU) v[j] = fmaxf(v[j], 0.f);
    }
    __half2 h0 = __floats2half2_rn(v[0], v[1]), h1 = __floats2half2_rn(v[2], v[3]);
    reinterpret_cast<uint2*>(out)[o] = make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
  }
}

// ------------------------------------------------------------------------------------ host side
static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;

template <int BN, int ST> static constexpr size_t tc_smem_bytes() {
  return (size_t)ST * (kBlockM * kBlockK * 2 + BN * kBlockK * 2) + 2 * ST * 8 + 16 + 1024 + 2 * BN * 4 + 32;
}
// Kernel configurations (BLOCK_N, stages, CTAs/SM): two co-resident CTAs per SM let one tile's epilogue overlap the other's main
// loop; both fit 2 x ~98 KB of an H100 SM's 228 KB of shared memory and its 64 K registers (2 x 288 threads x <= 112).
#define RYK_TC_N128 k_conv_tc<128, 3, 2>
#define RYK_TC_N64 k_conv_tc<64, 4, 2>

int tc_init() {
  if (!g_encode) {
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    RYK_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
    RYK_CHECK(qres == cudaDriverEntryPointSuccess && fn != nullptr, "cuTensorMapEncodeTiled not available from the driver");
    g_encode = (PFN_cuTensorMapEncodeTiled_v12000)fn;
  }
  RYK_CUDA(cudaFuncSetAttribute(RYK_TC_N128, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc_smem_bytes<128, 3>()));
  RYK_CUDA(cudaFuncSetAttribute(RYK_TC_N64, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc_smem_bytes<64, 4>()));
  return 0;
}

bool tc_layer_eligible(const ConvLayer& L) {
  const bool k2d = L.KH == 4 && L.KW == 4 && L.SH == 2 && L.SW == 2 && L.PH == 1 && L.PW == 1;
  const bool k1d = L.KH == 1 && L.KW == 4 && L.SH == 1 && L.SW == 2 && L.PH == 0 && L.PW == 1;
  if (!k2d && !k1d) return false;
  if (L.C0 % kBlockK != 0 || L.C1 % kBlockK != 0 || L.C0 == 0) return false;
  if (L.Cout % 64 != 0) return false;
  if (L.in_dtype != DT_F16 || L.out_dtype != DT_F16) return false;
  return true;
}

static int pow2_floor(int v) { int p = 1; while (p * 2 <= v) p *= 2; return p; }

static int make_act_map(CUtensorMap* m, const void* ptr, int C, int W, int H, int B, int box_w, int box_h, int stride_w, int stride_h) {
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {(cuuint32_t)kBlockK, (cuuint32_t)(box_w * stride_w), (cuuint32_t)(box_h * stride_h), 1};
  cuuint32_t estr[4] = {1, (cuuint32_t)stride_w, (cuuint32_t)stride_h, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(activation) failed: " + std::to_string((int)r)); return -1; }
  return 0;
}

// split-K workspace [ksplit][B][Hout][Wout][Cout] fp32 as a 5-D map: box = (32 channels, tile_w, tile_h, 1, 1) with the same
// W / H element strides as the output map (deconv parity classes write every other pixel)
static int make_ws_map(CUtensorMap* m, const void* ptr, int C, int W, int H, int B, int ksplit, int box_w, int box_h, int stride_w, int stride_h) {
  cuuint64_t dims[5] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B, (cuuint64_t)ksplit};
  cuuint64_t strides[4] = {(cuuint64_t)C * 4, (cuuint64_t)W * C * 4, (cuuint64_t)H * W * C * 4, (cuuint64_t)B * H * W * C * 4};
  cuuint32_t box[5] = {32, (cuuint32_t)(box_w * stride_w), (cuuint32_t)(box_h * stride_h), 1, 1};
  cuuint32_t estr[5] = {1, (cuuint32_t)stride_w, (cuuint32_t)stride_h, 1, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<void*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(split-K workspace) failed: " + std::to_string((int)r)); return -1; }
  return 0;
}

static int make_weight_map(CUtensorMap* m, const void* ptr, size_t K, size_t rows, int block_n) {
  cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)K * 2};
  cuuint32_t box[2] = {(cuuint32_t)kBlockK, (cuuint32_t)block_n};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(weights) failed: " + std::to_string((int)r)); return -1; }
  return 0;
}

static void tc_tile_shape(const ConvLayer& L, int* tile_w, int* tile_h) {
  const int Wc = L.transposed ? L.Win : L.Wout;
  *tile_w = pow2_floor(Wc < kBlockM ? Wc : kBlockM);
  *tile_h = kBlockM / *tile_w;
}

int tc_tile_rows(const ConvLayer& L) { int tw, th; tc_tile_shape(L, &tw, &th); return th; }

int tc_tile_count(const ConvLayer& L) {
  int tw, th;
  tc_tile_shape(L, &tw, &th);
  const int Wc = L.transposed ? L.Win : L.Wout;
  const int band_tiles_h = (layer_band_end(L) - L.band_y0 + th - 1) / th;
  const int bn = L.Cout >= 128 ? 128 : 64;
  const int classes = L.transposed ? L.SH * L.SW : 1;
  return L.B * ((Wc + tw - 1) / tw) * band_tiles_h * (L.Cout / bn) * classes;
}

// Tile shape, N block and split-K of a layer.  Split-K fills the SMs when the band has few tiles, so a banded layer may split
// K further than the same layer over every row (L.ksplit_tiles overrides the tile count this rule sees).
static void tc_geometry(const ConvLayer& L, int num_sms, int* tile_w, int* tile_h, int* block_n, int* ksplit) {
  int tw, th;
  tc_tile_shape(L, &tw, &th);
  int bn = L.Cout >= 128 ? 128 : 64;
  int tiles = L.ksplit_tiles > 0 ? L.ksplit_tiles : tc_tile_count(L);
  int ntaps = L.transposed ? (L.KH / L.SH) * (L.KW / L.SW) : L.KH * L.KW;
  int total_chunks = ntaps * (L.C0 + L.C1) / kBlockK;
  int ks = 1;
  int slots = num_sms * 2;                            // two co-resident CTAs per SM
  if (tiles < slots) {
    constexpr int kMinChunks = 8;                       // at least this many K chunks per split
    ks = slots / tiles;
    if (ks > total_chunks / kMinChunks) ks = total_chunks / kMinChunks;
    if (ks < 1) ks = 1;
    int cps = (total_chunks + ks - 1) / ks;
    ks = (total_chunks + cps - 1) / cps;                // every split owns at least one chunk
  }
  *tile_w = tw; *tile_h = th; *block_n = bn; *ksplit = ks;
}

// Rows of one batch item in the split-K workspace: the band's output rows [r0, r1) less the skipped tail rows, which leave a gap of
// `gap` rows after workspace row `gap_at` (workspace row w holds output row r0 + w, or r0 + w + gap from gap_at on).
static int tc_ws_rows(const ConvLayer& L, int* r0, int* gap_at, int* gap) {
  int r1;
  layer_band_out_rows(L, r0, &r1);
  *gap = L.skip_y1 - L.skip_y0;
  *gap_at = *gap ? L.skip_y0 - *r0 : 0;
  return r1 - *r0 - *gap;
}

size_t tc_splitk_ws_bytes(const ConvLayer& L, int num_sms) {
  int tw, th, bn, ks;
  tc_geometry(L, num_sms, &tw, &th, &bn, &ks);
  int r0, gap_at, gap;
  const int rows = tc_ws_rows(L, &r0, &gap_at, &gap);
  return ks > 1 ? (size_t)ks * L.B * rows * L.Wout * L.Cout * sizeof(float) : 0;
}

int tc_layer_weight_maps(ConvLayer& L) {
  RYK_CHECK(L.n_voices >= 1 && L.n_voices <= kMaxGroupVoices, "a layer holds 1..8 voices");
  const int classes = L.transposed ? L.SH * L.SW : 1;
  const int ntaps = L.transposed ? (L.KH / L.SH) * (L.KW / L.SW) : L.KH * L.KW;
  const size_t K = (size_t)ntaps * (L.C0 + L.C1), rows = (size_t)classes * L.Cout;
  for (int v = 0; v < L.n_voices; ++v) {
    RYK_CHECK(L.w_tc[v] != nullptr, "tensor-core layer without packed weights for one of its voices");
    if (make_weight_map(&L.tmB.m[v], L.w_tc[v], K, rows, L.block_n)) return -1;
  }
  for (int v = L.n_voices; v < kMaxGroupVoices; ++v) L.tmB.m[v] = L.tmB.m[0];    // never selected
  return 0;
}

int tc_layer_prepare(ConvLayer& L, int num_sms) {
  RYK_CHECK(g_encode != nullptr, "tc_init() was not called");
  RYK_CHECK(tc_layer_eligible(L), "layer is not eligible for the tensor-core path");
  tc_geometry(L, num_sms, &L.tile_w, &L.tile_h, &L.block_n, &L.ksplit);
  int stw = L.transposed ? 1 : L.SW, sth = L.transposed ? 1 : L.SH;
  if (make_act_map(&L.tmA0, L.in0, L.C0, L.Win, L.Hin, L.B, L.tile_w, L.tile_h, stw, sth)) return -1;
  if (L.C1 > 0) { if (make_act_map(&L.tmA1, L.in1, L.C1, L.Win, L.Hin, L.B, L.tile_w, L.tile_h, stw, sth)) return -1; }
  else L.tmA1 = L.tmA0;
  if (tc_layer_weight_maps(L)) return -1;
  // output map for the TMA-store epilogue: deconv classes write every other pixel (element strides = conv strides)
  if (make_act_map(&L.tmO, L.out, L.Cout, L.Wout, L.Hout, L.B, L.tile_w, L.tile_h, L.transposed ? L.SW : 1, L.transposed ? L.SH : 1)) return -1;
  RYK_CHECK(L.ksplit == 1 || L.splitk_ws != nullptr, "split-K layer without a workspace");
  RYK_CHECK(L.band_y0 >= 0 && L.band_y0 % L.tile_h == 0 && L.band_y0 < layer_band_end(L) && layer_band_end(L) <= layer_class_rows(L) &&
            (layer_band_end(L) % L.tile_h == 0 || layer_band_end(L) == layer_class_rows(L)), "row band is not a range of whole tile rows");
  RYK_CHECK(L.skip_y1 == 0 || (!L.transposed && L.skip_y0 % L.tile_h == 0 && L.skip_y1 % L.tile_h == 0 && L.band_y0 <= L.skip_y0 &&
                               L.skip_y0 < L.skip_y1 && L.skip_y1 <= layer_band_end(L)),
            "skipped rows are not a range of whole tile rows inside the band of a convolution");
  if (L.ksplit > 1) {
    // the workspace holds the band's computed output rows only
    int r0, gap_at, gap;
    const int rows = tc_ws_rows(L, &r0, &gap_at, &gap);
    if (make_ws_map(&L.tmW, L.splitk_ws, L.Cout, L.Wout, rows, L.B, L.ksplit, L.tile_w, L.tile_h, L.transposed ? L.SW : 1, L.transposed ? L.SH : 1)) return -1;
  } else L.tmW = L.tmO;
  L.tc_ready = true;
  return 0;
}

// Launch with the programmatic-stream-serialization attribute (see pdl_trigger / pdl_wait).
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

int conv_tc_run(const ConvLayer& L, cudaStream_t st) {
  RYK_CHECK(L.tc_ready, "tc layer not prepared");
  TcParams p;
  p.transposed = L.transposed; p.B = L.B; p.Hout = L.Hout; p.Wout = L.Wout; p.Cout = L.Cout;
  p.Hc = L.transposed ? L.Hin : L.Hout; p.Wc = L.transposed ? L.Win : L.Wout;
  p.tile_w = L.tile_w; p.tile_h = L.tile_h;
  // the grid covers the band's tile rows of the layer's tile grid less the skipped ones: every output pixel keeps its tile and so
  // its K order
  p.skip_t0 = L.skip_y0 / L.tile_h; p.skip_tn = (L.skip_y1 - L.skip_y0) / L.tile_h;
  p.tiles_w = (p.Wc + L.tile_w - 1) / L.tile_w; p.tiles_h = (layer_band_end(L) - L.band_y0 + L.tile_h - 1) / L.tile_h - p.skip_tn;
  p.th0 = L.band_y0 / L.tile_h;
  p.run_y0 = L.run_y0; p.run_y1 = L.run_y1;
  int r0, gap_at, gap;
  const int ws_rows = tc_ws_rows(L, &r0, &gap_at, &gap);
  p.ws_y0 = r0;
  p.chunks0 = L.C0 / kBlockK; p.chunks1 = L.C1 / kBlockK;
  p.taps_w = L.transposed ? L.KW / L.SW : L.KW;
  p.ntaps = L.transposed ? (L.KH / L.SH) * (L.KW / L.SW) : L.KH * L.KW;
  p.sh = L.SH; p.sw = L.SW; p.ph = L.PH; p.pw = L.PW;
  p.classes_w = L.transposed ? L.SW : 1;
  const int classes = L.transposed ? L.SH * L.SW : 1;
  p.ksplit = L.ksplit;
  int total_chunks = p.ntaps * (p.chunks0 + p.chunks1);
  p.chunks_per_split = (total_chunks + L.ksplit - 1) / L.ksplit;
  p.act = L.act; p.wt = L.wt;
  p.ws = L.ksplit > 1 ? L.splitk_ws : nullptr;
  p.out_pixels = (size_t)L.B * L.Hout * L.Wout;
  const size_t row_elems = (size_t)L.Wout * L.Cout;
  const size_t band_elems = (size_t)L.B * ws_rows * row_elems;        // one workspace slice
  dim3 grid(L.B * p.tiles_w * p.tiles_h, L.Cout / L.block_n, classes * L.ksplit);
  if (L.block_n == 128) RYK_CUDA(launch_pdl(RYK_TC_N128, grid, dim3(kTcThreads), tc_smem_bytes<128, 3>(), st, L.tmA0, L.tmA1, L.tmB, L.tmO, L.tmW, p));
  else RYK_CUDA(launch_pdl(RYK_TC_N64, grid, dim3(kTcThreads), tc_smem_bytes<64, 4>(), st, L.tmA0, L.tmA1, L.tmB, L.tmO, L.tmW, p));
  RYK_CUDA(cudaGetLastError());
  if (p.ws) {
    const size_t total4 = band_elems / 4, band4 = ws_rows * row_elems / 4, stride4 = L.Hout * row_elems / 4, off4 = r0 * row_elems / 4;
    const size_t gap_at4 = gap_at * row_elems / 4, gap4 = gap * row_elems / 4;
    if (L.ksplit <= 4) {
      int blocks = (int)((total4 + 255) / 256); if (blocks > 2112) blocks = 2112;     // 16 per SM of 132
      RYK_CUDA(launch_pdl(k_splitk_reduce_few, dim3(blocks), dim3(256), 0, st, (const float*)p.ws, total4, band_elems, L.ksplit, L.Cout, L.wt, L.act,
                          (__half*)L.out, band4, stride4, off4, gap_at4, gap4));
    } else {
      RYK_CUDA(launch_pdl(k_splitk_reduce, dim3((unsigned)((total4 + 31) / 32)), dim3(256), 0, st, (const float*)p.ws, total4, band_elems, L.ksplit, L.Cout, L.wt, L.act,
                          (__half*)L.out, band4, stride4, off4, gap_at4, gap4));
    }
    RYK_CUDA(cudaGetLastError());
  }
  return 0;
}

}  // namespace ryk
