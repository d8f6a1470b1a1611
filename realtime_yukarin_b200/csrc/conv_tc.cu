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
//   stream over all SMs.  The ksplit CTAs of one tile run as one thread-block cluster: each stages its FP32 partial tile in its
//   own shared memory, and each reduces a share of the tile's pixels over all ranks' partials through distributed shared memory
//   (splitk_sum fixes the order) before applying the epilogue.
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
  int skip_t0, skip_tn;          // tile rows [skip_t0, skip_t0 + skip_tn) are not launched (padded tail)
  int run_y0, run_y1;            // rows [run_y0, run_y1) of source 0 repeat row run_y0: a box wholly inside them reads from run_y0
  int chunks0, chunks1;          // 64-channel chunks of source 0 / 1
  int taps_w, ntaps;             // taps per class: conv KH*KW (taps_w = KW); deconv (KH/SH)*(KW/SW)
  int sh, sw, ph, pw;            // conv stride / padding per dimension (1-D nets: sh = 1, ph = 0)
  int classes_w;                 // deconv output-parity classes along W (SW); along H it is SH
  int ksplit, chunks_per_split;  // ksplit > 1: the grid runs in clusters of (1, 1, ksplit), one tile's K splits each
  int act;
  LayerWeights wt;               // per-voice scale / shift and the voice of each batch item (weights: the per-voice tensor maps)
  __half* out;                   // NHWC [B][Hout][Wout][Cout]: split-K layers store their reduced tiles here directly
};

template <int BLOCK_N>
__device__ __forceinline__ void wgmma_tile(float (&acc)[BLOCK_N / 2], uint64_t adesc, uint64_t bdesc) {
  if constexpr (BLOCK_N == 128) wgmma_m64n128(acc, adesc, bdesc);
  else wgmma_m64n64(acc, adesc, bdesc);
}

// Largest split-K factor: one cluster holds one tile's splits, and 16 CTAs is the largest (non-portable) cluster of sm_90.
constexpr int kMaxSplits = 16;

__device__ __forceinline__ void add4(float4& a, const float4& b) { a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w; }

// The split-K summation order.  This is a contract: it fixes the FP32 rounding of every split layer's outputs, so the network's
// results are bitwise the same however the splits are scheduled.  v[s] is split s's partial sum, s < ks <= kMaxSplits.
//   ks <= 4: a = v[0]; a += v[1]; ...; a += v[ks - 1]
//   ks >  4: part[g] = 0.f; part[g] += v[g]; part[g] += v[g + 8] (terms with index >= ks left out), g = 0..7;
//            a = part[0]; a += part[1]; ...; a += part[7]
__device__ __forceinline__ float4 splitk_sum(const float4 (&v)[kMaxSplits], int ks) {
  float4 a = v[0];
  if (ks <= 4) {
#pragma unroll
    for (int s = 1; s < 4; ++s) if (s < ks) add4(a, v[s]);
    return a;
  }
#pragma unroll
  for (int g = 0; g < 8; ++g) {
    float4 part = make_float4(0.f, 0.f, 0.f, 0.f);
    if (g < ks) add4(part, v[g]);
    if (g + 8 < ks) add4(part, v[g + 8]);
    if (g == 0) a = part; else add4(a, part);
  }
  return a;
}

// Byte offset of 16-byte chunk c (4 channels) of tile row (pixel) `row` in a split CTA's FP32 partial tile [128][BLOCK_N]; the
// chunk index is XOR-swizzled by row so that both the accumulator stores and the reducers' row reads spread over all banks.
template <int BLOCK_N>
__device__ __forceinline__ uint32_t partial_offset(int row, int c) { return (uint32_t)(row * BLOCK_N * 4 + ((c ^ (row & 7)) << 4)); }

template <int BLOCK_N, int kStages, int kMinBlocks>
__global__ void __launch_bounds__(kTcThreads, kMinBlocks)
k_conv_tc(const __grid_constant__ CUtensorMap tmA0, const __grid_constant__ CUtensorMap tmA1,
          const __grid_constant__ TcWeightMaps tmB, const __grid_constant__ CUtensorMap tmO, const __grid_constant__ TcParams p) {
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
  th += th >= p.skip_t0 ? p.skip_tn : 0;
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
    if (p.ksplit == 1) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmO) : "memory");
    for (int i = 0; i < kStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kTcConsumers / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (threadIdx.x < kTcConsumers) {
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
    if (p.ksplit > 1) { cluster_sync_all(); cluster_sync_all(); }     // the split epilogue's two cluster barriers count every thread
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
    if (p.ksplit > 1) {
      // split-K: this split's raw FP32 partial tile -> its own stage buffers; the cluster's ranks then each reduce a share of the
      // tile's valid pixels over every rank's partial
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; i += 2) {
        const int row = rbase + 8 * ((i >> 1) & 1);
        const int col = 8 * (i >> 2) + cq;
        *reinterpret_cast<float2*>(smem + partial_offset<BLOCK_N>(row, col >> 2) + (col & 3) * 4) = make_float2(acc[i], acc[i + 1]);
      }
      cluster_sync_all();                                          // every rank's partial is in its shared memory
      // valid pixels of the tile: ragged tiles end at the class-local grid's last row / column
      const int vw = min(p.tile_w, p.Wc - ox0), vh = min(p.tile_h, p.Hc - oy0);
      constexpr int kChunks = BLOCK_N / 4;
      const int total = vw * vh * kChunks;
      const int j1 = (int)((long long)total * (split + 1) / p.ksplit);
      const uint32_t partial = smem_u32(smem);
      for (int j = (int)((long long)total * split / p.ksplit) + threadIdx.x; j < j1; j += kTcConsumers) {
        const int q = j / kChunks, c = j - q * kChunks;
        const int y = q / vw, x = q - y * vw;
        const uint32_t off = partial + partial_offset<BLOCK_N>(y * p.tile_w + x, c);
        float4 v[kMaxSplits];
#pragma unroll
        for (int s = 0; s < kMaxSplits; ++s)
          if (s < p.ksplit) v[s] = ld_cluster_f4(cluster_map(off, s));
        const float4 a = splitk_sum(v, p.ksplit);
        const int n = 4 * c;
        float o[4] = {fmaf(a.x, s_scale[n], s_shift[n]), fmaf(a.y, s_scale[n + 1], s_shift[n + 1]),
                      fmaf(a.z, s_scale[n + 2], s_shift[n + 2]), fmaf(a.w, s_scale[n + 3], s_shift[n + 3])};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          if (p.act == ACT_LEAKY) o[k] = o[k] > 0.f ? o[k] : 0.2f * o[k]; else if (p.act == ACT_RELU) o[k] = fmaxf(o[k], 0.f);
        }
        const int ys = p.transposed ? (oy0 + y) * p.sh + py : oy0 + y;
        const int xs = p.transposed ? (ox0 + x) * p.sw + px : ox0 + x;
        __half2 h0 = __floats2half2_rn(o[0], o[1]), h1 = __floats2half2_rn(o[2], o[3]);
        *reinterpret_cast<uint2*>(p.out + (((size_t)b * p.Hout + ys) * p.Wout + xs) * p.Cout + n0 + n) =
            make_uint2(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1));
      }
      cluster_sync_all();                                          // the peers have read this CTA's partial: its shared memory may go
      return;
    }
    // (out-of-range pixels of ragged tiles need no masking: the TMA store below clips at the tensor-map bounds)
#pragma unroll
    for (int i = 0; i < BLOCK_N / 2; i += 2) {
      const int row = rbase + 8 * ((i >> 1) & 1);
      const int col = 8 * (i >> 2) + cq;
      // scale/shift/activation -> FP16 -> 128B-swizzled [128 pixels][64 channels] blocks; one TMA store per block writes full
      // 128-byte rows
      float v0 = fmaf(acc[i], s_scale[col], s_shift[col]);
      float v1 = fmaf(acc[i + 1], s_scale[col + 1], s_shift[col + 1]);
      if (p.act == ACT_LEAKY) { v0 = v0 > 0.f ? v0 : 0.2f * v0; v1 = v1 > 0.f ? v1 : 0.2f * v1; }
      else if (p.act == ACT_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
      uint8_t* blk = smem + (col >> 6) * (kBlockM * 128) + row * 128;
      *reinterpret_cast<__half2*>(blk + ((((col & 63) >> 3) ^ (row & 7)) << 4) + (col & 7) * 2) = __floats2half2_rn(v0, v1);
    }
    if (my_chunks > 0) {
      // generic-proxy smem writes -> visible to the async proxy; one thread hands the tile to the TMA unit
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      asm volatile("bar.sync 1, %0;" ::"n"(kTcConsumers) : "memory");
      if (threadIdx.x == 0) {
        const int xs = p.transposed ? ox0 * p.sw + px : ox0;
        const int ys = p.transposed ? oy0 * p.sh + py : oy0;
#pragma unroll
        for (int jb = 0; jb < BLOCK_N / 64; ++jb)
          asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                       ::"l"(&tmO), "r"(smem_u32(smem + jb * (kBlockM * 128))), "r"(n0 + jb * 64), "r"(xs), "r"(ys), "r"(b) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      }
    }
  }
}

// ------------------------------------------------------------------------------------ host side
static PFN_cuTensorMapEncodeTiled_v12000 g_encode = nullptr;
// g_clusters[ks]: clusters of (1, 1, ks) k_conv_tc CTAs the device holds at once (the smaller of the two kernel configurations)
static int g_clusters[kMaxSplits + 1] = {};

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
  RYK_CUDA(cudaFuncSetAttribute(RYK_TC_N128, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  RYK_CUDA(cudaFuncSetAttribute(RYK_TC_N64, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  if (g_clusters[1] == 0) {
    auto active = [](auto kernel, size_t smem, int ks) {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(1, 1, ks); cfg.blockDim = dim3(kTcThreads); cfg.dynamicSmemBytes = smem;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = 1; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = ks;
      cfg.attrs = at; cfg.numAttrs = 1;
      int n = 0;
      if (cudaOccupancyMaxActiveClusters(&n, kernel, &cfg) != cudaSuccess) { cudaGetLastError(); n = 0; }
      return n;
    };
    for (int ks = 1; ks <= kMaxSplits; ++ks)
      g_clusters[ks] = std::min(active(RYK_TC_N128, tc_smem_bytes<128, 3>(), ks), active(RYK_TC_N64, tc_smem_bytes<64, 4>(), ks));
    RYK_CHECK(g_clusters[1] > 0, "the tensor-core convolution kernel does not fit an SM");
  }
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
// K further than the same layer over every row (L.ksplit_tiles overrides the tile count this rule sees).  One tile's splits run as one
// thread-block cluster, and ks is lowered until the device holds all of the layer's clusters at once: a cluster is placed inside
// one GPC, so the CTA slots left over in each GPC do not add up (an H100 SXM holds 14 clusters of 16 and 30 of 8, fewer than its
// 264 slots suggest; a layer whose clusters do not all fit would run a second wave of them).
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
    if (ks > kMaxSplits) ks = kMaxSplits;
    if (ks < 1) ks = 1;
    while (ks > 1 && tiles > g_clusters[ks]) --ks;
    int cps = (total_chunks + ks - 1) / ks;
    ks = (total_chunks + cps - 1) / cps;                // every split owns at least one chunk
  }
  *tile_w = tw; *tile_h = th; *block_n = bn; *ksplit = ks;
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
  RYK_CHECK(L.band_y0 >= 0 && L.band_y0 % L.tile_h == 0 && L.band_y0 < layer_band_end(L) && layer_band_end(L) <= layer_class_rows(L) &&
            (layer_band_end(L) % L.tile_h == 0 || layer_band_end(L) == layer_class_rows(L)), "row band is not a range of whole tile rows");
  RYK_CHECK(L.skip_y1 == 0 || (!L.transposed && L.skip_y0 % L.tile_h == 0 && L.skip_y1 % L.tile_h == 0 && L.band_y0 <= L.skip_y0 &&
                               L.skip_y0 < L.skip_y1 && L.skip_y1 <= layer_band_end(L)),
            "skipped rows are not a range of whole tile rows inside the band of a convolution");
  L.tc_ready = true;
  return 0;
}

// Launch with the programmatic-stream-serialization attribute (see pdl_trigger / pdl_wait) and, for cluster_z > 1, in clusters of
// (1, 1, cluster_z) CTAs.
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, int cluster_z, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[0].val.programmaticStreamSerializationAllowed = 1;
  attr[1].id = cudaLaunchAttributeClusterDimension; attr[1].val.clusterDim.x = 1; attr[1].val.clusterDim.y = 1; attr[1].val.clusterDim.z = cluster_z;
  cfg.attrs = attr; cfg.numAttrs = cluster_z > 1 ? 2 : 1;
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
  p.out = (__half*)L.out;
  // blockIdx.z = class * ksplit + split: one cluster of ksplit consecutive z is one tile's splits, and a CTA's rank in it is its split
  dim3 grid(L.B * p.tiles_w * p.tiles_h, L.Cout / L.block_n, classes * L.ksplit);
  if (L.block_n == 128) RYK_CUDA(launch_pdl(RYK_TC_N128, grid, dim3(kTcThreads), tc_smem_bytes<128, 3>(), st, L.ksplit, L.tmA0, L.tmA1, L.tmB, L.tmO, p));
  else RYK_CUDA(launch_pdl(RYK_TC_N64, grid, dim3(kTcThreads), tc_smem_bytes<64, 4>(), st, L.ksplit, L.tmA0, L.tmA1, L.tmB, L.tmO, p));
  RYK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace ryk
