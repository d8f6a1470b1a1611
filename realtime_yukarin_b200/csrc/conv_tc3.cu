// conv_tc3.cu -- "halo" wgmma kernel for the k4 s2 p1 2-D layers of the stage-2 U-Net (sm_90a).
//
// The per-tap kernel of conv_tc.cu stages one A tile (128 pixels x 64 channels) per tap.  This kernel cuts the A bytes per FLOP:
//   * HALO ROWS.  An output tile is tile_h x tile_w pixels with tile_w = 8 or 16, so one image row of the tile is a whole number of
//     8-row swizzle atoms (1024 B).  The two taps of a k4 s2 conv that share a column tap and a row parity (ky = 0 / 2 or 1 / 3)
//     read the SAME strided input rows shifted by one; the two row taps of a transposed-conv parity class likewise.  One TMA box
//     with tile_h + 1 rows therefore serves both taps: the second tap's wgmma descriptor simply starts tile_w * 128 B further
//     (1024-B aligned, so the 128B-swizzle phase is unchanged).
//   * MT STACKED M TILES (RYK_TC3_MT = 2): a box of 2 tile_h + 1 rows and 256 pixels per CTA share every weight tile.
//   * PERSISTENT (one CTA per SM, tiles round-robin; the smem ring streams across tile boundaries and the epilogue has its own
//     staging buffer, so the next tile's loads are in flight during the epilogue) or ONE tile per CTA (RYK_TC3_ONE = 2).
// One stage = one halo box + the two weight tiles (BLOCK_N x 64) of the taps it serves.
// Roles: warp 8 = TMA producer; warpgroups 0 / 1 = MMA + epilogue, warpgroup g owns pixel rows [64 MT g, 64 MT (g + 1)) of the tile.
#include <cuda.h>
#include <cudaTypedefs.h>
#include <stdlib.h>

#include "conv.h"
#include "tc_ptx.cuh"

namespace ryk {

struct HaloParams {
  int transposed, B, Cout, Hc, Wc;            // class-local output grid Hc x Wc
  int tile_w, tile_h, tiles_w, tiles_hs;      // tiles_hs: super tiles (MT stacked tiles) along H
  int n_tiles, classes_w, classes, chunks0, chunks1, act, total_tiles;
  uint32_t box_bytes;                         // (MT tile_h + 1) tile_w 128
  const float* scale; const float* shift;
};

template <int BLOCK_N, int MT, int kStages> struct HaloSmem {
  static constexpr uint32_t kA = MT * 16384 + 2048;                  // largest halo box (tile_w 16)
  static constexpr uint32_t kB = BLOCK_N * kBlockK * 2;              // one weight tile
  static constexpr uint32_t kStage = kA + 2 * kB;
  static constexpr uint32_t kStaging = MT * (BLOCK_N / 64) * 16384;  // [M tile][64-channel block][128 pixels][128 B]
  static constexpr size_t bytes() { return (size_t)kStages * kStage + kStaging + 2 * kStages * 8 + 1024; }
};

template <int BLOCK_N, int MT, int kStages>
__global__ void __launch_bounds__(kTcThreads, 1)
k_conv_halo(const __grid_constant__ CUtensorMap tA0, const __grid_constant__ CUtensorMap tA1, const __grid_constant__ CUtensorMap tmB,
            const __grid_constant__ CUtensorMap tO, const HaloParams p) {
  using S = HaloSmem<BLOCK_N, MT, kStages>;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* staging = smem + kStages * S::kStage;
  uint64_t* full_bar = (uint64_t*)(staging + S::kStaging);
  uint64_t* empty_bar = full_bar + kStages;
  const int warp = threadIdx.x >> 5;
  const int nbox = p.transposed ? 2 : 8;                 // halo boxes per channel chunk: deconv 2 column taps; conv 4 columns x 2 row parities
  const int chunks = p.chunks0 + p.chunks1;
  const int per_tile = chunks * nbox;
  pdl_trigger();
  if (threadIdx.x == kTcConsumers) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tA0) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tmB) : "memory");
    if (p.chunks1 > 0) asm volatile("prefetch.tensormap [%0];" ::"l"(&tA1) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&tO) : "memory");
    for (int i = 0; i < kStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], kTcConsumers / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();

  // tile t -> class-local origin of the super tile, image, first output channel, parity class (m fastest: co-running CTAs share weights)
  auto decode = [&](int t, int& ox0, int& oy0, int& b, int& n0, int& cls) {
    ox0 = (t % p.tiles_w) * p.tile_w; t /= p.tiles_w;
    oy0 = (t % p.tiles_hs) * (MT * p.tile_h); t /= p.tiles_hs;
    b = t % p.B; t /= p.B;
    n0 = (t % p.n_tiles) * BLOCK_N; cls = t / p.n_tiles;
  };

  if (warp == kTcConsumers / 32) {
    // ===== TMA producer =====
    int it = 0;
    for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
      int ox0, oy0, b, n0, cls;
      decode(t, ox0, oy0, b, n0, cls);
      const int py = cls / p.classes_w, px = cls % p.classes_w;
      for (int q = 0; q < per_tile; ++q, ++it) {
        const int s = it % kStages;
        mbar_wait(&empty_bar[s], ((it / kStages) & 1) ^ 1);
        const int cc = q / nbox, bx = q % nbox;
        int ix, iy, tap1, tap2;
        if (!p.transposed) {             // taps (r, tx) and (r + 2, tx): input rows 2 oy + r - 1 and the next strided row
          const int tx = bx & 3, r = bx >> 2;
          ix = ox0 * 2 + tx - 1; iy = oy0 * 2 + r - 1; tap1 = r * 4 + tx; tap2 = (r + 2) * 4 + tx;
        } else {                         // class (py, px), taps (0, dx) and (1, dx): input rows oy - 1 + py and the next row
          ix = ox0 + bx - 1 + px; iy = oy0 - 1 + py; tap1 = bx; tap2 = 2 + bx;
        }
        uint8_t* st = smem + s * S::kStage;
        if (elect_one()) {
          mbar_expect_tx(&full_bar[s], p.box_bytes + 2 * S::kB);
          if (cc < p.chunks0) tma_load_4d(st, &tA0, &full_bar[s], cc * kBlockK, ix, iy, b);
          else tma_load_4d(st, &tA1, &full_bar[s], (cc - p.chunks0) * kBlockK, ix, iy, b);
          tma_load_2d(st + S::kA, &tmB, &full_bar[s], (tap1 * chunks + cc) * kBlockK, cls * p.Cout + n0);
          tma_load_2d(st + S::kA + S::kB, &tmB, &full_bar[s], (tap2 * chunks + cc) * kBlockK, cls * p.Cout + n0);
        }
      }
    }
  } else if (warp < kTcConsumers / 32) {
    // ===== MMA + epilogue =====
    const int g = threadIdx.x >> 7, wl = warp & 3, lane = threadIdx.x & 31;
    float acc[MT][BLOCK_N / 2];
#pragma unroll
    for (int j = 0; j < MT; ++j)
#pragma unroll
      for (int i = 0; i < BLOCK_N / 2; ++i) acc[j][i] = 0.f;
#pragma unroll
    for (int j = 0; j < MT; ++j) wgmma_fence_acc(acc[j]);
    int it = 0;
    for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
      int ox0, oy0, b, n0, cls;
      decode(t, ox0, oy0, b, n0, cls);
      const int py = cls / p.classes_w, px = cls % p.classes_w;
      for (int q = 0; q < per_tile; ++q, ++it) {
        const int s = it % kStages;
        mbar_wait(&full_bar[s], (it / kStages) & 1);
        const uint8_t* st = smem + s * S::kStage;
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 2; ++tap) {
          const uint32_t abase = smem_u32(st) + (uint32_t)(tap * p.tile_w * 128) + (uint32_t)(g * 64 * MT * 128);
          const uint64_t bdesc = make_sw128_desc(smem_u32(st + S::kA + tap * S::kB));
#pragma unroll
          for (int j = 0; j < MT; ++j) {
            const uint64_t adesc = make_sw128_desc(abase + (uint32_t)(j * 64 * 128));
#pragma unroll
            for (int k = 0; k < kBlockK / kMmaK; ++k) {
              if constexpr (BLOCK_N == 128) wgmma_m64n128(acc[j], adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2));
              else wgmma_m64n64(acc[j], adesc + (uint64_t)(k * 2), bdesc + (uint64_t)(k * 2));
            }
          }
        }
        wgmma_commit();
        wgmma_wait<1>();
#pragma unroll
        for (int j = 0; j < MT; ++j) wgmma_fence_acc(acc[j]);
        if (q > 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty_bar[(it - 1) % kStages]); }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int j = 0; j < MT; ++j) wgmma_fence_acc(acc[j]);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[(it - 1) % kStages]);
      // epilogue: the previous tile's TMA stores must have finished reading the staging buffer
      if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      asm volatile("bar.sync 1, %0;" ::"n"(kTcConsumers) : "memory");
      const int cq = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < MT; ++j) {
#pragma unroll
        for (int i = 0; i < BLOCK_N / 2; i += 2) {
          const int row = g * 64 * MT + j * 64 + wl * 16 + (lane >> 2) + 8 * ((i >> 1) & 1);       // pixel row of the super tile
          const int col = 8 * (i >> 2) + cq;
          float v0 = fmaf(acc[j][i], __ldg(p.scale + n0 + col), __ldg(p.shift + n0 + col));
          float v1 = fmaf(acc[j][i + 1], __ldg(p.scale + n0 + col + 1), __ldg(p.shift + n0 + col + 1));
          if (p.act == ACT_LEAKY) { v0 = v0 > 0.f ? v0 : 0.2f * v0; v1 = v1 > 0.f ? v1 : 0.2f * v1; }
          else if (p.act == ACT_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
          const int mtile = row >> 7, r = row & 127;
          uint8_t* blk = staging + (mtile * (BLOCK_N / 64) + (col >> 6)) * 16384 + r * 128;
          *reinterpret_cast<__half2*>(blk + ((((col & 63) >> 3) ^ (r & 7)) << 4) + (col & 7) * 2) = __floats2half2_rn(v0, v1);
          acc[j][i] = 0.f; acc[j][i + 1] = 0.f;
        }
        wgmma_fence_acc(acc[j]);
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      asm volatile("bar.sync 1, %0;" ::"n"(kTcConsumers) : "memory");
      if (threadIdx.x == 0) {
        // out-of-range pixels of ragged tiles are clipped by the tensor map
        for (int mtile = 0; mtile < MT; ++mtile) {
          const int oy = oy0 + mtile * p.tile_h;
          const int xs = p.transposed ? ox0 * 2 + px : ox0, ys = p.transposed ? oy * 2 + py : oy;
          for (int jb = 0; jb < BLOCK_N / 64; ++jb)
            asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                         ::"l"(&tO), "r"(smem_u32(staging + (mtile * (BLOCK_N / 64) + jb) * 16384)), "r"(n0 + jb * 64), "r"(xs), "r"(ys), "r"(b)
                         : "memory");
        }
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
    }
    if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  }
}

// ------------------------------------------------------------------------------------ host side
#define RYK_HALO_VARIANTS(X) X(128, 1, 3) X(128, 1, 2) X(128, 2, 2) X(64, 1, 3) X(64, 1, 2) X(64, 2, 3) X(64, 2, 2)

int tc3_init() {
#define RYK_HALO_ATTR(BN, MT, ST) \
  RYK_CUDA(cudaFuncSetAttribute(k_conv_halo<BN, MT, ST>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)HaloSmem<BN, MT, ST>::bytes()));
  RYK_HALO_VARIANTS(RYK_HALO_ATTR)
#undef RYK_HALO_ATTR
  return 0;
}

static int t3_env(const char* name, int dflt) { const char* v = getenv(name); return v ? atoi(v) : dflt; }

// RYK_TC3: 0 (default) = never, 1 = where every CTA gets at least three tiles (or one-tile mode is forced), 2 = wherever the shape
// allows (tests).  RYK_TC3_TW: tile width 8 (default) or 16; RYK_TC3_MT: stacked M tiles 1 (default) or 2; RYK_TC3_DEPTH: 1 (default)
// = three stages where they fit, 0 = two; RYK_TC3_ONE: 0 = persistent, 2 = one tile per CTA, 1 (default) = one tile per CTA when there
// are fewer than three tiles per SM.  Read at every plan so that a test can switch them.  Off by default: not measured to be faster
// than the per-tap kernel on H100.
bool tc3_layer_config(const ConvLayer& L, int num_sms, ConvLayer::Halo* cfg) {
  const int mode = t3_env("RYK_TC3", 0);
  if (mode <= 0 || !tc_layer_eligible(L)) return false;
  if (!(L.KH == 4 && L.KW == 4 && L.SH == 2 && L.SW == 2)) return false;      // 2-D layers only
  const int tw = t3_env("RYK_TC3_TW", 8) == 16 ? 16 : 8, th = kBlockM / tw;
  const int mt = t3_env("RYK_TC3_MT", 1) == 2 ? 2 : 1;
  const int Wc = L.transposed ? L.Win : L.Wout, Hc = L.transposed ? L.Hin : L.Hout;
  const int bn = L.Cout >= 128 ? 128 : 64;
  const int tiles = L.B * ((Wc + tw - 1) / tw) * ((Hc + mt * th - 1) / (mt * th)) * (L.Cout / bn) * (L.transposed ? 4 : 1);
  const int one_env = t3_env("RYK_TC3_ONE", 1);
  if (mode == 1 && one_env != 2 && tiles < 3 * num_sms) return false;
  if (cfg) {
    cfg->tile_w = tw; cfg->tile_h = th; cfg->mt = mt;
    cfg->one = one_env == 2 || (one_env == 1 && tiles < 3 * num_sms);
    cfg->stages = (t3_env("RYK_TC3_DEPTH", 1) >= 1 && !(bn == 128 && mt == 2)) ? 3 : 2;
  }
  return true;
}

static int t3_map(PFN_cuTensorMapEncodeTiled_v12000 encode, CUtensorMap* m, const void* ptr, int C, int W, int H, int B, int box_w, int box_h,
                  int stride) {
  cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)C * 2, (cuuint64_t)W * C * 2, (cuuint64_t)H * W * C * 2};
  cuuint32_t box[4] = {(cuuint32_t)kBlockK, (cuuint32_t)(box_w * stride), (cuuint32_t)(box_h * stride), 1};
  cuuint32_t estr[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
  CUresult r = encode(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled(halo) failed: " + std::to_string((int)r)); return -1; }
  return 0;
}

int tc3_layer_prepare(ConvLayer& L, PFN_cuTensorMapEncodeTiled_v12000 encode) {
  const auto& h = L.t3;
  const int sa = L.transposed ? 1 : 2;                     // conv: strided input rows / columns; deconv: dense input
  if (t3_map(encode, &L.t3A0, L.in0, L.C0, L.Win, L.Hin, L.B, h.tile_w, h.mt * h.tile_h + 1, sa)) return -1;
  if (L.C1 > 0) { if (t3_map(encode, &L.t3A1, L.in1, L.C1, L.Win, L.Hin, L.B, h.tile_w, h.mt * h.tile_h + 1, sa)) return -1; }
  else L.t3A1 = L.t3A0;
  // deconv classes write every other output pixel (element strides 2)
  return t3_map(encode, &L.t3O, L.out, L.Cout, L.Wout, L.Hout, L.B, h.tile_w, h.tile_h, L.transposed ? 2 : 1);
}

int conv_tc3_run(const ConvLayer& L, cudaStream_t st, bool pdl) {
  const auto& h = L.t3;
  HaloParams p;
  p.transposed = L.transposed; p.B = L.B; p.Cout = L.Cout;
  p.Hc = L.transposed ? L.Hin : L.Hout; p.Wc = L.transposed ? L.Win : L.Wout;
  p.tile_w = h.tile_w; p.tile_h = h.tile_h;
  p.tiles_w = (p.Wc + h.tile_w - 1) / h.tile_w; p.tiles_hs = (p.Hc + h.mt * h.tile_h - 1) / (h.mt * h.tile_h);
  const int bn = L.Cout >= 128 ? 128 : 64;
  p.n_tiles = L.Cout / bn;
  p.classes_w = L.transposed ? 2 : 1; p.classes = L.transposed ? 4 : 1;
  p.chunks0 = L.C0 / kBlockK; p.chunks1 = L.C1 / kBlockK;
  p.act = L.act; p.scale = L.scale; p.shift = L.shift;
  p.total_tiles = L.B * p.tiles_w * p.tiles_hs * p.n_tiles * p.classes;
  p.box_bytes = (uint32_t)((h.mt * h.tile_h + 1) * h.tile_w * 128);
  int num_sms = 132;
  cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, 0);
  const int grid = h.one ? p.total_tiles : (p.total_tiles < num_sms ? p.total_tiles : num_sms);
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(kTcThreads); cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
  cudaError_t err = cudaErrorInvalidConfiguration;
#define RYK_HALO_LAUNCH(BN, MT, ST) \
  else if (bn == BN && h.mt == MT && h.stages == ST) { \
    cfg.dynamicSmemBytes = HaloSmem<BN, MT, ST>::bytes(); \
    err = cudaLaunchKernelEx(&cfg, k_conv_halo<BN, MT, ST>, L.t3A0, L.t3A1, L.tmB, L.t3O, p); \
  }
  if (false) {}
  RYK_HALO_VARIANTS(RYK_HALO_LAUNCH)
#undef RYK_HALO_LAUNCH
  RYK_CUDA(err);
  RYK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace ryk
