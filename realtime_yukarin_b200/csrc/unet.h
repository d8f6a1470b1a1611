// unet.h -- U-Net containers (weights + per-shape plans).
#pragma once
#include <map>
#include <tuple>
#include <vector>

#include "conv.h"

namespace ryk {

struct Engine;

struct UNetLayerW {
  int transposed = 0, cin = 0, cout = 0, k = 3, s = 1, p = 1, act = 0;
  float* d_w_direct = nullptr;
  __half* d_w_tc = nullptr;
  __half* d_w_frag = nullptr;            // fused stage-1 kernel (1-D nets, k4 layers)
  float* d_scale = nullptr;
  float* d_shift = nullptr;
  float h_scale0 = 1.f, h_shift0 = 0.f;   // first channel's scale/shift (used by the Cout = 1 kernel)
  bool loaded = false;
};

struct UNetPlan {
  int B = 1, H = 1, W = 0, precision = 0;
  int keep_begin = 0, keep_len = 0;   // output rows of every batch item the plan computes (keep_len == 0: all); see unet_derive_bands
  int tail_begin = 0;                 // > 0: input rows >= tail_begin repeat one row, and the encoder skips them (unet_derive_tail)
  std::vector<ConvLayer> layers;
  void* arena = nullptr;    // one device allocation holding every buffer below
  std::vector<void*> buffers;          // enc[0..7], dec[0..6], d_in, d_out
  std::vector<size_t> buffer_bytes;
  void* d_in = nullptr;     // fp32 NHWC input  [B][H][W][in_ch]
  void* d_out = nullptr;    // fp32 NHWC output [B][H][W][out_ch]
  bool fused = false;       // 1-D FP16 plan that s1_fused.cu can run as one launch
};

struct UNet {
  int ndim = 2, in_ch = 1, out_ch = 1, base = 64;
  std::vector<UNetLayerW> layers;                                  // 0..7 encoder, 8..15 decoder
  // (B, H, W, precision, owner, keep_begin, keep_len, ksplit as for full layers, tail_begin)
  std::map<std::tuple<int, int, int, int, int, int, int, int, int>, UNetPlan*> plans;
};

UNet* unet_create(int ndim, int in_ch, int out_ch, int base);
void unet_destroy(UNet* n);
int unet_set_layer(Engine* e, UNet* n, int idx, const float* W, const float* scale, const float* shift);
// owner: 0 = the engine's shared plans (per-op host API, serialised on the engine stream); every session / group passes its own
// id so that concurrently running streams never share activation buffers.
// keep_len > 0 (2-D FP16 plans): the caller reads only output rows [keep_begin, keep_begin + keep_len) of every batch item, and
// the decoder computes only the row bands those rows depend on (unet_derive_bands); the other rows of d_out are not written.
// full_ksplit: each banded layer splits K as it would over every row (tests: bitwise comparison with the full plan).
// tail_begin > 0 (banded plans): the caller fills input rows [tail_begin, H) of every batch item with one and the same row (a
// session's padded window), and the encoder computes only one copy of the rows that depend on nothing else (unet_derive_tail).
int unet_get_plan(Engine* e, UNet* n, int B, int H, int W, int precision, UNetPlan** out, int owner = 0, int keep_begin = 0,
                  int keep_len = 0, bool full_ksplit = false, int tail_begin = 0);
void unet_release_owner(UNet* n, int owner);
// Per-batch-item weights of a mixed-voice group's plan (built on nets[0]): batch item b runs on the weights of nets[voice_of[b]].  The
// nets must have the same shape; the tile grid, K order and split-K stay those of the plan, so only the weights differ per item.
int unet_plan_set_voices(UNetPlan* p, const std::vector<const UNet*>& nets, const std::vector<int>& voice_of);
// Fill the geometry of layer i of net n for a (B, H, W) input (shapes, kernel, stride, padding, channels; no pointers).
void unet_layer_shape(const UNet* n, int i, int B, int H, int W, ConvLayer& L);
// Row bands of the 2-D decoder (layers 8..15) for a caller that reads output rows [keep_begin, keep_begin + keep_len): writes
// band_y0 / band_y1 of those layers, rounded out to each layer's tile rows.  Layers 0..7 and every layer whose band covers all its
// rows stay full.
void unet_derive_bands(std::vector<ConvLayer>& layers, int keep_begin, int keep_len);
// Padded tail of the 2-D encoder (layers 0..6, after unet_derive_bands) for an input whose rows [tail_begin, H) are equal: writes
// skip_y0 / skip_y1 of the layers that skip rows and run_y0 / run_y1 of the layers that read them.
void unet_derive_tail(std::vector<ConvLayer>& layers, int tail_begin);
// smallest row range [*begin, *begin + *len) that holds the n ranges [begins[i], begins[i] + lens[i])
void keep_hull(int n, const int* begins, const int* lens, int* begin, int* len);
int unet_forward(Engine* e, UNetPlan* p, cudaStream_t st, int first_layer = 0, int last_layer = 15);
// s1_fused.cu
bool s1_fused_eligible(const UNet* n, const UNetPlan* p);
int s1_fused_run(Engine* e, const UNetPlan* p, cudaStream_t st);

}  // namespace ryk
