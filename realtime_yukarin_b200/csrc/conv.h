// conv.h -- convolution layer descriptors shared by the FP32 CUDA-core path (conv_direct.cu), the
// FP16 wgmma tensor-core path (conv_tc.cu) and the U-Net scheduler (unet.cu).
#pragma once
#include <cuda.h>

#include "common.cuh"

namespace ryk {

enum Act { ACT_NONE = 0, ACT_LEAKY = 1, ACT_RELU = 2 };
enum DType { DT_F32 = 0, DT_F16 = 1 };

constexpr int kMaxGroupVoices = 8;      // distinct voices of one mixed-voice group
constexpr int kMaxGroupBatch = 64;      // sessions of one group

// A layer's weights per batch item, as the kernels receive them (by value): batch item b reads entry voice_of[b] of each array.
// Every plan except a mixed-voice group's has one entry and voice_of all 0.
struct LayerWeights {
  const float* w[kMaxGroupVoices];                                  // [KH][KW][Cin][Cout] fp32 (CUDA-core kernels)
  const float* scale[kMaxGroupVoices];                              // [Cout] folded BN scale (1 when no BN)
  const float* shift[kMaxGroupVoices];                              // [Cout] folded bias / BN shift
  float host_scale[kMaxGroupVoices], host_shift[kMaxGroupVoices];   // Cout == 1 layers: the scalar scale / shift
  uint8_t voice_of[kMaxGroupBatch];
};
// Plans with more batch items than a group holds have one voice.
__host__ __device__ inline int item_voice(const LayerWeights& wt, int b) { return b < kMaxGroupBatch ? wt.voice_of[b] : 0; }
// The tensor-core kernel's weight tensor maps, one per voice (one __grid_constant__ kernel parameter).
struct TcWeightMaps { CUtensorMap m[kMaxGroupVoices]; };

// One conv / transposed-conv layer over NHWC activations (1-D nets use H = 1, KH = 1).
// The input is the channel-concatenation of up to two tensors (U-Net skip "concat by pointer").
struct ConvLayer {
  int transposed = 0;
  int B = 1, Hin = 1, Win = 1, Hout = 1, Wout = 1;
  int C0 = 0, C1 = 0, Cout = 0;           // Cin = C0 + C1
  int KH = 1, KW = 1, SH = 1, SW = 1, PH = 0, PW = 0;
  int act = ACT_NONE;
  // Output row band: the layer computes only class-local output rows [band_y0, band_y1) of every batch item (transposed layers:
  // output rows SH * band_y0 .. SH * band_y1 - 1).  The band is a range of whole tile rows (band_y1 may also be the last row);
  // band_y1 == 0 means every row.  See unet_derive_bands.
  int band_y0 = 0, band_y1 = 0;
  // Padded tail (encoder layers of a session's stage-2 plan; see unet_derive_tail): output rows [skip_y0, skip_y1) repeat the
  // representative row of their run and are not computed (whole tile rows; skip_y1 == 0: none).  Rows [run_y0, run_y1) of in0
  // repeat row run_y0: a load box wholly inside them reads from run_y0 instead (run_y1 == 0: no remapping).
  int skip_y0 = 0, skip_y1 = 0;
  int run_y0 = 0, run_y1 = 0;
  // device pointers
  const void* in0 = nullptr; const void* in1 = nullptr; int in_dtype = DT_F32;
  void* out = nullptr; int out_dtype = DT_F32;
  // weights of voices 0 .. n_voices - 1 (n_voices > 1 only in a mixed-voice group's stage-2 plan; see unet_plan_set_voices)
  int n_voices = 1;
  LayerWeights wt = {};
  bool host_scale_valid = false;          // Cout == 1 layers: scalar scale/shift mirrored on the host (wt.host_scale / host_shift)
  // tensor-core path (filled by tc_layer_prepare)
  const __half* w_tc[kMaxGroupVoices] = {};   // per voice; conv: [Cout][KH*KW*Cin]; deconv: [4 classes][Cout][4*Cin]
  const __half* w_frag = nullptr;         // 1-D k4 layers: mma.sync B-fragment order for the fused stage-1 kernel (s1_map.h)
  int ksplit = 1;                         // > 1: the K splits of one output tile run as one thread-block cluster
  int ksplit_tiles = 0;                   // > 0: split K as for a layer of this many output tiles instead of the band's own count
  CUtensorMap tmA0, tmA1, tmO;            // inputs, fp16 output
  TcWeightMaps tmB;                       // weights, per voice
  int tile_w = 0, tile_h = 0;             // pixel tile = tile_w x tile_h = 128
  int block_n = 0;
  bool tc_ready = false;
};

// class-local output rows of a layer (transposed convs run per output-parity class) and the end of its row band
inline int layer_class_rows(const ConvLayer& L) { return L.transposed ? L.Hin : L.Hout; }
inline int layer_band_end(const ConvLayer& L) { return L.band_y1 > 0 ? L.band_y1 : layer_class_rows(L); }
// output rows [*r0, *r1) of one batch item that the band covers
inline void layer_band_out_rows(const ConvLayer& L, int* r0, int* r1) {
  const int s = L.transposed ? L.SH : 1;
  *r0 = L.band_y0 * s;
  *r1 = layer_band_end(L) * s < L.Hout ? layer_band_end(L) * s : L.Hout;
}

// Weight repacking from the Chainer layouts the model files use:
//   conv   W: (Cout, Cin, KH, KW)      deconv W: (Cin, Cout, KH, KW)
int pack_weights_direct(const float* d_w_chainer, int transposed, int Cin, int Cout, int KH, int KW, float* d_out, cudaStream_t st);
int pack_weights_tc(const float* d_w_chainer, int transposed, int Cin, int Cout, int KH, int KW, int SH, int SW, __half* d_out, cudaStream_t st);

int conv_direct_run(const ConvLayer& L, cudaStream_t st);
bool conv_direct_band_supported(const ConvLayer& L);
// the first layer of stage-2 plans (k_conv3x3_cin1), which skips the padded tail in blocks of kCin1Rows output rows
bool conv_direct_cin1(const ConvLayer& L);
constexpr int kCin1Rows = 8;
// the CUDA-core kernels that read weights per batch item (LayerWeights::voice_of): the stage-2 edge layers of FP16 plans
bool conv_direct_per_item_weights(const ConvLayer& L);

bool tc_layer_eligible(const ConvLayer& L);
int tc_init();                                           // resolves cuTensorMapEncodeTiled, sets smem attributes
int tc_layer_prepare(ConvLayer& L, int num_sms);         // builds tensor maps, picks tiles / split-K (needs final pointers)
int tc_layer_weight_maps(ConvLayer& L);                  // (re)builds the weight maps of voices 0 .. n_voices - 1 of a prepared layer
int conv_tc_run(const ConvLayer& L, cudaStream_t st);
int tc_tile_rows(const ConvLayer& L);                    // class-local output rows per tile of the tensor-core kernel
int tc_tile_count(const ConvLayer& L);                   // output tiles (all classes, all N blocks) of the layer's band

// s1_fused.cu: the whole 1-D U-Net as one cluster kernel
int s1_pack_weights(const float* d_w_chainer, int transposed, int Cin, int Cout, __half* d_out, cudaStream_t st);
int s1_fused_init();
int s1_fused_cluster_size();                             // CTAs of the cluster the kernel runs on (<= 0: unavailable)

}  // namespace ryk
