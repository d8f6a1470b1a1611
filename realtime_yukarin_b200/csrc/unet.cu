// unet.cu -- the two pix2pix-style U-Nets of the hot path as static layer schedules over
// device-resident weights and per-shape activation plans.
//   stage 1: yukarin acoustic-feature converter, 1-D (SURVEY a10 / App. A.6):  (T, 9) -> (T, 9)
//   stage 2: become-yukarin spectrogram super-resolution, 2-D (a13 / App. A.7): (T, 512) -> (T, 512)
// Topology (both): enc c0 = conv k3 s1 p1 + LeakyReLU(0.2); enc c1..c7 = conv k4 s2 p1 + BN + LeakyReLU;
// dec c0..c6 = deconv k4 s2 p1 + BN + ReLU with skip concat (by pointer) before c1..c7;
// dec c7 = conv k3 s1 p1.  BatchNorm (eval, eps 2e-5) and biases arrive folded into scale/shift.
#include <algorithm>
#include <vector>

#include "conv.h"
#include "engine.h"
#include "unet.h"

namespace ryk {

static int level_channels(int base, int level) {   // encoder output channels at level 0..7
  static const int mult[8] = {1, 2, 4, 8, 8, 8, 8, 8};
  return base * mult[level];
}
static int dec_out_channels(int base, int i) {     // decoder c0..c6 output channels
  static const int mult[7] = {8, 8, 8, 8, 4, 2, 1};
  return base * mult[i];
}

// The layer shapes are restated in Python (engine._unet_layer_shapes, which checks the model files of voices >= 1); change both together.
UNet* unet_create(int ndim, int in_ch, int out_ch, int base) {
  UNet* n = new UNet();
  n->ndim = ndim; n->in_ch = in_ch; n->out_ch = out_ch; n->base = base;
  n->layers.resize(16);
  for (int i = 0; i < 16; ++i) {
    UNetLayerW& L = n->layers[i];
    if (i == 0) { L.transposed = 0; L.cin = in_ch; L.cout = base; L.k = 3; L.s = 1; L.p = 1; L.act = ACT_LEAKY; }
    else if (i < 8) { L.transposed = 0; L.cin = level_channels(base, i - 1); L.cout = level_channels(base, i); L.k = 4; L.s = 2; L.p = 1; L.act = ACT_LEAKY; }
    else if (i < 15) {
      int d = i - 8;
      L.transposed = 1; L.k = 4; L.s = 2; L.p = 1; L.act = ACT_RELU;
      L.cout = dec_out_channels(base, d);
      L.cin = d == 0 ? level_channels(base, 7) : dec_out_channels(base, d - 1) + level_channels(base, 7 - d);
    } else { L.transposed = 0; L.cin = 2 * base; L.cout = out_ch; L.k = 3; L.s = 1; L.p = 1; L.act = ACT_NONE; }
  }
  return n;
}

static void free_plan(UNetPlan* p) {
  if (p->arena) cudaFree(p->arena);          // every buffer of the plan lives in it
  delete p;
}

void unet_destroy(UNet* n) {
  if (!n) return;
  for (auto& L : n->layers) {
    if (L.d_w_direct) cudaFree(L.d_w_direct);
    if (L.d_w_tc) cudaFree(L.d_w_tc);
    if (L.d_w_frag) cudaFree(L.d_w_frag);
    if (L.d_scale) cudaFree(L.d_scale);
    if (L.d_shift) cudaFree(L.d_shift);
  }
  for (auto& kv : n->plans) free_plan(kv.second);
  delete n;
}

// Drop every plan a destroyed session / group owned (call with its streams idle).
void unet_release_owner(UNet* n, int owner) {
  if (!n || owner == 0) return;
  for (auto it = n->plans.begin(); it != n->plans.end();) {
    if (std::get<4>(it->first) == owner) { free_plan(it->second); it = n->plans.erase(it); }
    else ++it;
  }
}

// W in the model file's (Chainer) layout: conv (Cout, Cin, k[, k]), deconv (Cin, Cout, k[, k]); host pointers.
int unet_set_layer(Engine* e, UNet* n, int idx, const float* W, const float* scale, const float* shift) {
  RYK_CHECK(idx >= 0 && idx < 16, "layer index out of range");
  UNetLayerW& L = n->layers[idx];
  int KH = n->ndim == 2 ? L.k : 1, KW = L.k;
  size_t nw = (size_t)L.cin * L.cout * KH * KW;
  float* d_tmp = nullptr;
  RYK_CUDA(cudaMalloc(&d_tmp, nw * sizeof(float)));
  RYK_CUDA(cudaMemcpyAsync(d_tmp, W, nw * sizeof(float), cudaMemcpyHostToDevice, e->stream));
  if (!L.d_w_direct) RYK_CUDA(cudaMalloc(&L.d_w_direct, nw * sizeof(float)));
  if (pack_weights_direct(d_tmp, L.transposed, L.cin, L.cout, KH, KW, L.d_w_direct, e->stream)) return -1;
  bool tc_shape = L.k == 4 && L.cin % 64 == 0 && L.cout % 64 == 0;
  if (tc_shape) {
    if (!L.d_w_tc) RYK_CUDA(cudaMalloc(&L.d_w_tc, nw * sizeof(__half)));
    if (pack_weights_tc(d_tmp, L.transposed, L.cin, L.cout, KH, KW, n->ndim == 2 ? L.s : 1, L.s, L.d_w_tc, e->stream)) return -1;
  }
  if (n->ndim == 1 && L.k == 4 && L.s == 2 && L.cin % 64 == 0 && L.cout % 16 == 0) {
    if (!L.d_w_frag) RYK_CUDA(cudaMalloc(&L.d_w_frag, nw * sizeof(__half)));
    if (s1_pack_weights(d_tmp, L.transposed, L.cin, L.cout, L.d_w_frag, e->stream)) return -1;
  }
  if (!L.d_scale) RYK_CUDA(cudaMalloc(&L.d_scale, L.cout * sizeof(float)));
  if (!L.d_shift) RYK_CUDA(cudaMalloc(&L.d_shift, L.cout * sizeof(float)));
  RYK_CUDA(cudaMemcpyAsync(L.d_scale, scale, L.cout * sizeof(float), cudaMemcpyHostToDevice, e->stream));
  RYK_CUDA(cudaMemcpyAsync(L.d_shift, shift, L.cout * sizeof(float), cudaMemcpyHostToDevice, e->stream));
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  RYK_CUDA(cudaFree(d_tmp));
  L.h_scale0 = scale[0]; L.h_shift0 = shift[0];
  L.loaded = true;
  return 0;
}

void unet_layer_shape(const UNet* n, int i, int B, int H, int W, ConvLayer& L) {
  const UNetLayerW& LW = n->layers[i];
  auto lvlH = [&](int l) { return n->ndim == 2 ? H >> l : 1; };
  auto lvlW = [&](int l) { return W >> l; };
  L.transposed = LW.transposed; L.B = B; L.Cout = LW.cout; L.act = LW.act;
  L.KH = n->ndim == 2 ? LW.k : 1; L.KW = LW.k;
  L.SH = n->ndim == 2 ? LW.s : 1; L.SW = LW.s;
  L.PH = n->ndim == 2 ? LW.p : 0; L.PW = LW.p;
  if (i == 0) {
    L.Hin = lvlH(0); L.Win = lvlW(0); L.Hout = lvlH(0); L.Wout = lvlW(0); L.C0 = n->in_ch; L.C1 = 0;
  } else if (i < 8) {
    L.Hin = lvlH(i - 1); L.Win = lvlW(i - 1); L.Hout = lvlH(i); L.Wout = lvlW(i); L.C0 = LW.cin; L.C1 = 0;
  } else if (i < 15) {
    int d = i - 8;
    L.Hin = lvlH(7 - d); L.Win = lvlW(7 - d); L.Hout = lvlH(6 - d); L.Wout = lvlW(6 - d);
    if (d == 0) { L.C0 = LW.cin; L.C1 = 0; }
    else { L.C0 = dec_out_channels(n->base, d - 1); L.C1 = level_channels(n->base, 7 - d); }
  } else {
    L.Hin = lvlH(0); L.Win = lvlW(0); L.Hout = lvlH(0); L.Wout = lvlW(0); L.C0 = n->base; L.C1 = n->base;
  }
}

// Walks back from the last layer.  Layer i must produce output rows [lo, hi); its band is the class-local rows those come from
// (transposed k4 s2 p1: output row 2m + py is class-local row m), rounded out to whole tile rows of the kernel that runs the layer
// (the tensor-core tile grid; one row for the 3x3 CUDA-core layer).  The rows the next layer down must produce are then the input
// rows the ROUNDED band reads, so every row that a computed tile reads has itself been computed.  Tiles keep their place in the
// layer's tile grid, so each computed pixel is summed exactly as in the full layer (same tile, same K order).
void unet_derive_bands(std::vector<ConvLayer>& layers, int keep_begin, int keep_len) {
  int lo = keep_begin, hi = keep_begin + keep_len;
  for (int i = 15; i >= 8; --i) {
    ConvLayer& L = layers[i];
    const int rows = layer_class_rows(L);
    const int th = L.transposed ? tc_tile_rows(L) : 1;
    const int m0 = L.transposed ? lo / L.SH : lo, m1 = L.transposed ? (hi - 1) / L.SH + 1 : hi;
    const int y0 = m0 / th * th, y1 = std::min(rows, (m1 + th - 1) / th * th);
    if (y0 == 0 && y1 == rows) { L.band_y0 = 0; L.band_y1 = 0; }
    else { L.band_y0 = y0; L.band_y1 = y1; }
    if (L.transposed) {   // class-local row m of parity py reads input rows m - 1 + py + ty, ty in {0, 1} (k4 s2 p1); m (k1 s1 p0)
      lo = L.SH == 2 ? y0 - 1 : y0;
      hi = L.SH == 2 ? y1 + 1 : y1;
    } else {
      lo = y0 * L.SH - L.PH;
      hi = (y1 - 1) * L.SH - L.PH + L.KH;
    }
    lo = std::max(lo, 0); hi = std::min(hi, L.Hin);
  }
}

static int floor_div(int a, int b) { return a >= 0 ? a / b : -((-a + b - 1) / b); }
static int round_up(int a, int m) { return -floor_div(-a, m) * m; }
static int round_down(int a, int m) { return floor_div(a, m) * m; }

// rows [*r0, *r1) of the output of encoder layer i (0..6) that the decoder reads: layer 15 - i takes it as its second source, over the
// rows its band reads (3x3 s1 p1 conv and k4 s2 p1 transposed conv alike: class-local row m reads rows m - 1 .. m + 1)
static void decoder_reads(const std::vector<ConvLayer>& layers, int i, int* r0, int* r1) {
  const ConvLayer& D = layers[15 - i];
  *r0 = std::max(D.band_y0 - 1, 0);
  *r1 = std::min(layer_band_end(D) + 1, D.Hin);
}

// Rows [Tw, H) of the input all hold one vector (the padded tail of a session's window).  Walking forward, each encoder layer's
// output rows that read only such rows form a run [lo, hi] of equal rows: a conv of stride s, padding p and k taps maps the run
// [lo, hi] of its input to the output rows o with o s - p >= lo and o s - p + k - 1 <= hi.
// Walking back from layer 6, layer i skips whole tile rows [a, b) of its run (rows of kCin1Rows for layer 0).  Layer i + 1 reads
// a load box of rows iy, iy + 2, .., iy + 2 (tile_h - 1); a box wholly inside the run reads the first rows of the run instead (the
// representative rows, which stay computed), so [a, b) starts after them.  Every other box of a tile that layer i + 1 computes
// crosses the end of the run and must miss [a, b), and so must the rows the decoder reads.  Rows of equal inputs get equal sums
// (same kernel, tile row position and K order), so the remapped boxes load exactly the values the skipped rows would have held.
void unet_derive_tail(std::vector<ConvLayer>& layers, int tail_begin) {
  int lo[8], hi[8];
  int l = tail_begin, h = layers[0].Hin - 1;
  for (int i = 0; i < 8; ++i) {
    const ConvLayer& L = layers[i];
    l = -floor_div(-(l + L.PH), L.SH);
    h = floor_div(h + L.PH - L.KH + 1, L.SH);
    lo[i] = l; hi[i] = h;
  }
  for (int i = 6; i >= 0; --i) {
    ConvLayer& L = layers[i];
    ConvLayer& N = layers[i + 1];
    if (lo[i] > hi[i]) continue;
    const int th = i == 0 ? kCin1Rows : tc_tile_rows(L);
    const int nth = tc_tile_rows(N), span = N.SH * (nth - 1) + 1;
    int a = round_up(lo[i] + span, th), b = round_down(hi[i] + 1, th);
    for (int t = 0; t * nth < N.Hout; ++t) {
      if (t * nth >= N.skip_y0 && t * nth < N.skip_y1) continue;        // not computed
      for (int ty = 0; ty < N.KH; ++ty) {
        const int s = t * nth * N.SH + ty - N.PH, e = s + span - 1;
        if ((s >= lo[i] && e <= hi[i]) || e < a || s >= b) continue;
        if (s >= a) b = round_down(s, th); else a = round_up(e + 1, th);
      }
    }
    int r0, r1;
    decoder_reads(layers, i, &r0, &r1);
    if (r0 < b && r1 > a) {
      if (round_down(r0, th) - a >= b - round_up(r1, th)) b = round_down(r0, th);
      else a = round_up(r1, th);
    }
    if (a < b) { L.skip_y0 = a; L.skip_y1 = b; N.run_y0 = lo[i]; N.run_y1 = hi[i] + 1; }
  }
}

void keep_hull(int n, const int* begins, const int* lens, int* begin, int* len) {
  int lo = begins[0], hi = begins[0] + lens[0];
  for (int i = 1; i < n; ++i) { lo = std::min(lo, begins[i]); hi = std::max(hi, begins[i] + lens[i]); }
  *begin = lo; *len = hi - lo;
}

// Plan for a (batch, H, W) input; H = 1 for 1-D nets. precision: 0 = FP32 everywhere, 1 = FP16 activations + wgmma.
int unet_get_plan(Engine* e, UNet* n, int B, int H, int W, int precision, UNetPlan** out, int owner, int keep_begin, int keep_len,
                  bool full_ksplit, int tail_begin) {
  for (auto& L : n->layers) RYK_CHECK(L.loaded, "U-Net layer weights not loaded");
  if (keep_len > 0) RYK_CHECK(keep_begin >= 0 && keep_begin + keep_len <= H, "kept rows outside the U-Net input");
  if (keep_len <= 0 || (keep_begin == 0 && keep_len == H)) { keep_begin = 0; keep_len = 0; full_ksplit = false; }
  if (keep_len == 0 || tail_begin <= 0 || tail_begin >= H) tail_begin = 0;     // the full decoder reads every encoder row
  auto key = std::make_tuple(B, H, W, precision, owner, keep_begin, keep_len, full_ksplit ? 1 : 0, tail_begin);
  auto it = n->plans.find(key);
  if (it != n->plans.end()) { *out = it->second; return 0; }
  RYK_CHECK(W % 128 == 0 && (n->ndim == 1 || H % 128 == 0), "U-Net input extent must be a multiple of 128");
  UNetPlan* p = new UNetPlan();
  p->B = B; p->H = H; p->W = W; p->precision = precision;
  int num_sms = 132;
  cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, e->device);
  const int act_dt = precision ? DT_F16 : DT_F32;
  const size_t esz = precision ? 2 : 4;
  auto lvlH = [&](int l) { return n->ndim == 2 ? H >> l : 1; };
  auto lvlW = [&](int l) { return W >> l; };
  p->layers.resize(16);
  for (int i = 0; i < 16; ++i) {
    const UNetLayerW& LW = n->layers[i];
    ConvLayer& L = p->layers[i];
    unet_layer_shape(n, i, B, H, W, L);
    L.wt.w[0] = LW.d_w_direct; L.w_tc[0] = LW.d_w_tc; L.w_frag = LW.d_w_frag; L.wt.scale[0] = LW.d_scale; L.wt.shift[0] = LW.d_shift;
    L.host_scale_valid = true; L.wt.host_scale[0] = LW.h_scale0; L.wt.host_shift[0] = LW.h_shift0;
    L.in_dtype = act_dt; L.out_dtype = act_dt;
    if (i == 0) L.in_dtype = DT_F32;
    if (i == 15) L.out_dtype = DT_F32;
    L.tc_ready = false;
  }
  // The decoder computes a row band only where every layer of it runs on a kernel that supports one.
  bool bandable = keep_len > 0 && n->ndim == 2 && precision == 1 && conv_direct_band_supported(p->layers[15]);
  for (int i = 8; i < 15; ++i) bandable = bandable && p->layers[i].w_tc[0] && tc_layer_eligible(p->layers[i]);
  if (bandable) {
    p->keep_begin = keep_begin; p->keep_len = keep_len;
    unet_derive_bands(p->layers, keep_begin, keep_len);
    if (full_ksplit)
      for (int i = 8; i < 15; ++i) {
        ConvLayer full = p->layers[i];
        full.band_y0 = full.band_y1 = 0;
        p->layers[i].ksplit_tiles = tc_tile_count(full);
      }
    // The encoder skips the rows that repeat the padded tail where its first layer is the Cin = 1 kernel and the others run on
    // tensor cores (every stage-2 net of base 64).
    bool tail = tail_begin > 0 && conv_direct_cin1(p->layers[0]);
    for (int i = 1; i < 8; ++i) tail = tail && p->layers[i].w_tc[0] && tc_layer_eligible(p->layers[i]);
    if (tail) {
      p->tail_begin = tail_begin;
      unet_derive_tail(p->layers, tail_begin);
      for (int i = 0; i < 7; ++i) {
        int r0, r1;
        decoder_reads(p->layers, i, &r0, &r1);
        const ConvLayer& L = p->layers[i];
        RYK_CHECK(L.skip_y1 <= r0 || L.skip_y0 >= r1, "the decoder reads an encoder row that the padded-tail skip does not compute");
      }
    }
  }
  // Every buffer of the plan is carved from one zeroed allocation: plans are built and freed whenever a group's members change, and
  // separate small buffers would share the allocator's pages with other plans' and keep them in use after this plan is freed.
  std::vector<size_t> bytes;
  for (int l = 0; l < 8; ++l) bytes.push_back((size_t)B * lvlH(l) * lvlW(l) * level_channels(n->base, l) * esz);        // enc[l]
  for (int d = 0; d < 7; ++d) bytes.push_back((size_t)B * lvlH(6 - d) * lvlW(6 - d) * dec_out_channels(n->base, d) * esz);  // dec[d]
  bytes.push_back((size_t)B * H * W * n->in_ch * sizeof(float));                                                          // d_in
  bytes.push_back((size_t)B * H * W * n->out_ch * sizeof(float));                                                         // d_out
  constexpr size_t kAlign = 1024;
  size_t total = 0;
  for (size_t b : bytes) total += (b + kAlign - 1) / kAlign * kAlign;
  RYK_CUDA(cudaMalloc(&p->arena, total));
  RYK_CUDA(cudaMemsetAsync(p->arena, 0, total, e->stream));
  for (size_t i = 0, off = 0; i < bytes.size(); off += (bytes[i] + kAlign - 1) / kAlign * kAlign, ++i) {
    p->buffers.push_back((char*)p->arena + off);
    p->buffer_bytes.push_back(bytes[i]);
  }
  void* const* enc = p->buffers.data();
  void* const* dec = p->buffers.data() + 8;
  p->d_in = p->buffers[15];
  p->d_out = p->buffers[16];
  for (int i = 0; i < 16; ++i) {
    ConvLayer& L = p->layers[i];
    if (i == 0) {
      L.in0 = p->d_in; L.out = enc[0];
    } else if (i < 8) {
      L.in0 = enc[i - 1]; L.out = enc[i];
    } else if (i < 15) {
      int d = i - 8;
      if (d == 0) L.in0 = enc[7];
      else { L.in0 = dec[d - 1]; L.in1 = enc[7 - d]; }
      L.out = dec[d];
    } else {
      L.in0 = dec[6]; L.in1 = enc[0]; L.out = p->d_out;
    }
  }
  for (int i = 0; i < 16; ++i) {
    ConvLayer& L = p->layers[i];
    if (precision == 1 && L.w_tc[0] && tc_layer_eligible(L) && tc_layer_prepare(L, num_sms)) return -1;
  }
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  p->fused = s1_fused_eligible(n, p);
  n->plans[key] = p;
  *out = p;
  return 0;
}

int unet_plan_set_voices(UNetPlan* p, const std::vector<const UNet*>& nets, const std::vector<int>& voice_of) {
  const int V = (int)nets.size();
  RYK_CHECK(V >= 1 && V <= kMaxGroupVoices && (int)voice_of.size() == p->B && p->B <= kMaxGroupBatch, "a plan holds 1..8 voices over 1..64 batch items");
  for (const UNet* n : nets)
    RYK_CHECK(n->ndim == nets[0]->ndim && n->in_ch == nets[0]->in_ch && n->out_ch == nets[0]->out_ch && n->base == nets[0]->base,
              "the voices of one plan must have U-Nets of the same shape");
  for (int b = 0; b < p->B; ++b) RYK_CHECK(voice_of[b] >= 0 && voice_of[b] < V, "batch item of an unknown voice");
  // Only the tensor-core kernel and the stage-2 edge-layer kernels read weights per batch item: at other widths than base 64 some
  // layer runs on the generic CUDA-core kernel, so a plan of several voices is refused here, before any forward is captured.
  if (V > 1)
    for (const ConvLayer& L : p->layers)
      RYK_CHECK(L.tc_ready || conv_direct_per_item_weights(L),
                "a plan of several voices needs every layer on a kernel that reads weights per batch item (FP16 stage-2 nets of base 64)");
  for (int i = 0; i < 16; ++i) {
    ConvLayer& L = p->layers[i];
    L.n_voices = V;
    for (int v = 0; v < V; ++v) {
      const UNetLayerW& LW = nets[v]->layers[i];
      RYK_CHECK(LW.loaded, "U-Net layer weights not loaded");
      L.wt.w[v] = LW.d_w_direct; L.w_tc[v] = LW.d_w_tc; L.wt.scale[v] = LW.d_scale; L.wt.shift[v] = LW.d_shift;
      L.wt.host_scale[v] = LW.h_scale0; L.wt.host_shift[v] = LW.h_shift0;
    }
    for (int b = 0; b < p->B; ++b) L.wt.voice_of[b] = (uint8_t)voice_of[b];
    if (L.tc_ready && tc_layer_weight_maps(L)) return -1;
  }
  return 0;
}

// d_in / d_out live in the plan (p->d_in, p->d_out); callers fill / read them stream-ordered.
int unet_forward(Engine* e, UNetPlan* p, cudaStream_t st, int first_layer, int last_layer) {
  if (p->fused && e->s1_fused && first_layer == 0 && last_layer == 15) return s1_fused_run(e, p, st);
  for (int i = first_layer; i <= last_layer; ++i) {
    const ConvLayer& L = p->layers[i];
    int rc = L.tc_ready ? conv_tc_run(L, st) : conv_direct_run(L, st);
    if (rc) return rc;
  }
  return 0;
}

}  // namespace ryk
