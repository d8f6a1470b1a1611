// convert.cu -- VoiceChanger.convert_from_acoustic_feature as one device-resident sequence
// (realtime_voice_conversion/yukarin_wrapper/voice_changer.py:24-42; SURVEY rows a8-a13):
//   silence gate -> gather effective frames -> stage-1 U-Net (+ f0 conversion) -> scatter into the
//   silent template -> mc2sp (+1e-16) -> stage-2 U-Net on the log spectrogram -> exp.
#include "engine.h"
#include "features.h"
#include "unet.h"

namespace ryk {

int convert_buffers_get(Engine* e, int T, int n_wave, int nb, int C, ConvertBuffers* cb) {
  size_t sizes[] = {sizeof(float) * (size_t)n_wave, sizeof(float) * T, sizeof(float) * (size_t)T * nb, sizeof(float) * (size_t)T * C, (size_t)T,
                    sizeof(double) * T, (size_t)T, sizeof(int) * T, sizeof(int) * 2,
                    sizeof(float) * (size_t)T * C, sizeof(float) * T, sizeof(float) * (size_t)T * nb, sizeof(float) * (size_t)T * nb,
                    sizeof(float) * (size_t)T * nb, (size_t)T};
  size_t total = 0;
  for (size_t s : sizes) total = ((total + 255) & ~(size_t)255) + s;
  void* base = nullptr;
  if (engine_scratch(e, total + 512, &base)) return -1;
  char* p = (char*)base; size_t off = 0; int i = 0;
  auto take = [&]() { off = (off + 255) & ~(size_t)255; void* r = p + off; off += sizes[i++]; return r; };
  cb->d_wave = (float*)take(); cb->d_f0 = (float*)take(); cb->d_ap = (float*)take(); cb->d_mc = (float*)take(); cb->d_voiced = (uint8_t*)take();
  cb->d_mse = (double*)take(); cb->d_mask = (uint8_t*)take(); cb->d_index = (int*)take(); cb->d_count = (int*)take();
  cb->d_mc_out = (float*)take(); cb->d_f0_out = (float*)take(); cb->d_ap_out = (float*)take(); cb->d_sp_mid = (float*)take();
  cb->d_sp_out = (float*)take(); cb->d_voiced_out = (uint8_t*)take();
  return 0;
}

int convert_window_device(Engine* e, const ConvertBuffers& cb, int T, int n_wave, int frame_length, int hop, double threshold_db,
                          int order, int fftlen, const double* d_H, cudaStream_t st) {
  const int nb = fftlen / 2 + 1, C = order + 1;
  const Voice* v = e->voices[0];                 // the per-op API converts into the built-in voice
  if (gate_mask_run(e, cb.d_wave, n_wave, frame_length, hop, threshold_db, T, cb.d_mse, cb.d_mask, cb.d_index, cb.d_count, st)) return -1;
  int cnt[2] = {0, 0};
  RYK_CUDA(cudaMemcpyAsync(cnt, cb.d_count, sizeof(cnt), cudaMemcpyDeviceToHost, st));
  RYK_CUDA(cudaStreamSynchronize(st));
  const float* d_y = nullptr;
  if (cnt[0] > 0) {   // voice_changer.py:32-35: stage 1 is skipped when no frame is effective
    UNetPlan* p1 = nullptr;
    if (unet_get_plan(e, v->stage1, 1, 1, cnt[1], e->precision, &p1)) return -1;
    if (stage1_prologue_run(v, cb.d_mc, cb.d_index, cb.d_count, C, (float*)p1->d_in, cnt[1], st)) return -1;
    if (unet_forward(e, p1, st)) return -1;
    d_y = (const float*)p1->d_out;
  }
  if (stage1_epilogue_run(v, d_y, cb.d_index, cb.d_mask, cb.d_count, T, C, cb.d_f0, cb.d_ap, cb.d_voiced, nb, kSilentMc0,
                          cb.d_mc_out, cb.d_f0_out, cb.d_ap_out, cb.d_voiced_out, nullptr, st)) return -1;
  if (mc2sp_run(e, d_H, cb.d_mc_out, T, order, fftlen, 1e-16, cb.d_sp_mid, nullptr, st)) return -1;
  const int Tp = T + (128 - T % 128);
  UNetPlan* p2 = nullptr;
  if (unet_get_plan(e, v->stage2, 1, Tp, 512, e->precision, &p2)) return -1;
  if (sr_prologue_run(e, cb.d_sp_mid, T, Tp, nb, (float*)p2->d_in, st)) return -1;
  if (unet_forward(e, p2, st)) return -1;
  if (sr_epilogue_run(e, (const float*)p2->d_out, T, nb, cb.d_sp_out, st)) return -1;
  return 0;
}

}  // namespace ryk
