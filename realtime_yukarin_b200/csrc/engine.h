// engine.h -- internal state of one libryk engine (one per process / GPU).
#pragma once
#include <string.h>
#include <algorithm>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <vector>

#include "common.cuh"
#include "unet.h"
#include "synth.h"

namespace ryk {

struct DioPlan;
struct HarvestPlan;
struct CrepePlan;
struct Session;
struct Group;
struct Reblock;
struct Drift;

// One target voice: the two U-Nets and the statistics that convert into one speaker.  Voice 0 is the engine's built-in voice (the
// ryk_model_* / ryk_stage1_set_stats / ryk_f0_set_stats calls and the per-op API); voices >= 1 come from ryk_voice_create.
struct Voice {
  UNet* stage1 = nullptr;
  UNet* stage2 = nullptr;
  // stage-1 statistics
  std::vector<float> s1_in_mean, s1_in_std, s1_out_mean, s1_out_std;
  float *d_s1_in_mean = nullptr, *d_s1_in_std = nullptr, *d_s1_out_mean = nullptr, *d_s1_out_std = nullptr;
  double f0_in_mean = 0, f0_in_std = 1, f0_tgt_mean = 0, f0_tgt_std = 1;
  bool has_f0_stats = false;
  int users = 0;                     // sessions and groups that convert into this voice
};

// The SPTK conversions of one (order, alpha, fft_size) as linear maps (features.cu: sptk_prepare)
struct SptkMats {
  double* d_G = nullptr;             // sp2mc: (order+1) x nb
  double* d_H = nullptr;             // mc2sp: nb x (order+1)
};

// The device and pinned host buffers of one session or re-blocker, freed with their owner.  Every buffer starts zeroed: device memory
// by a cudaMemsetAsync on `stream` (the engine stream: work queued there later, such as a session's template fill, runs after the
// zeros, and the owner synchronises it before other streams use the buffers), pinned memory by memset.  Allocating into a pointer
// that holds one of the owner's buffers replaces that buffer.
struct BufferSet {
  cudaStream_t stream = nullptr;
  BufferSet() = default;
  BufferSet(const BufferSet&) = delete;
  ~BufferSet() { for (void* p : dev_) cudaFree(p); for (void* p : host_) cudaFreeHost(p); }
  template <typename T> int device(T** p, size_t n) { return get((void**)p, sizeof(T) * n, false); }
  template <typename T> int pinned(T** p, size_t n) { return get((void**)p, sizeof(T) * n, true); }

 private:
  std::vector<void*> dev_, host_;
  int get(void** p, size_t bytes, bool host) {
    std::vector<void*>& owned = host ? host_ : dev_;
    const auto it = std::find(owned.begin(), owned.end(), *p);
    if (*p && it != owned.end()) { if (host) cudaFreeHost(*p); else cudaFree(*p); owned.erase(it); }
    *p = nullptr;
    if (!bytes) bytes = 16;
    if (host) RYK_CUDA(cudaMallocHost(p, bytes)); else RYK_CUDA(cudaMalloc(p, bytes));
    owned.push_back(*p);
    if (host) memset(*p, 0, bytes); else RYK_CUDA(cudaMemsetAsync(*p, 0, bytes, stream));
    return 0;
  }
};

struct Engine {
  int device = 0;
  cudaStream_t stream = nullptr;
  int precision = 1;                 // 0: FP32 CUDA-core convs everywhere, 1: FP16 wgmma tensor-core convs where eligible
  int f0_method = 0;                 // 0: DIO + StoneMask, 1: Harvest + StoneMask (world_harvest.cu), 2: CREPE (sessions only, crepe.cu)
  bool s1_fused = true;              // FP16 mode: stage 1 as ONE cluster kernel (s1_fused.cu) instead of 16 layer launches
  // FFT twiddles
  double2* d_twiddle = nullptr;
  // xorshift128 jump-ahead matrices (synthesis noise stream)
  uint32_t* d_jump = nullptr;
  // SPTK matrices keyed by (order, alpha, fft_size), alpha compared exactly.  Built on first use and freed only with the engine:
  // captured session graphs hold their addresses, so a per-op call or a session at another key must not replace them.
  std::map<std::tuple<int, double, int>, SptkMats> sptk;
  // DIO plans keyed by (n, fs, frame_period*1000, floor*1000, ceil*1000)
  std::map<std::tuple<int, int, int, int, int>, DioPlan*> dio_plans;
  // voices by id (voice 0 always exists; a destroyed voice leaves nullptr)
  std::vector<Voice*> voices;
  // synthesizers
  std::vector<Synth*> synths;
  std::vector<Session*> sessions;
  std::vector<Group*> groups;
  std::vector<Reblock*> reblocks;     // output re-blockers + silence gates (decode_worker.py:38-59)
  std::vector<Drift*> drifts;         // clock drift stages of played streams (drift.cu)
  float* d_colmin = nullptr;         // stage-2 prologue column-minimum partials
  // scratch arena for the per-op host-pointer API (grown on demand)
  void* d_scratch = nullptr; size_t scratch_bytes = 0;
  void* h_pinned = nullptr; size_t pinned_bytes = 0;
  // kernels run by session and group steps (ryk_engine_launch_count): the kernel nodes of the stage graphs they launch plus the
  // synthesizer's noise top-up; the device counter gets the kernels of the stage-1 SWITCH bodies the device selected
  long long launches = 0;
  unsigned long long* d_launches = nullptr;
  int plan_owners = 0;               // U-Net plan owner ids handed out to sessions and groups (0 is the engine's own plans)
  // optional device-side timing of the stage-2 tensor-core layers of session and group steps (bench roofline): event pairs per forward
  bool profile = false;
  cudaEvent_t timer_ev[2] = {nullptr, nullptr};
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> prof_events;
  // the last session or re-blocker snapshot / restore (ryk_snapshot_last_times): wall time waiting for its staged copies, and the rest
  double snap_device_ms = 0.0, snap_host_ms = 0.0;
};

// The sub-buffers of one engine buffer, each at the next 256-byte boundary in the order they are taken.  Over a null base it only adds
// up the size.
struct Arena {
  char* base;
  size_t off = 0;
  explicit Arena(void* b) : base((char*)b) {}
  template <typename T> T* take(size_t count) {
    off = (off + 255) & ~(size_t)255;
    T* p = base ? (T*)(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
};
// Lay out the device scratch (engine_scratch) or the pinned staging (engine_pinned_layout) of a call: `carve` runs over a null arena,
// which adds up the size, then over the buffer grown to that size.  It runs twice, so it may only take buffers.  Both buffers are the
// engine's, reused by the next call: a call is done with them when it returns.
int engine_scratch(Engine* e, const std::function<void(Arena&)>& carve);
int engine_pinned_layout(Engine* e, const std::function<void(Arena&)>& carve);
// the pinned staging as one block of `bytes`
int engine_pinned(Engine* e, size_t bytes, void** out);
inline Voice* engine_voice(Engine* e, int id) { return id >= 0 && id < (int)e->voices.size() ? e->voices[id] : nullptr; }
// identity stage-1 statistics of C channels unless statistics of C channels are loaded
int voice_default_stage1_stats(Voice* v, int C);
// both U-Nets created and every layer loaded
bool voice_models_loaded(const Voice* v);

// world_analysis.cu
int analysis_kernels_init();
int dio_plan_create(Engine* e, int n, int fs, double frame_period, double f0_floor, double f0_ceil, DioPlan** out, int f0_method = 0);
void dio_plan_free(DioPlan* p);
int dio_get_plan(Engine* e, int n, int fs, double frame_period, double f0_floor, double f0_ceil, DioPlan** out);
int dio_stonemask_run(Engine* e, DioPlan* p, const float* d_x, cudaStream_t st);
const double* dio_plan_f0(DioPlan* p);      // refined f0 (double) after dio_stonemask_run
double* dio_plan_f0_mut(DioPlan* p);
int dio_plan_frames(DioPlan* p);
HarvestPlan* dio_plan_harvest(DioPlan* p);
const double* dio_plan_f0_raw(DioPlan* p);     // f0 contour before StoneMask
// world_harvest.cu
int harvest_plan_create(Engine* e, int n, int fs, double frame_period, double f0_floor, double f0_ceil, HarvestPlan** out);
void harvest_plan_free(HarvestPlan* p);
int harvest_run(Engine* e, HarvestPlan* p, const float* d_x, double* d_f0, cudaStream_t st);
int harvest_plan_debug_copy(HarvestPlan* p, int* info, double* y, double* raw, double* cand, double* score, double* best, double* basic,
                            cudaStream_t st);
// crepe.cu: CREPE f0 front-end (acoustic_feature_wrapper.py:65-80)
int crepe_create(Engine* e, int capacity_multiplier);
void crepe_destroy();
int crepe_set_conv(Engine* e, int layer, const float* W, const float* bias, const float* gamma, const float* beta, const float* mean, const float* var);
int crepe_set_dense(Engine* e, const float* W, const float* bias);
int crepe_set_tables(Engine* e, const double* log_trans, const double* cents_mapping, double log_start, double log_emit_self, double log_emit_other);
int crepe_num_frames(int n16, double step_ms);
int crepe_predict(Engine* e, const float* audio16k, int n, double step_ms, double* f0, float* confidence, int* voicing, float* activation, int* path_out);
int crepe_set_resampler(Engine* e, int fs, int up, int down, const double* taps, int n_taps);
// why a CREPE plan at rate fs cannot be made (no complete model, no resampler taps for fs), or nullptr
const char* crepe_plan_refusal(int fs);
int crepe_plan_create(Engine* e, int n, int fs, double frame_period, CrepePlan** out);
void crepe_plan_free(CrepePlan* p);
int crepe_plan_run(Engine* e, CrepePlan* p, const float* d_x, cudaStream_t st);
const double* crepe_plan_f0(const CrepePlan* p);
int crepe_test_conv(Engine* e, int backend, int F, int Win, int Cin, int Cout, int k, const float* x, const float* W, const float* bias, float* y);
int crepe_test_network(Engine* e, int backend, const float* audio16k, int n, double step_ms, float* activation, int* path, int* voicing,
                       int repeat, float* ms_per_run);
// side (only while st is being captured into a graph): D4C becomes a branch of its own, concurrent with CheapTrick
// d_G: sp2mc matrix of (order, alpha, fft_size) from sptk_prepare
int spectral_analysis_run(Engine* e, const float* d_x, int n, int fs, double frame_period, const double* d_f0, int n_out,
                          int fft_size, int order, const double* d_G, float* d_sp, float* d_ap, float* d_mc, float* d_f0_out,
                          uint8_t* d_voiced, cudaStream_t st, cudaStream_t side = nullptr);

// world_synth.cu: offline Synthesis() (pyworld.synthesize) and the output silence gate
int world_synthesize_run(Engine* e, const double* f0, int n_frames, const float* sp, const float* ap, int fs, double frame_period_ms,
                         int fft_size, double* y, int y_length, long long* pulse_index, double* pulse_shift, int* pulse_vuv, int max_pulses);
int output_gate_async(Engine* e, const double* d_wave, const int* d_n_valid, int n, int n_fft, int hop, double threshold_db,
                      double* d_scratch, double* d_power, int* d_status, cudaStream_t st);
size_t output_gate_scratch_doubles(int n, int n_fft, int hop);

// sptk.cu
// the engine's G and H of (order, alpha, fft_size), built on the device on first use
int sptk_prepare(Engine* e, int order, double alpha, int fft_size, SptkMats* out);
// d_H: mc2sp matrix of (order, alpha, fft_size) from sptk_prepare
int mc2sp_run(Engine* e, const double* d_H, const float* d_mc, int T, int order, int fft_size, double add, float* d_sp_f32, double* d_sp_f64,
              cudaStream_t st);

// features.cu: polyphase resampler (wav I/O row)
int resample_poly_run(Engine* e, const float* d_x, int n, int up, int down, const double* d_h, int n_taps, float* d_y, int n_out, cudaStream_t st);

// gate.cu
int gate_mask_run(Engine* e, const float* d_wave, int n, int frame_length, int hop, double threshold_db, int n_frames,
                  double* d_mse_scratch, uint8_t* d_mask, int* d_index /*compacted frame ids*/, int* d_count, cudaStream_t st);

}  // namespace ryk

// The engine behind the public handle (include/ryk.h declares it opaque).
struct ryk_engine { ryk::Engine impl; };
