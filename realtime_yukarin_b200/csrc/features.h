// features.h -- declarations for features.cu / convert.cu / session.cu
#pragma once
#include "common.cuh"

namespace ryk {

struct Engine;
struct Voice;

// The f0 map of one session, exp((ln f0 - mu_in) / sd_in * sd_tgt + mu_tgt), and its formant ratio, as one block of device memory
// that the stage-1 epilogue reads at run time (DESIGN.md §4a).  The host stages a new block between steps; in follow mode k_f0_measure
// rewrites mu_in / sd_in (never formant).
struct F0Map {
  double mu_in, sd_in, mu_tgt, sd_tgt;
  double sd_floor;                  // follow mode: lower bound of the measured sd_in
  int has_stats;                    // 0: identity map (a voice without f0 statistics and no map set on the session)
  int follow, min_voiced;           // follow mode: input side = the measured statistics once min_voiced voiced frames are counted
  int pad_;
  double formant;                   // formant ratio of the stage-2 envelope (session_build sets 1; voice_f0_map leaves 0, never read)
};
// running statistics of ln f0 over the voiced frames of a session's input: count, mean, sum of squared deviations
struct F0Stats { long long n; double mean, m2; };

// normalisation with the stage-1 statistics of voice v
int stage1_prologue_run(const Voice* v, const float* d_mc, const int* d_index, const int* d_count, int C, float* d_x, int Tp_capacity, cudaStream_t st);
// de-normalisation with the statistics of voice v, and f0 conversion with the map in *d_map (nullptr: the f0 statistics of voice v);
// with a map, d_formant_out (non-null) receives d_map->formant, the ratio the stage-2 epilogue of the same step applies
int stage1_epilogue_run(const Voice* v, const float* d_y, const int* d_index, const uint8_t* d_mask, const int* d_count, int T, int C,
                        const float* d_f0_in, const float* d_ap_in, const uint8_t* d_voiced_in, int nb, float silent_mc0,
                        float* d_mc_out, float* d_f0_out, float* d_ap_out, uint8_t* d_voiced_out, const F0Map* d_map, cudaStream_t st,
                        double* d_formant_out = nullptr);
F0Map voice_f0_map(const Voice* v);
// merge the n frames of one chunk into *d_stats; in follow mode (d_map->follow) also write the measured input side into *d_map
int f0_measure_run(const float* d_f0, const uint8_t* d_voiced, int n, F0Stats* d_stats, F0Map* d_map, cudaStream_t st);
constexpr int kColminFloats = 64 * 512;      // column-minimum partials of the stage-2 prologue (one scratch per concurrent stream)
int sr_prologue_run(Engine* e, const float* d_sp, int T, int Tp, int nb, float* d_x, cudaStream_t st, float* d_colmin = nullptr);
// frames [t0, t1) of the T-frame window (t1 < 0: T); the other rows of d_sp_out are not written.  The envelope is warped by the
// formant ratio *d_formant (non-null: read at run time) or else `formant` (DESIGN.md DECIDE F1); ratio 1 is the plain epilogue, bitwise.
int sr_epilogue_run(Engine* e, const float* d_y, int T, int nb, float* d_sp_out, cudaStream_t st, int t0 = 0, int t1 = -1,
                    double formant = 1.0, const double* d_formant = nullptr);

constexpr float kSilentMc0 = -18.420680743952367f;   // ln(1e-8): silent template mel-cepstrum c0 (DESIGN.md, DECIDE)

// device buffers of one VoiceChanger.convert_from_acoustic_feature evaluation (window of T frames)
struct ConvertBuffers {
  float *d_wave, *d_f0, *d_ap, *d_mc; uint8_t* d_voiced;                 // inputs
  double* d_mse; uint8_t* d_mask; int* d_index; int* d_count;           // gate
  float *d_mc_out, *d_f0_out, *d_ap_out, *d_sp_mid, *d_sp_out; uint8_t* d_voiced_out;
};
int convert_buffers_get(Engine* e, int T, int n_wave, int nb, int C, ConvertBuffers* out);
// stream-ordered except for one 8-byte D2H of the effective-frame count (picks the stage-1 plan); d_H: mc2sp matrix of the key
int convert_window_device(Engine* e, const ConvertBuffers& cb, int T, int n_wave, int frame_length, int hop, double threshold_db,
                          int order, int fftlen, const double* d_H, cudaStream_t st);

// polyphase resampler (features.cu: k_resample_poly): the whole-signal call of ryk_resample_poly and the two streaming sides of a
// session's device-rate conversion.  Streaming positions live on the device, double-buffered by step parity.
struct ResampleState { long long in_end, out_end; };     // input samples received, output samples emitted (before the step)
enum PolyMode { kPolyWhole = 0, kPolyStreamIn = 1, kPolyStreamOut = 2 };
template <typename Tin, typename Tout>
struct PolyArgs {
  int mode;
  const double* h; int n_taps, up, down;
  const Tin* x; int x_len;                 // whole signal | history window ending at the newest sample | kept history
  const Tin* x_new; const int* n_new;      // stream out: the step's new samples and their count
  int chunk, delay;                        // stream in: samples per step, leading zeros of the output (model-rate samples)
  Tout* y; int n_out;                      // outputs (stream out: the most one step may emit)
  int* n_out_dev;                          // stream out: outputs emitted by the step
  const ResampleState* st; ResampleState* st_next;
  Tin* hist_next;                          // stream out: the kept history after the step (x_len samples)
};
int resample_stream_in_run(Engine* e, const float* d_window, int window, int chunk, int delay, int up, int down, const double* d_h, int n_taps,
                           const ResampleState* d_st, ResampleState* d_st_next, float* d_y, int n_out, cudaStream_t st);
int resample_stream_out_run(Engine* e, const double* d_hist, double* d_hist_next, int hist, const double* d_new, const int* d_n_new, int up,
                            int down, const double* d_h, int n_taps, const ResampleState* d_st, ResampleState* d_st_next, double* d_y,
                            int max_out, int* d_n_out, cudaStream_t st);

void session_destroy_all(Engine* e);
// what the re-blocker (reblock.cu) reads of session `id`: the samples and sample count of its last step in device memory, the most
// samples a step returns, and the decode stream that orders work on them
int session_last_output(Engine* e, int id, const double** out, const int** n_out, int* max_out, cudaStream_t* sD);
void reblock_destroy_all(Engine* e);
int session_streams_fork(Engine* e, cudaEvent_t ev);
int session_streams_join(Engine* e);

}  // namespace ryk
