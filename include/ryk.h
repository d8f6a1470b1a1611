/*
 * ryk.h -- C ABI of libryk.so: the H100-native per-chunk hot path of realtime-yukarin
 *          (encode -> stage 1 -> stage 2 -> vocode).  Plain pointers and sizes only.
 *
 * Every entry point replaces one call the reference makes into an un-vendored third-party library
 * (file:line are paths under the reference checkout, realtime_voice_conversion/ abbreviated rvc/):
 *
 *   ryk_world_analyze          <- yukarin.AcousticFeature.extract (pyworld dio/stonemask/cheaptrick/d4c + pysptk.sp2mc)
 *                                 rvc/yukarin_wrapper/vocoder.py:26-48, rvc/yukarin_wrapper/acoustic_feature_wrapper.py:28-33
 *   ryk_world_f0               <- yukarin.AcousticFeature.extract_f0 (override hook at acoustic_feature_wrapper.py:66-80)
 *   ryk_silence_mask           <- AcousticConverter.separate_effective (librosa _signal_to_frame_nonsilent)  rvc/yukarin_wrapper/voice_changer.py:27-31
 *   ryk_stage1_load/_convert   <- yukarin.AcousticConverter(...)/.convert (Chainer forward)                   voice_changer.py:33, converter/yukarin_converter.py:40-46
 *   ryk_mc2sp                  <- AcousticConverter.decode_spectrogram (pysptk.mc2sp)                           voice_changer.py:38
 *   ryk_stage2_load/_convert   <- become_yukarin.SuperResolution(...)/.convert (Chainer forward)               voice_changer.py:41, converter/yukarin_converter.py:50-55
 *   ryk_convert_window         <- VoiceChanger.convert_from_acoustic_feature, fused on device                   voice_changer.py:24-42
 *   ryk_synth_create           <- world4py apidefinitions._InitializeSynthesizer                                rvc/yukarin_wrapper/vocoder.py:79-87
 *   ryk_synth_add_parameters   <- world4py apidefinitions._AddParameters                                        vocoder.py:99
 *   ryk_synth_synthesis2       <- world4py apidefinitions._Synthesis2 (+ the per-sample buffer read-out)        vocoder.py:102-104
 *   ryk_synth_decode           <- RealtimeVocoder.decode as one call (add + drain)                              vocoder.py:89-120
 *   ryk_session_*              <- the encode/convert/decode StreamWrapper chain of one audio stream kept on
 *                                 device                                                                       rvc/worker/, rvc/stream/ (all modules)
 *   ryk_world_synthesize       <- pyworld.synthesize (Vocoder.decode, offline)                                  rvc/yukarin_wrapper/vocoder.py:50-62
 *   ryk_output_gate, ryk_reblock_* <- decode worker: wave_fragment re-blocking + librosa stft/power_to_db gate   rvc/worker/decode_worker.py:38-59
 *   ryk_resample_poly          <- librosa.load(path, sr=input_rate) resampling                                  check.py:80
 *
 * Conventions: all functions return 0 on success and a negative value on error unless stated otherwise
 * (ryk_last_error() describes the failure); "host" pointers are ordinary process memory, "dev"
 * pointers are CUDA device memory of the engine's GPU.  One engine per process per GPU; an engine is
 * NOT thread-safe (the reference drives each stage from a single thread as well).
 */
#ifndef RYK_H_
#define RYK_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ryk_engine ryk_engine;

int ryk_abi_version(void);
const char* ryk_last_error(void);

/* ---- engine ---------------------------------------------------------------------------- */
int ryk_engine_create(int device, ryk_engine** out);
int ryk_engine_destroy(ryk_engine* e);
/* 0: FP32 CUDA-core convolutions everywhere (bisecting / numerics reference)
 * 1: FP16 operands + FP32 accumulate on the tensor cores (wgmma) for the stage-2 k4 layers (default) */
int ryk_engine_set_precision(ryk_engine* e, int mode);
int ryk_engine_get_precision(ryk_engine* e);
/* FP16 mode: run the stage-1 1-D U-Net (AcousticConverter.convert_from_feature, voice_changer.py:36) as ONE thread-block-cluster
 * kernel (default, s1_fused.cu) or as 16 layer launches (enable = 0).  Returns the cluster size in use, <= 0 when the kernel is
 * unavailable.  Sessions capture their stage-1 graphs at creation, so switch before ryk_session_create. */
int ryk_engine_set_stage1_fused(ryk_engine* e, int enable);
/* Kernels run by the steps of this engine's sessions and groups so far: the kernel nodes of every stage graph a step launches
 * (cuFFT's included), the kernels of the stage-1 body the device selected, and the synthesizer's noise top-up.  The per-op calls
 * below and re-blocker pushes are not counted.  Synchronises the device; -1 on a CUDA error. */
long long ryk_engine_launch_count(ryk_engine* e);
int ryk_engine_synchronize(ryk_engine* e);
/* CUDA-event timing of the stage-2 k4-layer block (layers 1..14, the wgmma kernel) on the engine's stream */
int ryk_engine_timer_start(ryk_engine* e);                    /* cudaEventRecord on the engine's stream */
int ryk_engine_timer_stop(ryk_engine* e, float* elapsed_ms);  /* record + synchronize + elapsed */
/* Time the stage-2 forwards of session and group steps (only those; per-op calls are never timed) */
int ryk_engine_profile(ryk_engine* e, int enable);
/* Device time (ms) of the stage-2 k4-layer block over all session and group forwards since the last read: the sum of the per-forward
 * durations and the UNION of the per-forward intervals (a session alternates its stage-2 forwards between two streams, so they overlap) */
int ryk_engine_profile_read2(ryk_engine* e, double* stage2_ms_total, double* stage2_ms_union, int* stage2_runs);

/* ---- WORLD analysis (encode) -------------------------------------------------------------- */
/* wave_host: n float32 samples.  Outputs are n_frames = n / hop rows (hop = fs * frame_period / 1000):
 * f0 [n_frames], sp/ap [n_frames][fft_length/2+1], mc [n_frames][order+1], voiced [n_frames] (0/1).
 * f0_override (nullable, double[n_frames_world = n/hop + 1]) replaces DIO+StoneMask. Any output may be NULL. */
int ryk_world_analyze(ryk_engine* e, const float* wave_host, int n, int fs, double frame_period_ms,
                      double f0_floor, double f0_ceil, int fft_length, int order, double alpha,
                      const double* f0_override, float* f0, float* sp, float* ap, float* mc, uint8_t* voiced);
/* DIO + StoneMask only; f0/t are double[n / hop + 1] (WORLD's own frame count). */
int ryk_world_f0(ryk_engine* e, const float* wave_host, int n, int fs, double frame_period_ms,
                 double f0_floor, double f0_ceil, double* f0, double* t);
int ryk_world_num_frames(int n, int fs, double frame_period_ms);
/* f0 extractor behind ryk_world_f0 / ryk_world_analyze and sessions created afterwards -- the f0 hook of yukarin's
 * AcousticFeature.extract (acoustic_feature_wrapper.py:28-33; f0_estimating_method, SURVEY A.2 / A.7):
 *   0 = pyworld.dio + pyworld.stonemask (default), 1 = pyworld.harvest + pyworld.stonemask,
 *   2 = CREPE (crepe.predict + predict_voicing, no StoneMask) for sessions created afterwards.  Method 2 needs a complete CREPE model,
 *       its decoder tables and the resampler taps for the session's fs (see below); each step's encode window is analysed on its own.
 *       ryk_world_f0, and ryk_world_analyze without f0_override, fail in method 2: for a single signal use ryk_crepe_predict and pass
 *       its f0 as f0_override (CrepeAcousticFeatureWrapper does). */
int ryk_engine_set_f0_method(ryk_engine* e, int method);
int ryk_engine_get_f0_method(ryk_engine* e);

/* ---- CREPE f0 front-end (CrepeAcousticFeatureWrapper.extract_f0, acoustic_feature_wrapper.py:65-80) --------------------------
 * crepe.predict(x, fs, viterbi=True, model_capacity=..., step_size=frame_period) + crepe.predict_voicing on the device.  The caller
 * resamples to 16 kHz (ryk_resample_poly) and applies the reference's rule voiced = (voicing == 1) | (confidence > 0.1).
 * capacity_multiplier: 4 tiny, 8 small, 16 medium, 24 large, 32 full.  Conv weights W (cout, cin, k) for blocks 0..5 with widths
 * 512, 64 x 5 and filters m * {32, 4, 4, 4, 8, 16}; BatchNorm statistics per block (eps 1e-3); dense W (360, 64 m).
 * log_trans: the 360 x 360 log transition matrix of the pitch HMM, its start / emission log-probabilities and the bin -> cents table, computed by the host
 * mirror exactly as crepe.to_viterbi_cents does (shared tables make the Viterbi sums bit-identical to the CPU restatement). */
int ryk_crepe_create(ryk_engine* e, int capacity_multiplier);
int ryk_crepe_set_conv(ryk_engine* e, int block, const float* W, const float* bias, const float* bn_gamma, const float* bn_beta,
                       const float* bn_mean, const float* bn_var);
int ryk_crepe_set_dense(ryk_engine* e, const float* W, const float* bias);
int ryk_crepe_set_decoder_tables(ryk_engine* e, const double* log_trans, const double* cents_mapping /* [360] */, double log_start,
                                 double log_emit_self, double log_emit_other);
/* Polyphase filter fs -> 16 kHz for the sessions' CREPE analysis (f0 method 2): up / down = 16000 / fs reduced, taps as for
 * ryk_resample_poly (realtime_yukarin_b200/wave_io.py: resample_filter(up, down)).  One filter per fs; a new upload replaces it.
 * ryk_crepe_create / _set_* fail while a session in f0 method 2 exists: its captured graphs point at the model. */
int ryk_crepe_set_resampler(ryk_engine* e, int fs, int up, int down, const double* taps, int n_taps);
int ryk_crepe_num_frames(int n16, double step_ms);
/* f0 / confidence / voicing (HMM state) [frames], activation [frames][360], path [frames] (pitch-bin Viterbi path); any may be NULL */
int ryk_crepe_predict(ryk_engine* e, const float* audio16k, int n, double step_ms, double* f0, float* confidence, int* voicing,
                      float* activation, int* path);

/* ---- silence gate --------------------------------------------------------------------------- */
/* mask[n_frames] (0/1): a frame is effective when it lies within threshold_db of the loudest frame of the window
 * (dB - max dB > -threshold_db).  The same rule holds wherever a threshold_db is passed (ryk_convert_window, ryk_session_config):
 *   threshold_db > 0   the gate of the reference (60 by default);
 *   threshold_db == 0  every frame is gated, the loudest included: stage 1 is skipped and the window is the silent template;
 *   threshold_db < 0   no gate, whatever the value: every frame is effective. */
int ryk_silence_mask(ryk_engine* e, const float* wave_host, int n, int frame_length, int hop,
                     double threshold_db, int n_frames, uint8_t* mask);

/* ---- networks ------------------------------------------------------------------------------- */
/* stage: 1 (1-D, yukarin) or 2 (2-D, become-yukarin).  Layers 0..7 = encoder c0..c7, 8..15 = decoder c0..c7.
 * W is the model file's (Chainer) layout: conv (Cout, Cin, k[, k]), transposed conv (Cin, Cout, k[, k]);
 * scale/shift [Cout] are the bias and eval-mode BatchNorm folded together (y = conv(x) * scale + shift). */
int ryk_model_create(ryk_engine* e, int stage, int in_channels, int out_channels, int base_channels);
int ryk_model_set_layer(ryk_engine* e, int stage, int layer, const float* W, const float* scale, const float* shift);
int ryk_model_layer_shape(ryk_engine* e, int stage, int layer, int* transposed, int* cin, int* cout, int* k);
/* per-channel normalisation of the stage-1 input/output features and the log-f0 statistics */
int ryk_stage1_set_stats(ryk_engine* e, int channels, const float* in_mean, const float* in_std,
                         const float* out_mean, const float* out_std);
int ryk_f0_set_stats(ryk_engine* e, double in_mean, double in_std, double target_mean, double target_std);
/* Voices: an engine holds several target voices, each its own pair of models with their statistics.  Voice 0 is the engine's built-in
 * voice, the one the calls above and the per-op conversions address.  ryk_voice_create returns ids >= 1; the ryk_voice_* calls take
 * the same arguments as the calls above plus the voice.  A voice >= 1 is fixed while a session or group uses it: changing its models
 * or statistics, or destroying it (which frees its weights), fails until those are destroyed. */
int ryk_voice_create(ryk_engine* e, int* voice_id);
int ryk_voice_destroy(ryk_engine* e, int voice_id);
int ryk_voice_model_create(ryk_engine* e, int voice_id, int stage, int in_channels, int out_channels, int base_channels);
int ryk_voice_model_set_layer(ryk_engine* e, int voice_id, int stage, int layer, const float* W, const float* scale, const float* shift);
int ryk_voice_stage1_set_stats(ryk_engine* e, int voice_id, int channels, const float* in_mean, const float* in_std,
                               const float* out_mean, const float* out_std);
int ryk_voice_f0_set_stats(ryk_engine* e, int voice_id, double in_mean, double in_std, double target_mean, double target_std);
/* x, y: [T][channels] float32 (T >= 1; internally padded to the next multiple of 128 with the per-channel minimum) */
int ryk_stage1_convert(ryk_engine* e, const float* x, int T, float* y);
/* f0_out[i] = voiced[i] ? exp((ln f0[i] - mu_in) / sd_in * sd_tgt + mu_tgt) : 0 */
int ryk_f0_convert(ryk_engine* e, const float* f0, const uint8_t* voiced, int T, float* f0_out);
/* mc [T][order+1] float32 -> sp [T][fftlen/2+1] float64 = exp(H mc) (pysptk.mc2sp) */
int ryk_mc2sp(ryk_engine* e, const float* mc, int T, int order, double alpha, int fftlen, double* sp);
/* sp, out: [T][513] float32 */
int ryk_stage2_convert(ryk_engine* e, const float* sp, int T, float* out);
/* ryk_stage2_convert with the envelope warped by a formant ratio in [0.5, 2] (see ryk_session_set_formant); ratio 1 is bitwise
 * ryk_stage2_convert.  Refused: a non-finite ratio or one outside [0.5, 2]. */
int ryk_stage2_convert_formant(ryk_engine* e, const float* sp, int T, double ratio, float* out);

/* The whole VoiceChanger.convert_from_acoustic_feature on device: one upload, one download.
 * in : wave [n_wave], f0 [T], ap [T][nb], mc [T][order+1], voiced [T]
 * out: f0 [T], ap [T][nb], sp [T][nb], voiced [T], mc [T][order+1] (nullable)      nb = fftlen/2+1 */
int ryk_convert_window(ryk_engine* e, const float* wave, int n_wave, int fs, int frame_length, int hop, double threshold_db,
                       const float* f0, const float* ap, const float* mc, const uint8_t* voiced, int T,
                       int order, double alpha, int fftlen,
                       float* f0_out, float* ap_out, float* sp_out, uint8_t* voiced_out, float* mc_out);

/* ---- WORLD realtime synthesizer (vocode) ------------------------------------------------------ */
int ryk_synth_create(ryk_engine* e, int fs, double frame_period_ms, int fft_size, int buffer_size,
                     int number_of_pointers, int* synth_id);
int ryk_synth_destroy(ryk_engine* e, int synth_id);
/* returns 1 when the frames were queued, 0 when the ring is full (world4py semantics), < 0 on error */
int ryk_synth_add_parameters(ryk_engine* e, int synth_id, const double* f0, int n, const float* sp, const float* ap);
/* returns 1 and writes buffer_size doubles when a block was produced, 0 when not enough pulses are queued */
int ryk_synth_synthesis2(ryk_engine* e, int synth_id, double* buffer);
/* add + drain in one call: out receives *n_blocks * buffer_size doubles (at most max_blocks blocks) */
int ryk_synth_decode(ryk_engine* e, int synth_id, const double* f0, int n, const float* sp, const float* ap,
                     double* out, int max_blocks, int* n_blocks);

/* ---- offline synthesis: Vocoder.decode = pyworld.synthesize (SURVEY 8(f) rank 3) ---------------------
 * Replaces realtime_voice_conversion/yukarin_wrapper/vocoder.py:50-62 (pyworld.synthesize -> WORLD Synthesis()):
 * whole-utterance time base, fractional pulse shift, Hanning dc-remover, overlap-add.  y receives
 * ryk_world_synthesize_length(n_frames, frame_period_ms, fs) = (int)(n_frames * frame_period_ms * fs / 1000) doubles.
 * pulse_index / pulse_shift / pulse_vuv (each may be NULL, max_pulses entries) expose the pulse plan for parity tests. */
int ryk_world_synthesize_length(int n_frames, double frame_period_ms, int fs);
int ryk_world_synthesize(ryk_engine* e, const double* f0, int n_frames, const float* sp, const float* ap, int fs,
                         double frame_period_ms, int fft_size, double* y, int y_capacity, int* y_length,
                         long long* pulse_index, double* pulse_shift, int* pulse_vuv, int max_pulses, int* n_pulses);

/* ---- output silence gate and re-blocking (SURVEY 8(f) rank 2) ------------------------------------------
 * Replaces realtime_voice_conversion/worker/decode_worker.py:38-59: the synthesizer's 1024-sample blocks are queued in a
 * fragment, one out_audio_chunk is cut off its front per step when enough samples are queued, and the chunk is dropped
 * when librosa.power_to_db(abs(librosa.stft(chunk)) ** 2).mean() < -output_silent_threshold
 * (n_fft 2048, hop 512, periodic Hann, reflect-centred, amin 1e-10, top_db 80).
 * ryk_output_gate: the gate alone on a host chunk; *pass = 1 keeps the chunk.
 * ryk_reblock_*: device-resident fragment + gate.  push_device is stream-ordered and never syncs the host: with
 * session_id >= 0 it is queued on that session's decode stream right behind its latest step (wave_dev == NULL consumes the
 * step's blocks and count in place); results go to ring slot ticket % 8.  collect: *status 0 = no chunk this step,
 * 1 = chunk copied to chunk_out, 2 = chunk was silent (the reference forwards None). */
int ryk_output_gate(ryk_engine* e, const double* wave, int n, int n_fft, int hop, double threshold_db, double* power_db, int* pass);
int ryk_reblock_create(ryk_engine* e, int out_audio_chunk, int max_in, int n_fft, int hop, double threshold_db, int* reblock_id);
int ryk_reblock_destroy(ryk_engine* e, int reblock_id);
int ryk_reblock_push(ryk_engine* e, int reblock_id, const double* wave, int n, double* chunk_out, int* status, double* power_db);
int ryk_reblock_push_device(ryk_engine* e, int reblock_id, int session_id, const double* wave_dev, const int* n_dev, long long* ticket);
int ryk_reblock_collect(ryk_engine* e, int reblock_id, long long ticket, double* chunk_out, int* status, double* power_db);
/* Non-blocking: *done = 1 when ryk_reblock_collect(ticket) would not wait (queue_output_wave.get_nowait, run.py:176-182).
 * collect fails (instead of dropping samples) when a step produced more than the fragment can hold: the reference's
 * wave_fragment is unbounded (decode_worker.py:47-52), the device fragment holds 2 * (out_audio_chunk + max_in) samples. */
int ryk_reblock_poll(ryk_engine* e, int reblock_id, long long ticket, int* done);
int ryk_reblock_result_device(ryk_engine* e, int reblock_id, long long ticket, const double** chunk_dev, const int** status_dev,
                              const double** power_dev);

/* ---- sample-rate conversion for wav input (SURVEY 8(f) rank 3; check.py:80 librosa.load(path, sr=input_rate)) --------
 * Polyphase FIR resampling, the upfirdn step of scipy.signal.resample_poly: up / down must be coprime, `taps` is the
 * odd-length low-pass filter already scaled by `up` (realtime_yukarin_b200/wave_io.py: resample_filter), edges are
 * zero-padded; y receives ryk_resample_length(n, up, down) = ceil(n * up / down) samples. */
int ryk_resample_length(int n, int up, int down);
int ryk_resample_poly(ryk_engine* e, const float* x, int n, int up, int down, const double* taps, int n_taps, float* y,
                      int y_capacity, int* n_out);

/* ---- device-resident streaming session (one audio stream) -------------------------------------- */
typedef struct {
  int fs;                       /* 24000 */
  double frame_period_ms;       /* 5 */
  double f0_floor, f0_ceil;     /* 71, 800 */
  int fft_length, order;        /* 1024, 8 */
  double alpha;                 /* 0.466 */
  double buffer_time;           /* seconds of audio per pushed chunk (0.3) */
  double encode_extra_time, convert_extra_time, decode_extra_time;   /* 0, 0.5, 0 */
  double threshold_db;          /* silence gate (see ryk_silence_mask): 0 gates every frame, < 0 disables the gate */
  int vocoder_buffer_size;      /* 1024 */
} ryk_session_config;

int ryk_session_create(ryk_engine* e, const ryk_session_config* cfg, int* session_id);
/* A session that converts into voice_id until ryk_session_set_voice switches it (ryk_session_create: voice 0).  A voice >= 1 needs
 * both models with every layer loaded; without stage-1 statistics it uses identity statistics. */
int ryk_session_create_voice(ryk_engine* e, const ryk_session_config* cfg, int voice_id, int* session_id);
int ryk_session_voice(ryk_engine* e, int session_id);        /* the voice a session converts into, or -1 */
/* Converts the session into voice_id from its next submitted step on.  Windows, synthesizer, resamplers, step count, speaker
 * statistics, follow mode, formant ratio, attached re-blockers and group membership carry over.  A hard cut at the step boundary (no
 * crossfade): every later step converts its whole window with the new voice, so only the synthesizer's history differs from a session
 * created on that voice.
 * f0 map: both sides become the new voice's f0 statistics (identity without them), as a session created on it starts; a caller's own
 *   input side or pitch offset is set again with ryk_session_set_f0_map after the switch (it lands on the same next step).
 * Needs every host-API chunk of the session collected, and of its group for a member (device-resident steps count as collected).  The
 * call waits for the device, builds the new voice's stage-1 graphs and stage-2 plans (a member: the group's new batched plan, its slot
 * unchanged) and launches no kernel; the steps after it allocate nothing, and only the first two capture graphs, as on a new session.
 * The old voice is unlocked, the new one locked.  Switching to the current voice does nothing and does not wait.
 * Refused, changing nothing: an unknown session or voice, a voice without both models fully loaded or whose stage-1 channels differ from
 * order + 1, an uncollected chunk, a group rule the member's new voice would break, follow mode on with a voice without f0 statistics,
 * an engine precision or stage-1 mode changed since the session was created. */
int ryk_session_set_voice(ryk_engine* e, int session_id, int voice_id);
int ryk_session_destroy(ryk_engine* e, int session_id);
/* One chunk through encode -> convert -> decode with host buffers (H2D + kernels + D2H inside).
 * wave: round(fs * buffer_time) float32 samples; out: up to out_capacity float64 samples; *n_out is a
 * multiple of vocoder_buffer_size (the remainder stays in the synthesizer, as in the reference). */
int ryk_session_push(ryk_engine* e, int session_id, const float* wave, int n, double* out, int out_capacity, int* n_out);
/* Pipelined host API: submit queues a chunk and returns at once (ticket = chunk number), collect waits for that
 * chunk's output.  Up to 5 chunks may be in flight; encode / convert / decode of consecutive chunks then overlap on
 * three CUDA streams, exactly like the reference's three worker processes (run.py:58-93).  push == submit + collect. */
int ryk_session_submit(ryk_engine* e, int session_id, const float* wave, int n, long long* ticket);
int ryk_session_collect(ryk_engine* e, int session_id, long long ticket, double* out, int out_capacity, int* n_out);
/* Non-blocking: *done = 1 when ryk_session_collect(ticket) would not wait (ticket among the last 8 steps). */
int ryk_session_poll(ryk_engine* e, int session_id, long long ticket, int* done);
/* Same chunk step with the input already resident in HBM and the output left there (throughput measurement);
 * asynchronous: returns when the work is queued, results are valid after ryk_engine_synchronize. */
int ryk_session_push_device(ryk_engine* e, int session_id, const float* wave_dev, int n, double* out_dev, int out_capacity,
                            int* n_out_dev);

/* Device rates.  A session analyses, converts and synthesises at cfg.fs; it may also take its chunks at a sound card's input rate and
 * return its samples at the card's output rate, resampling on the GPU inside its captured stages (no host synchronisation).
 * `taps` is the odd-length low-pass filter of ryk_resample_poly (realtime_yukarin_b200/wave_io.py: resample_filter(up, down)), up / down
 * the coprime ratio of the resampler's output rate to its input rate: fs / rate on the input side, rate / fs on the output side.
 * rate == fs leaves that side without a resampler.  Valid only on a fresh session (no chunk pushed, not in a group); each side once.
 * Input:  a chunk is n_in = round(rate * buffer_time) samples, and n_in * up must equal round(fs * buffer_time) * down.  Step k
 *         analyses samples [k n, (k + 1) n) of zeros(delay_in) followed by resample_poly(all chunks so far), n = round(fs * buffer_time).
 * Output: after step k the session has returned resample_poly(y)[:M_k], y = the synthesizer's samples of steps 0..k (N_k of them) and
 *         M_k = the outputs whose filter support lies inside [0, N_k); a step returns M_k - M_{k-1} samples, at most max_out.
 * ryk_session_io_geometry: n_in = samples per pushed chunk, max_out = the most samples one step returns (out_capacity of
 * ryk_session_push_device, max_in of an attached re-blocker), delay_in = the input delay in model-rate samples, in_rate / out_rate =
 * the device rates (fs when unset).  Any output pointer may be NULL.  Groups need members with the same device rates. */
int ryk_session_set_input_rate(ryk_engine* e, int session_id, int rate, int up, int down, const double* taps, int n_taps);
int ryk_session_set_output_rate(ryk_engine* e, int session_id, int rate, int up, int down, const double* taps, int n_taps);
int ryk_session_io_geometry(ryk_engine* e, int session_id, int* n_in, int* max_out, int* delay_in, int* in_rate, int* out_rate);

/* The f0 map of a session and the log-f0 statistics of its speaker.  A session converts f0 by
 * exp((ln f0 - in_mean) / in_std * target_std + target_mean) (yukarin's F0Converter).  The map starts as the f0 statistics of the
 * session's voice and belongs to the session from then on: setting it never touches the voice or another session, so several callers
 * converting into one voice can each have the input statistics of their own speaker, and target_mean + s * ln(2) / 12 shifts the pitch
 * by s semitones (the spectral envelope is not moved: see ryk_session_set_formant).
 * ryk_session_get_f0_map: the values the NEXT submitted step will use (in follow mode: the fallback input side).
 * ryk_session_set_f0_map: takes effect at the next submitted step and for every later one; steps already submitted keep the map they
 *   were submitted with.  Allowed with chunks in flight and for a group member; it does not wait for the device and launches nothing.
 *   On a session whose voice has no f0 statistics (identity map) it turns the map on for this session only.
 * ryk_session_f0_measure: fresh session only (no chunk pushed).  Each step then adds the voiced frames of its chunk -- every 5 ms
 *   frame of the input exactly once, whatever the silence gate decides about it -- to a running count, mean and variance of ln f0
 *   kept on the device in FP64 (one more kernel per step).  The result depends on the input stream alone: it is bit-identical from
 *   run to run and does not depend on what else the engine runs.
 * ryk_session_f0_follow: needs measuring and a map.  With follow = 1, from the next submitted step on, every step whose running count
 *   (its own chunk included) has reached min_voiced_frames (>= 1) converts with in_mean = the measured mean and in_std =
 *   max(measured std, sd_floor); before that it uses the input side last set from the host.  sd_floor (finite, > 0; 0.05, about 0.9
 *   semitones, is a reasonable value) keeps a monotone speaker from dividing by zero.  The estimate is cumulative (no forgetting).
 *   ryk_session_set_f0_map while following replaces the target side and the fallback input side.  follow = 0 (the other two arguments
 *   are ignored) returns to the host's input side.
 * ryk_session_f0_measure_reset: the statistics restart from zero at the next submitted step (in follow mode the input side falls
 *   back to the host's until min_voiced_frames are counted again).
 * ryk_session_f0_measured: waits for stage 1 of the session's submitted steps, then returns the voiced frames counted and the mean
 *   and (population) standard deviation of ln f0 over them (std 0 when fewer than 2 frames).  The variance std * std and the mean are
 *   what an input_statistics file holds.  Any output pointer may be NULL.
 * Refused, changing nothing: a non-finite value, a standard deviation <= 0, follow without measuring or without a map, measuring
 * switched on a session that has run a step, an unknown session. */
typedef struct { double in_mean, in_std, target_mean, target_std; } ryk_f0_map;
int ryk_session_get_f0_map(ryk_engine* e, int session_id, ryk_f0_map* map);
int ryk_session_set_f0_map(ryk_engine* e, int session_id, const ryk_f0_map* map);
int ryk_session_f0_measure(ryk_engine* e, int session_id, int enable);
int ryk_session_f0_follow(ryk_engine* e, int session_id, int follow, int min_voiced_frames, double sd_floor);
int ryk_session_f0_measure_reset(ryk_engine* e, int session_id);
int ryk_session_f0_measured(ryk_engine* e, int session_id, long long* n_voiced, double* mean, double* std);

/* Formant ratio r of a session's converted spectral envelope, in [0.5, 2]; a session starts at 1 (no warp).
 * r > 1 moves the envelope up in frequency, sp'(f) = sp(f / r); r = 2^(s/12) moves it by s semitones.  Paired with a pitch shift
 * (ryk_session_set_f0_map) it changes the apparent size of the speaker rather than only the pitch.
 * Where (DECIDE F1): on stage 2's output, the envelope the synthesizer reads.  Neither network's input changes.  With the edge-padded
 *   log row L[j] = y[min(j, 511)] of the network output y, j = 0 .. 512, bin k becomes exp(L at x = k / r), linearly interpolated in
 *   FP64 and rounded to FP32 (numpy.interp(k / r, arange(513), L)); bins with x >= 512 hold L[512] (r < 1).  r == 1 is the unwarped
 *   expression, bitwise.
 * Not warped (DECIDE F2): aperiodicity (it describes the source); the energy of the envelope is not renormalised; a change is not
 *   smoothed.
 * ryk_session_set_formant: from the next submitted step on; steps already submitted keep theirs.  Allowed with chunks in flight and on
 *   a group member; no device wait, no kernel.  Refused, changing nothing: non-finite, outside [0.5, 2], unknown session.
 * ryk_session_get_formant: the value the NEXT submitted step uses. */
int ryk_session_set_formant(ryk_engine* e, int session_id, double ratio);
int ryk_session_get_formant(ryk_engine* e, int session_id, double* ratio);

/* Input noise suppression (DESIGN.md §4f, DECIDE N1-N3): a decision-directed Wiener filter (Ephraim-Malah) on the model-rate input,
 * ahead of the WORLD analysis, so analysis, silence gate, CREPE and f0 measuring all see the filtered signal.  Frames of N = 512
 * samples at a hop of H = 128 (21.3 ms / 5.3 ms at 24 kHz), periodic sqrt-Hann analysis and synthesis windows, FP64 spectra of 257
 * bins.  Per bin k with noise power profile phi[k], P_m = |X_m[k]|^2 and g = 10^(-reduction_db / 20):
 *   xi_m = 0.98 G_{m-1}^2 P_{m-1} / phi + 0.02 max(P_m / phi - 1, 0),   G_m = max(xi_m / (1 + xi_m), g),   G_{-1} = 1, P_{-1} = 0;
 *   G = 1 where phi[k] == 0.  reduction_db in [0, 40] is the most a bin is attenuated; at 0 the filter only round-trips the FFT.
 * ryk_session_denoise: fresh session only (no chunk pushed); either order with ryk_session_set_input_rate.  The session then analyses
 *   concat(zeros(511), z), z = the filtered model-rate input (511 = N - 1, the least delay that completes every emitted sample), and
 *   ryk_session_io_geometry's delay_in includes the 511.  It starts at reduction_db = 20 with no profile, which passes the signal
 *   through.  Three more kernels per step, on the gate stream; a session without the filter runs exactly the kernels it ran before.
 * ryk_session_set_denoise: from the next submitted step on; steps already submitted keep theirs.  Allowed with chunks in flight and on
 *   a group member; no device wait, no kernel.
 * ryk_session_denoise_learn: the first n_frames frames processed from the next submitted step on (a step processes the frames whose
 *   last sample it brings: 56 or 57 at a 0.3 s chunk) add their P to per-bin FP64 sums in frame order; when the last one is added,
 *   phi = sum / n_frames applies from the following step.  The result depends on the input stream alone: it is bit-identical from run
 *   to run and does not depend on other work on the engine.  A new call restarts the learning.  About 1 s of the user staying quiet
 *   (188 frames at 24 kHz) is a reasonable choice.
 * ryk_session_set_noise_profile: phi[257] from the next submitted step on; it cancels a learning in progress.  This is how a saved
 *   profile is loaded.
 * ryk_session_noise_profile: waits for the gate stream of the submitted steps, then writes the profile the next submitted step uses
 *   and the frames still to learn (0: no learning in progress).  Either pointer may be NULL.
 * ryk_denoise: the same filter over a whole signal on the same kernels: a fresh state, x zero outside [0, n), z = n samples with no
 *   delay.  A session's z with constant settings and profile is bitwise ryk_denoise of its input.  phi may be NULL (no profile).
 * Refused, changing nothing: an unknown session, enabling on a session that ran a step, set / learn / profile calls on a session
 * without the filter, a non-finite reduction_db or one outside [0, 40], n_frames < 1, a profile entry that is negative or not
 * finite. */
int ryk_session_denoise(ryk_engine* e, int session_id);
int ryk_session_set_denoise(ryk_engine* e, int session_id, double reduction_db);
int ryk_session_denoise_learn(ryk_engine* e, int session_id, long long n_frames);
int ryk_session_set_noise_profile(ryk_engine* e, int session_id, const double* phi);
int ryk_session_noise_profile(ryk_engine* e, int session_id, double* phi, long long* frames_left);
int ryk_denoise(ryk_engine* e, const float* x, int n, double reduction_db, const double* phi, float* z);

/* Echo cancellation (DESIGN.md §4g, DECIDE E1-E4): removes from the model-rate input the echo of the far end (what the host played
 * while the chunk was recorded), ahead of the noise suppression and the WORLD analysis.  The microphone and the far end are framed as
 * the noise suppression frames its input (N = 512, H = 128, sqrt-Hann, FP64, 257 bins).  Per bin, a complex FIR over the far end's
 * frames, Y_m = sum_{p < taps} W_p X_{m - delay_frames - p}, is adapted by NLMS (mu = 0.5, delta = 1e-6) in two copies: a background
 * filter B that adapts every frame and a foreground filter F that produces E = D - Y^f.  B is copied into F after 3 consecutive frames
 * with S_b < 0.5 S_f and S_b < S_d (powers smoothed with lambda = 0.9); F is copied into B, skipping B's update, when S_b > 4 S_f;
 * F is cleared when S_f > S_d (it would make the output louder than the microphone, as a far end correlated with the near end can).
 * The output is Z = G E^f with the residual suppression G = max(g_e, 1 - Yhat / (Ehat + 1e-12)), g_e = 10^(-db / 20) (Yhat, Ehat:
 * smoothed |Y^f|^2, |E^f|^2).  With noise suppression on, its gain scan then runs on Z.
 * ryk_session_echo_cancel: fresh session only (no chunk pushed); either order with ryk_session_denoise and
 *   ryk_session_set_input_rate.  taps in [1, 64] frames, delay_frames in [0, 256]: echoes up to (delay_frames + taps) * 128 model
 *   samples are covered.  The session then analyses concat(zeros(511), z) like the noise suppression; with both on they share one
 *   frame stage, so the delay grows by 511 once (ryk_session_io_geometry's delay_in).  Residual suppression starts at 0 dB.  Four
 *   more kernels per step on the gate stream (two forward transforms, the canceller's scan, the inverse transforms; one more kernel
 *   than the noise suppression alone when both are on), plus the far end's resampler at a device input rate.  A session without it
 *   runs exactly the kernels it ran before.
 * ryk_session_echo_reference: the far end of the next submitted step: far[n], n = the session's chunk length at its input rate
 *   (n_in).  A step submitted without one uses zeros; a second call before the step replaces the first.  It applies to
 *   ryk_session_submit / _push / _push_device, and for a group member to the next ryk_group_submit / _push_device.  At a device
 *   input rate the far end goes through its own streaming copy of the input resampler (same taps, same delay), aligned sample for
 *   sample with the microphone.
 * ryk_session_set_echo_suppression: db in [0, 40] from the next submitted step on; allowed with chunks in flight and on a group
 *   member; no device wait, no kernel.  0 dB is a gain of exactly 1: the output is the linear canceller's bit for bit.
 * ryk_session_echo_stats: waits for the gate stream of the submitted steps, then writes the frames of the last step and its echo
 *   return loss enhancement 10 log10(sum |D|^2 / sum |Z|^2) over its bins and frames (0 when the microphone was silent).  The per-bin
 *   sums are added on the host in bin order, so the value is deterministic.  Either pointer may be NULL.
 * ryk_echo_cancel: the same canceller over a whole signal on the same kernels: a fresh state, mic and far zero outside [0, n), z = n
 *   samples with no delay; phi == NULL skips the noise suppression (reduction_db is then checked but unused).  A session's z with
 *   constant settings is bitwise ryk_echo_cancel of its model-rate microphone and far end.
 * Refused, changing nothing: an unknown session, enabling on a session that ran a step or twice, taps or delay_frames out of range,
 * a reference of the wrong length, reference / suppression / stats calls on a session without the canceller, a non-finite db or one
 * outside [0, 40]. */
int ryk_session_echo_cancel(ryk_engine* e, int session_id, int taps, int delay_frames);
int ryk_session_echo_reference(ryk_engine* e, int session_id, const float* far, int n);
int ryk_session_set_echo_suppression(ryk_engine* e, int session_id, double db);
int ryk_session_echo_stats(ryk_engine* e, int session_id, long long* frames, double* erle_db);
int ryk_echo_cancel(ryk_engine* e, const float* mic, const float* far, int n, int taps, int delay_frames, double suppression_db,
                    double reduction_db, const double* phi, float* z);

/* Output limiter (DESIGN.md §4i, DECIDE L1-L4): a look-ahead peak limiter on the samples a session returns, at its output rate, after
 * the NaN scrub and the output resampler.  With y the stream the session returns without it, in FP64:
 *   g0[u] = 1 if G |y[u]| <= c else c / (G |y[u]|) (1 for u < 0), c = 10^(ceiling_db / 20), G = gain (the host's output scale: the
 *   ceiling applies to G y, the played level, while the session keeps returning unscaled samples);
 *   m[s] = min of g0[u] over u in [s - hold, s + lookahead - 1];  g[t] = (sum over s = t - lookahead + 1 .. t of m[s]) / lookahead,
 *   summed in ascending s from 0.0;  z[t] = g[t] y[t].
 * So |G z| <= c (1 + 1e-12); where G |y| <= c over the whole window z is y bit for bit; a lone peak lowers the gain with a linear ramp
 * over lookahead samples, a hold of hold samples and a linear ramp back.  No sample-to-sample recursion: the streamed output is bitwise
 * the whole-signal output.
 * ryk_session_limiter: fresh session only (no chunk pushed), once; either order with ryk_session_set_output_rate (which re-derives the
 *   limiter at the new rate).  lookahead_ms in [0.5, 10] gives lookahead = max(1, round(lookahead_ms * rate / 1000)) output-rate
 *   samples, hold_ms in [0, 500] gives hold = round(hold_ms * rate / 1000), both fixed from then on (rounded half to even).  The
 *   session then returns concat(zeros(lookahead), z): every step returns as many samples as before (max_out unchanged), the output
 *   delay grows by lookahead and the last lookahead samples of a finite input stay in the limiter.  The limiter starts at
 *   ceiling_db = -1 and gain = 1.  Three more kernels per step on the decode stream; a session without it runs exactly the kernels it
 *   ran before.  With constant settings the session's output is bitwise concat(zeros(lookahead), ryk_limit(y)) over its length.
 * ryk_session_set_limiter: ceiling_db in [-24, 0], gain finite and > 0, from the next submitted step on (g0[u] uses the settings of the
 *   step that returns y[u] from upstream); allowed with chunks in flight and on a group member; no device wait, no kernel.
 * ryk_session_get_limiter: the settings of the next step; lookahead and hold in output-rate samples (lookahead is the added output
 *   delay).  Any pointer may be NULL.
 * ryk_session_limiter_stats: waits for the decode stream of the submitted steps, then writes for the samples the last step returned
 *   (the leading zeros excluded) the largest reduction -20 log10(min g) (0 when none) and the number of samples with g < 1.  Either
 *   pointer may be NULL.
 * ryk_limit: the same limiter over a whole signal on the same kernels: a fresh state, y zero outside [0, n), z = n samples with no
 *   delay.
 * Refused, changing nothing: an unknown session, enabling on a session that ran a step or twice, settings out of range or not finite,
 * set / get / stats calls on a session without the limiter. */
int ryk_session_limiter(ryk_engine* e, int session_id, double lookahead_ms, double hold_ms);
int ryk_session_set_limiter(ryk_engine* e, int session_id, double ceiling_db, double gain);
int ryk_session_get_limiter(ryk_engine* e, int session_id, double* ceiling_db, double* gain, int* lookahead, int* hold);
int ryk_session_limiter_stats(ryk_engine* e, int session_id, double* reduction_db, long long* limited);
int ryk_limit(ryk_engine* e, const double* y, int n, int rate, double lookahead_ms, double hold_ms, double ceiling_db, double gain,
              double* z);

/* Automatic gain control (DESIGN.md §4j, DECIDE A1-A4): brings the speaker to a target level ahead of the WORLD analysis.  It runs on
 * the model-rate signal x the analysis would read (after the input resampler, the echo canceller and the noise suppression; the leading
 * zeros of delay_in included), in FP64 with + - * / sqrt min max only:
 *   P_m = mean of x^2 over block m = [256 m, 256 m + 256) (global positions; squares added in ascending order from 0.0);
 *   a block is active when P_m > Gt = 10^(gate_db / 10); the level E is P_m at the first active block, then E += a (P_m - E) at each
 *   active block, a = -expm1(-256 / (0.4 fs)); an inactive block leaves E and the gain;
 *   on an active block g_m = min(max(g*, g_{m-1} s_dn), g_{m-1} s_up), g* = min(max(sqrt(T / E), 1 / gmax), gmax),
 *   T = 10^(target_db / 10), gmax = 10^(max_gain_db / 20), s_up = 10^(6 * 256 / (20 fs)), s_dn = 10^(-24 * 256 / (20 fs))
 *   (at most +6 / -24 dB per second); g_m = 1 for m < 0;
 *   z[t] = (float)((g_{m-2} + (g_{m-1} - g_{m-2}) (j + 1) / 256) x[t]) for t = 256 m + j.
 * The gain uses only blocks completed before the sample: it is causal, continuous and adds no delay.  With max_gain_db = 0 from a
 * fresh state, or an input that never passes the gate, z is x bit for bit.
 * ryk_session_agc: fresh session only (no chunk pushed), once; either order with ryk_session_denoise, _echo_cancel and
 *   _set_input_rate (the AGC runs at the model rate, so no rate changes it).  One more kernel per step on the gate stream; delay_in,
 *   ryk_session_io_geometry and every capacity are unchanged.  A session without it runs exactly the kernels it ran before.  With
 *   constant settings the session analyses ryk_agc(x) bitwise, however the stream is cut into steps.
 * ryk_session_set_agc: from the next submitted step on (block m uses the settings of the step that brings its last sample); allowed with
 *   chunks in flight and on a group member; no device wait, no kernel.
 * ryk_session_get_agc: the settings of the next submitted step, and in linear[7] (may be NULL) the values the device uses: T, Gt, gmax,
 *   1 / gmax, a, s_up, s_dn, computed on the host with its libm.  Any pointer may be NULL.
 * ryk_session_agc_stats: waits for the gate stream of the submitted steps, then writes 10 log10 E (-inf while no block has been
 *   active), 20 log10 of the last completed block's gain, and the number of blocks completed in the last step that were active.  The
 *   logarithms are taken on the host.  Any pointer may be NULL.
 * ryk_agc: the same gain control over a whole signal at model rate fs on the same kernel: a fresh state, z = n samples, no delay.
 * Refused, changing nothing: an unknown session, enabling on a session that ran a step or twice, settings not finite or outside
 * target_db [-40, -6], max_gain_db [0, 30], gate_db [-80, -20], set / get / stats calls on a session without the AGC. */
int ryk_session_agc(ryk_engine* e, int session_id, double target_db, double max_gain_db, double gate_db);
int ryk_session_set_agc(ryk_engine* e, int session_id, double target_db, double max_gain_db, double gate_db);
int ryk_session_get_agc(ryk_engine* e, int session_id, double* target_db, double* max_gain_db, double* gate_db, double* linear);
int ryk_session_agc_stats(ryk_engine* e, int session_id, double* level_db, double* gain_db, int* active);
int ryk_agc(ryk_engine* e, const float* x, int n, int fs, double target_db, double max_gain_db, double gate_db, float* z);

/* Pitch correction (DESIGN.md §4m, DECIDE P1-P4): pulls each converted note toward the nearest pitch of a musical scale, with a retune
 * time.  It runs on the converted f0 the synthesizer is given, one value per frame (0: unvoiced), in stream order, in FP64:
 *   a voiced frame (0 < f0 < inf) sits at s = 69 + 12 (log2 f0 - log2 a4_hz) semitones; its target n is the nearest note whose pitch class
 *   (n - key) mod 12 is set in scale_mask (bit j: pitch class key + j; ties to the lower note), except that the previous voiced frame's
 *   target is kept while it is in the scale and |s - n_prev| < 0.65 (hysteresis: a note sung between two scale notes does not flap);
 *   d = n - s;  c = d on the first voiced frame after an unvoiced one (no glide across a gap), else c += beta (d - c),
 *   beta = -expm1(-frame_period / retune_ms), 1 for retune_ms = 0 (a hard snap);
 *   f0' = f0 exp2(amount c / 12).  Any other frame is returned as it is and keeps c and the previous target.
 * amount = 0 returns every frame bit for bit, so the correction can be faded out and in mid-stream.  The correction reaches 1 - 1/e of a
 * note change retune_ms after it.
 * ryk_session_pitch_correct: fresh session only (no chunk pushed), once.  The correction starts at amount 0 (key 0, the chromatic
 *   scale 0xfff, a4_hz 440, retune_ms 50), so it changes nothing until ryk_session_set_pitch_correct.  It corrects the frames each step
 *   appends to the decode window, once each and in stream order, so with a decode extra the synthesizer reads every frame of its window
 *   corrected exactly once.  One more kernel per step on the decode stream; latency, geometry and capacities are unchanged.  A session
 *   without it runs exactly the kernels it ran before.  With constant settings the synthesizer is given ryk_pitch_correct of the f0 the
 *   session gives it without the correction, bitwise (as float).  A voice switch and group membership keep its state.
 * ryk_session_set_pitch_correct: key in [0, 11], scale_mask a nonzero 12-bit mask, a4_hz in [400, 480], retune_ms in [0, 1000],
 *   amount in [0, 1]; from the next submitted step on (chunks in flight keep theirs); allowed with chunks in flight and on a group
 *   member; no device wait, no kernel.
 * ryk_session_get_pitch_correct: the settings of the next submitted step.  Any pointer may be NULL.
 * ryk_session_pitch_stats: waits for the decode stream of the submitted steps, then writes the voiced frames the last step corrected
 *   and the mean and largest |amount c| over them in cents (0 when none).  Any pointer may be NULL.
 * ryk_pitch_correct: the same correction over n frames of a whole signal on the same kernel from a fresh state (fs positive, frame_period
 *   the stream's frame period in ms, which sets beta).
 * Refused, changing nothing: an unknown session, enabling on a session that ran a step or twice, settings out of range or not finite,
 * an empty scale mask, set / get / stats calls on a session without the correction. */
int ryk_session_pitch_correct(ryk_engine* e, int session_id);
int ryk_session_set_pitch_correct(ryk_engine* e, int session_id, int key, int scale_mask, double a4_hz, double retune_ms, double amount);
int ryk_session_get_pitch_correct(ryk_engine* e, int session_id, int* key, int* scale_mask, double* a4_hz, double* retune_ms,
                                  double* amount);
int ryk_session_pitch_stats(ryk_engine* e, int session_id, long long* voiced, double* mean_cents, double* max_cents);
int ryk_pitch_correct(ryk_engine* e, const double* f0, int n, int fs, double frame_period, int key, int scale_mask, double a4_hz,
                      double retune_ms, double amount, double* out);

/* Moving a session (DESIGN.md §4k): a snapshot of a quiescent session's stream state, restored bit for bit as a new session on the same
 * engine, another engine of the same device or an engine of another device.  After k steps of session A, a snapshot restored as B, the
 * next chunks fed to A and B give the same outputs bit for bit: windows, resampler positions, the learned noise profile, the echo
 * canceller's filters and far-end ring, the AGC's level and gains, the limiter's histories, the f0 statistics and f0 map, the
 * synthesizer's rings and every setting made since the last step carry over.
 * ryk_session_snapshot_size / ryk_session_snapshot: the session must be quiescent: every ryk_session_submit chunk collected, and for a
 *   group member every ryk_group_submit chunk of its group.  The call waits for the session's streams, then copies its state into
 *   `buf` (bytes = the size the first call returned) through one pinned staging buffer.  It changes nothing in the session, which
 *   keeps running as if no snapshot had been taken.  A group member can be snapshotted: its stream state does not depend on the group.
 * ryk_session_restore: creates a session on engine e converting into voice_id, with the configuration the blob records (session
 *   config, device rates and their taps, f0 method, noise suppression, echo cancellation with its taps and delay, limiter with its
 *   look-ahead and hold, AGC, f0 measuring, pitch correction), through the same code ryk_session_create and the enabling calls run, copies the state
 *   into the new session's buffers and sets its step count to the source's.  *id receives the new session.  To restore a group,
 *   restore its members and group them again (ryk_group_create / ryk_group_add).
 *   voice_id names the source's voice as loaded on engine e: the stream continues, so the f0 map (both sides, a pitch offset or a
 *   measured input side included) and the formant ratio are carried as they are and nothing of the voice's statistics is applied.  To
 *   convert the moved stream into another voice, restore it and then call ryk_session_set_voice, which installs that voice's map.
 *   Refused before anything is allocated: a malformed, truncated or corrupt blob, an unknown format version, an engine whose precision
 *   or stage-1 mode differ from the recorded ones, a voice whose stage-1 or stage-2 (in, out, base) channels differ from the recorded
 *   ones, CREPE (f0 method 2) without a complete CREPE model and resampler taps for the session's rate.  A failure later frees
 *   whatever the call made.
 * ryk_reblock_snapshot_size / ryk_reblock_snapshot / ryk_reblock_restore: the same for a re-blocker (its fragment, length and
 *   ping-pong selector, and its push count); the snapshot waits for the re-blocker's last push.
 * ryk_snapshot_describe (host only, no engine or device): verifies a blob's header, size, checksum and section walk and reports its
 *   kind (1 session, 2 re-blocker, 3 pipeline, 4 drift stage), format version, the recorded configuration of a session or re-blocker (either
 *   pointer may be NULL) and up to `capacity` section tags (four characters, first in the lowest byte) and payload sizes.  Returns the
 *   number of sections.
 * ryk_snapshot_seal (host only): writes the total size and the checksum into the header of a blob of `bytes` bytes whose magic,
 *   version, kind and sections are in place (how a caller writes a blob of its own in the container, e.g. a pipeline blob). */
typedef struct {
  ryk_session_config cfg;
  int voice_id;                              /* the source session's voice */
  int precision, stage1_fused, f0_method;    /* the source engine's */
  int stage1_channels[3], stage2_channels[3];   /* (in, out, base) of the voice's U-Nets */
  int in_rate, in_up, in_down, in_taps;      /* device input rate (0: none) and its resampler */
  int out_rate, out_up, out_down, out_taps;  /* device output rate (0: none) and its resampler */
  int denoise, echo, echo_taps, echo_delay_frames, limiter, agc, f0_measure;
  double limiter_lookahead_ms, limiter_hold_ms;
  long long step;                            /* chunks the session has processed */
} ryk_snapshot_session;
typedef struct {
  int out_audio_chunk, max_in, n_fft, hop;
  double threshold_db;
  long long pushed;
} ryk_snapshot_reblock;
int ryk_session_snapshot_size(ryk_engine* e, int session_id, size_t* bytes);
int ryk_session_snapshot(ryk_engine* e, int session_id, void* buf, size_t bytes);
int ryk_session_restore(ryk_engine* e, int voice_id, const void* buf, size_t bytes, int* session_id);
int ryk_reblock_snapshot_size(ryk_engine* e, int reblock_id, size_t* bytes);
int ryk_reblock_snapshot(ryk_engine* e, int reblock_id, void* buf, size_t bytes);
int ryk_reblock_restore(ryk_engine* e, const void* buf, size_t bytes, int* reblock_id);
int ryk_snapshot_describe(const void* buf, size_t bytes, int* kind, int* version, ryk_snapshot_session* session,
                          ryk_snapshot_reblock* reblock, unsigned* tags, unsigned long long* sizes, int capacity);
int ryk_snapshot_seal(void* buf, size_t bytes);
/* Wall time of the engine's last successful snapshot or restore call, in ms: device_ms from enqueueing its staged copies to their end,
 * host_ms the rest of the call (the waits for the session's streams, building the session, packing, parsing and the checksum).
 * Either pointer may be NULL. */
int ryk_snapshot_last_times(ryk_engine* e, double* host_ms, double* device_ms);

/* Clock drift compensation (DESIGN.md §4l, DECIDE D1-D4): an asynchronous resampler on the played stream, for an output sound card
 * whose clock differs from the input card's.  A standalone object of the engine, like a re-blocker; no session runs it.  With
 * z = concat(zeros(W), x) the input stream and inc = llrint(2^32 / (1 + ppm 1e-6)) of the setting in force, output m reads z at
 * q_m = inc_0 + ... + inc_(m-1) (int64, 2^-32 samples).  For q = i 2^32 + f: phi = f >> 23, w = (f & (2^23 - 1)) 2^-23,
 *   c_t = T[(2W - 1 - t) P + phi] + w (T[(2W - 1 - t) P + phi + 1] - T[(2W - 1 - t) P + phi]),   t = 0 .. 2W - 1,
 *   y_m = sum over t of c_t z[i - W + 1 + t] in ascending t from 0.0, in FP64 with round-to-nearest operations only,
 * with the table T of P = 512 phases and half-width W = 16 (2WP + 1 entries, entry k at k / P - W; wave_io.drift_filter designs it).
 * Output m is emitted by the push that brings z[i + W]: after N input samples every m with q_m < N 2^32 has been emitted.  So the
 * delay is W samples, at ppm 0 the output is concat(zeros(W), x) bit for bit (the table's integer entries are 0 and its centre 1),
 * and however the input is cut into pushes the outputs are those of the whole signal.  The output runs (1 + ppm 1e-6) times as many
 * samples as the input.
 * ryk_drift_create: max_in in [1, 2^24] samples per push, max_ppm in (0, 2000], the table (phases 512, half_width 16, finite); the
 *   setting starts at ppm 0.  It works at whatever rate its caller's samples have and creates no device rate.
 * ryk_drift_set: ppm finite with |ppm| <= max_ppm, from the next push on; the position continues from where it is.  No device work.
 * ryk_drift_get: the setting of the next push and its inc.  Either pointer may be NULL.
 * ryk_drift_push: host buffers, synchronous (as ryk_reblock_push): n in [0, max_in] samples in, *n_out samples out; y_capacity must
 *   be at least n + ceil(n max_ppm 1e-6) + 2, the most one push can emit.  One kernel launch; the count is decided on the device.
 * ryk_drift_stats: input samples consumed and outputs produced since creation.  Either pointer may be NULL.
 * ryk_drift_resample: the same kernel over a whole signal from a fresh state, followed by W zeros: len = n + W samples in, y_capacity
 *   at least len + ceil(len |ppm| 1e-6) + 2, |ppm| <= 2000.
 * ryk_drift_snapshot_size / _snapshot / _restore: the object's state as a blob of the snapshot container, kind 4, sections DCNF
 *   (ryk_snapshot_drift followed by the table), DSTA (position, counts, inc and ppm of the next push) and DHIS (the 2W kept samples).
 *   The restored object continues the stream bit for bit, on this engine or another.  The restore refuses before it allocates: what
 *   ryk_snapshot_describe refuses, another kind, sections of other sizes, a configuration or setting ryk_drift_create / _set refuse,
 *   an inc that is not that of the recorded ppm, a position outside [0, 2^33).
 * Refused, changing nothing: an unknown id, the arguments named above out of range. */
typedef struct {
  int max_in, phases, half_width, reserved;
  double max_ppm;
  long long pushed;
} ryk_snapshot_drift;
int ryk_drift_create(ryk_engine* e, int max_in, double max_ppm, const double* table, int phases, int half_width, int* drift_id);
int ryk_drift_destroy(ryk_engine* e, int drift_id);
int ryk_drift_set(ryk_engine* e, int drift_id, double ppm);
int ryk_drift_get(ryk_engine* e, int drift_id, double* ppm, long long* inc);
int ryk_drift_push(ryk_engine* e, int drift_id, const double* x, int n, double* y, int y_capacity, int* n_out);
int ryk_drift_stats(ryk_engine* e, int drift_id, long long* consumed, long long* produced);
int ryk_drift_resample(ryk_engine* e, const double* x, int n, double ppm, const double* table, int phases, int half_width, double* y,
                       int y_capacity, int* n_out);
int ryk_drift_snapshot_size(ryk_engine* e, int drift_id, size_t* bytes);
int ryk_drift_snapshot(ryk_engine* e, int drift_id, void* buf, size_t bytes);
int ryk_drift_restore(ryk_engine* e, const void* buf, size_t bytes, int* drift_id);

/* Diagnostics: device timeline (ms) of the last <= 8 steps x 5 stages {gate, analysis, stage 1, stage 2, synthesis}; needs
 * RYK_STAGE_TIMES=1 in the environment at session creation.  start/end hold 40 floats; returns the number of steps. */
int ryk_session_stage_times(ryk_engine* e, int session_id, float* start, float* end);

/* ---- session groups: several streams of one GPU sharing one batched stage-2 forward -------------------
 * BASELINE config 5 / SURVEY 8(e) "per-GPU batch = streams resident on it": the reference would run one
 * SuperResolution.convert (voice_changer.py:41) per stream; a group stacks the members' padded log-spectrograms into
 * one (B, 1, Tp, 512) stage-2 input per step.  Analysis, gate, stage 1 and synthesis stay per stream (per-stream state,
 * data-dependent lengths).  Members are distinct sessions in no group, with the same window length, chunk length and device rates;
 * they may be fresh or may have run steps, alone or in another group.  Member i of every call is the session in slot i: session_ids[i]
 * after ryk_group_create, then as ryk_group_add / _remove change it (ryk_group_members lists it).  Outputs per member are those of an
 * ungrouped session up to the FP16 stage-2 rounding.
 * Members may convert into different voices when their stage-2 models have the same channels, the engine is in precision 1, every
 * stage-2 layer runs on a kernel that reads weights per batch item (the base-64 nets) and there are at most 8 distinct voices: the one
 * batched forward reads each member's weights from its voice.  Other groups of several voices are refused.
 * Membership changes between steps.  ryk_group_add makes the session the group's last member: its next step is the group's next step.
 * ryk_group_remove takes a member out (the members after it move down one slot); it continues as an ungrouped session
 * (ryk_session_submit / _collect / _push_device).  Either way the session's stream state (windows, synthesizer, step count) carries
 * over, so its audio continues as if nothing happened.  ryk_group_create and ryk_group_add refuse a session with an uncollected
 * ryk_session_submit chunk, and _add / _remove refuse while the group has an uncollected ryk_group_submit chunk; device-resident steps
 * count as collected.  The last member cannot be removed: destroy the group instead.  A refused call changes nothing.  A change waits
 * for the device (the group's stage-2 plan is rebuilt at the new batch size) and launches no kernel.
 * ryk_group_members returns the member count and writes up to `capacity` member ids in slot order (session_ids may be NULL). */
int ryk_group_create(ryk_engine* e, const int* session_ids, int n_sessions, int* group_id);
int ryk_group_destroy(ryk_engine* e, int group_id);        /* members survive, ungrouped */
int ryk_group_size(ryk_engine* e, int group_id);
int ryk_group_add(ryk_engine* e, int group_id, int session_id);
int ryk_group_remove(ryk_engine* e, int group_id, int session_id);
int ryk_group_members(ryk_engine* e, int group_id, int* session_ids, int capacity);
int ryk_group_submit(ryk_engine* e, int group_id, const float* const* waves, int n, long long* ticket);
int ryk_group_collect(ryk_engine* e, int group_id, long long ticket, double* const* outs, int out_capacity, int* n_outs);
int ryk_group_push_device(ryk_engine* e, int group_id, const float* const* waves_dev, int n, double* const* outs_dev,
                          int out_capacity, int* const* n_outs_dev);

/* ---- diagnostics -------------------------------------------------------------------------------------- */
/* Harvest internals of the most recent analysis with this plan (engine in f0 method 1): info = {channels, 1 ms frames, decimated
 * length, fft size, candidate columns, decimation ratio, used columns}; y [info[2]], raw [channels][frames], cand / score
 * [frames][columns] (after refinement and removal), best / basic [frames], f0_raw [n / hop + 1] (before StoneMask).  Any may be NULL. */
int ryk_debug_harvest(ryk_engine* e, int n, int fs, double frame_period_ms, double f0_floor, double f0_ceil, int* info, double* y,
                      double* raw, double* cand, double* score, double* best, double* basic, double* f0_raw);
/* Stage-2 row bands.  A streaming session keeps only the chunk's frames of each converted window, so its stage-2 forward computes
 * only the decoder rows those frames depend on.
 * ryk_stage2_row_bands (host only): for a (Tp, W) input of which rows [keep_begin, keep_begin + keep_len) are kept,
 *   bands[2 i], bands[2 i + 1] = the class-local output rows [y0, y1) that layer i (0..15) of an FP16 plan computes.
 * ryk_stage2_tail_rows (host only): a session pads its Tw-frame window to Tp rows with one repeated row, and the encoder computes
 *   one copy of the rows that depend only on that padding.  For such a window with the rows above kept, tail[4 i .. 4 i + 3] =
 *   {skip_y0, skip_y1, run_y0, run_y1} of layer i: it does not compute output rows [skip_y0, skip_y1), and its load boxes wholly
 *   inside input rows [run_y0, run_y1) read from row run_y0 instead (zeros: none).
 * ryk_test_stage2_forward: one forward of the loaded stage-2 net on a fresh plan whose buffers are first filled with NaN;
 *   x, y: [B][Tp][512] float32 network input / output.  mode 0 = every row; 1 = banded for the hull of the n_keep ranges
 *   [keep_begin[i], keep_begin[i] + keep_len[i]); 2 = as 1 with every layer split along K as in the full plan; 3 = as 2 with the
 *   encoder skipping the padded tail of an input whose rows [Tw, Tp) are equal.  Rows outside the band are left NaN. */
int ryk_stage2_row_bands(int Tp, int W, int keep_begin, int keep_len, int* bands);
int ryk_stage2_tail_rows(int Tp, int W, int Tw, int keep_begin, int keep_len, int* tail);
int ryk_test_stage2_forward(ryk_engine* e, int B, int Tp, int n_keep, const int* keep_begin, const int* keep_len, int mode, int Tw,
                            const float* x, float* y);
/* One conv (transposed = 0) or transposed-conv layer of the U-Nets in isolation, host fp32 NHWC tensors in and
 * out, weights in the Chainer layout; use_tc selects the FP16 wgmma kernel (1) or the FP32 CUDA-core kernel (0).
 * `repeat` extra timed runs report the mean device time per run (ms) -- used by the unit parity tests and ncu.
 * ksplit_tiles > 0 makes the wgmma kernel split K as for a layer of that many output tiles (0: the layer's own count);
 * *ksplit (may be NULL) receives the split factor the wgmma kernel ran with. */
int ryk_test_conv_layer(ryk_engine* e, int transposed, int k, int stride, int pad, int B, int Hin, int Win, int C0, int C1, int Cout,
                        const float* in0, const float* in1, const float* W, const float* scale, const float* shift, int act,
                        int use_tc, int repeat, int ksplit_tiles, float* out, float* ms_per_run, int* ksplit);
/* CREPE convolutions with an explicit back-end: 0 = the FP32 CUDA-core kernel (ryk_crepe_predict, sessions in precision 0),
 * 1 = the 3xTF32 tensor-core kernel (sessions in precision 1).
 * ryk_crepe_test_conv: one layer in isolation, x [F][Win][Cin], W (Cout, Cin, k), stride 1, no padding ->
 *   y = ReLU(conv + bias) [F][Win - k + 1][Cout]; CREPE's first layer is given in its im2col form (Win 256, Cin 512, k 1).
 * ryk_crepe_test_network: the loaded model and decoders on a host 16 kHz signal (frames as ryk_crepe_predict): activation
 *   [frames][360], path and voicing [frames] (any may be NULL); repeat > 0 further runs report their mean device time. */
int ryk_crepe_test_conv(ryk_engine* e, int backend, int F, int Win, int Cin, int Cout, int k, const float* x, const float* W,
                        const float* bias, float* y);
int ryk_crepe_test_network(ryk_engine* e, int backend, const float* audio16k, int n, double step_ms, float* activation, int* path,
                           int* voicing, int repeat, float* ms_per_run);

#ifdef __cplusplus
}
#endif
#endif  /* RYK_H_ */
