// session_controls.cu -- the host API of a session's optional stages (DESIGN.md §4a, §4f-§4j, §4m).  The setters change host state only;
// host_block_sync carries it to the device in front of the stage's readers of the next submitted step, alone or in a group.
#include <math.h>
#include <string.h>

#include "../../include/ryk.h"
#include "session.h"

namespace ryk {

// The session when its stage (&Session::dn, ...) is on, else nullptr with the error set: "no such session", or the stage's refusal.
template <typename S>
static Session* stage_session(Engine* e, int id, S Session::*stage) {
  Session* s = get_session(e, id);
  if (!s) set_error("no such session");
  else if (!(s->*stage).on) set_error(S::refusal);
  return s && (s->*stage).on ? s : nullptr;
}

// *out = the device struct *dev, copied behind everything queued on stream st (for a meter: behind every submitted step that writes it).
template <typename T>
static int read_back(Engine* e, const T* dev, cudaStream_t st, T* out) {
  void* hp = nullptr;
  if (engine_pinned(e, sizeof(T), &hp)) return -1;
  RYK_CUDA(cudaMemcpyAsync(hp, dev, sizeof(T), cudaMemcpyDeviceToHost, st));
  RYK_CUDA(cudaStreamSynchronize(st));
  memcpy(out, hp, sizeof(T));
  return 0;
}

// Copies the host value *v into *dev through the engine's pinned staging on the engine stream, behind the zero-fills of the stage's new
// buffers, and waits: the staging is the engine's, and the session's streams do not wait for the engine stream.
template <typename T>
static int upload_wait(Engine* e, T* dev, const T* v) {
  void* hp = nullptr;
  if (engine_pinned(e, sizeof(T), &hp)) return -1;
  memcpy(hp, v, sizeof(T));
  RYK_CUDA(cudaMemcpyAsync(dev, hp, sizeof(T), cudaMemcpyHostToDevice, e->stream));
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  return 0;
}

// (Re)allocates the output limiter at the session's output rate and max_out (DECIDE L1): its shape, scratch, meter and settings block,
// and each parity's history, position and output.  The next submitted step copies `first` into the settings block.
int limiter_alloc(Session* s, const LimParams& first) {
  BufferSet& m = s->mem;
  LimWork& w = s->lim.w;
  limiter_shape(s->out.rate ? s->out.rate : s->cfg.fs, s->lim.lookahead_ms, s->lim.hold_ms, &w.L, &w.R);
  w.max_n = s->max_out;
  size_t n_g0, n_t32, n_t1k, n_m;
  limiter_scratch_sizes(w, &n_g0, &n_t32, &n_t1k, &n_m);
  if (host_block_alloc(m, s->lim.block, &w.params, first) || m.device(&w.meter, 1) || m.device(&w.g0, n_g0) || m.device(&w.t32, n_t32) ||
      m.device(&w.t1k, n_t1k) || m.device(&w.m, n_m))
    return -1;
  for (ParitySet& p : s->par)
    if (m.device(&p.lim.g0, (size_t)w.R + 2 * w.L - 1) || m.device(&p.lim.y, w.L) || m.device(&p.lim.st, 1) ||
        m.device(&p.d_lim_out, s->max_out))
      return -1;
  return 0;
}

// The frame stage noise suppression and echo cancellation share (N1, E1): the microphone's transforms, overlap-add and stream state,
// allocated by whichever of the two is enabled first.  Step 0 reads par[0]: G_{-1} = 1.
static int frame_stage_alloc(Engine* e, Session* s) {
  DenoiseWork& w = s->frame.w;
  if (w.spec) return 0;
  BufferSet& m = s->mem;
  w.max_frames = denoise_max_frames(s->n_wave);
  if (m.device(&w.spec, (size_t)kDnBins * w.max_frames) || m.device(&w.frames, (size_t)kDnN * w.max_frames) || m.device(&w.done, 1) ||
      m.device(&s->frame.d_chunk, s->n_wave))
    return -1;
  for (ParitySet& p : s->par) if (m.device(&p.input[kMic].dn, 1)) return -1;
  DenoiseState st;
  denoise_state_init(&st);
  return upload_wait(e, s->par[0].input[kMic].dn, &st);
}

static void agc_set_next(Session* s, double target_db, double max_gain_db, double gate_db) {
  s->agc.db[0] = target_db; s->agc.db[1] = max_gain_db; s->agc.db[2] = gate_db;
  s->agc.block.edit() = agc_params(s->cfg.fs, target_db, max_gain_db, gate_db);
}

}  // namespace ryk

using namespace ryk;

extern "C" {

// ---- the session's f0 map and the statistics of its speaker (DESIGN.md §4a) ----
int ryk_session_get_f0_map(ryk_engine* h, int id, ryk_f0_map* map) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(map != nullptr, "null argument");
  const F0Map& f = s->f0.block.next;
  map->in_mean = f.mu_in; map->in_std = f.sd_in; map->target_mean = f.mu_tgt; map->target_std = f.sd_tgt;
  return 0;
}

int ryk_session_set_f0_map(ryk_engine* h, int id, const ryk_f0_map* map) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(map != nullptr, "null argument");
  RYK_CHECK(isfinite(map->in_mean) && isfinite(map->in_std) && isfinite(map->target_mean) && isfinite(map->target_std),
            "the f0 map must be finite");
  RYK_CHECK(map->in_std > 0 && map->target_std > 0, "the standard deviations of the f0 map must be positive");
  F0Map& f = s->f0.block.edit();
  f.mu_in = map->in_mean; f.sd_in = map->in_std; f.mu_tgt = map->target_mean; f.sd_tgt = map->target_std;
  f.has_stats = 1;
  return 0;
}

int ryk_session_f0_measure(ryk_engine* h, int id, int enable) {
  Session* s = fresh_session(&h->impl, id, "f0 measurement can only be switched on a fresh session (no chunk pushed): the head of stage 1 is captured at the first steps");
  if (!s) return -2;
  RYK_CHECK(enable || !s->f0.block.next.follow, "the session follows its measurement: turn follow mode off first");
  s->f0.on = enable != 0;
  return 0;
}

int ryk_session_f0_follow(ryk_engine* h, int id, int follow, int min_voiced_frames, double sd_floor) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  F0Map& f = s->f0.block.next;
  if (follow) {
    RYK_CHECK(s->f0.on, "follow mode needs f0 measurement (ryk_session_f0_measure)");
    RYK_CHECK(f.has_stats, "follow mode needs an f0 map: the voice has no f0 statistics and none were set on the session");
    RYK_CHECK(min_voiced_frames >= 1, "min_voiced_frames must be at least 1");
    RYK_CHECK(isfinite(sd_floor) && sd_floor > 0, "sd_floor must be finite and positive");
    f.min_voiced = min_voiced_frames; f.sd_floor = sd_floor;
  }
  f.follow = follow != 0;
  s->f0.block.dirty = true;
  return 0;
}

int ryk_session_f0_measure_reset(ryk_engine* h, int id) {
  Session* s = stage_session(&h->impl, id, &Session::f0);
  if (!s) return -2;
  s->f0.reset = true;
  s->f0.block.dirty = true;          // follow mode: back to the host's input side until min_voiced_frames are counted again
  return 0;
}

int ryk_session_f0_measured(ryk_engine* h, int id, long long* n_voiced, double* mean, double* std_) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = stage_session(e, id, &Session::f0);
  if (!s) return -2;
  F0Stats st = {};
  // behind the head of stage 1 of every submitted step (a reset not yet submitted already reads as empty)
  if (!s->f0.reset && read_back(e, s->f0.d_stats, s->sC, &st)) return -1;
  if (n_voiced) *n_voiced = st.n;
  if (mean) *mean = st.mean;
  if (std_) *std_ = st.n >= 2 ? sqrt(st.m2 / (double)st.n) : 0.0;
  return 0;
}

// The formant ratio travels in the f0 map block to stage 1 of the next submitted step, whose epilogue copies it into the step's hand-off
// slot for the stage-2 epilogue.
int ryk_session_set_formant(ryk_engine* h, int id, double ratio) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(isfinite(ratio) && ratio >= 0.5 && ratio <= 2.0, "the formant ratio must be finite and within [0.5, 2]");
  s->f0.block.edit().formant = ratio;
  return 0;
}

int ryk_session_get_formant(ryk_engine* h, int id, double* ratio) {
  Session* s = get_session(&h->impl, id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(ratio != nullptr, "null argument");
  *ratio = s->f0.block.next.formant;
  return 0;
}

// ---- input noise suppression (DESIGN.md §4f) ----
int ryk_session_denoise(ryk_engine* h, int id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = fresh_session(e, id, "noise suppression can only be enabled on a fresh session (no chunk pushed): the wave slides are captured at the first steps");
  if (!s) return -2;
  if (s->dn.on) return 0;
  if (frame_stage_alloc(e, s)) return -1;
  DenoiseWork& w = s->frame.w;
  // the parameter block starts at 20 dB without a profile
  if (host_block_alloc(s->mem, s->dn.block, &w.params, DenoiseParams{pow(10.0, -20.0 / 20.0)}) || s->mem.device(&w.learn, 1)) return -1;
  RYK_CUDA(cudaStreamSynchronize(e->stream));      // the zero-fills: the session's streams do not wait for the engine stream
  s->dn.on = true;
  return 0;
}

int ryk_session_set_denoise(ryk_engine* h, int id, double reduction_db) {
  Session* s = stage_session(&h->impl, id, &Session::dn);
  if (!s) return -2;
  if (int rc = denoise_check(reduction_db, nullptr)) return rc;
  s->dn.block.edit().gain_floor = pow(10.0, -reduction_db / 20.0);
  return 0;
}

int ryk_session_denoise_learn(ryk_engine* h, int id, long long n_frames) {
  Session* s = stage_session(&h->impl, id, &Session::dn);
  if (!s) return -2;
  RYK_CHECK(n_frames >= 1, "n_frames must be at least 1");
  DenoiseParams& P = s->dn.block.edit();
  P.learn_serial++;
  P.learn_frames = n_frames;
  return 0;
}

int ryk_session_set_noise_profile(ryk_engine* h, int id, const double* phi) {
  Session* s = stage_session(&h->impl, id, &Session::dn);
  if (!s) return -2;
  RYK_CHECK(phi != nullptr, "null argument");
  if (int rc = denoise_check(0.0, phi)) return rc;
  DenoiseParams& P = s->dn.block.edit();
  memcpy(P.phi, phi, sizeof(double) * kDnBins);
  P.profile_serial++;
  P.learn_serial++;                                // cancels a learning in progress
  P.learn_frames = 0;
  return 0;
}

int ryk_session_noise_profile(ryk_engine* h, int id, double* phi, long long* frames_left) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = stage_session(e, id, &Session::dn);
  if (!s) return -2;
  DenoiseLearn L;
  if (read_back(e, s->frame.w.learn, s->sE, &L)) return -1;     // behind the wave slides of every submitted step
  // requests not yet applied (not submitted yet: every submitted step's gain scan has run) are what the next step applies
  const DenoiseParams& P = s->dn.block.next;
  const bool new_profile = P.profile_serial != L.profile_serial, new_learn = P.learn_serial != L.learn_serial;
  if (phi) memcpy(phi, new_profile ? P.phi : L.phi, sizeof(double) * kDnBins);
  if (frames_left) *frames_left = new_learn ? P.learn_frames : L.remaining;
  return 0;
}

// ---- echo cancellation (DESIGN.md §4g) ----
int ryk_session_echo_cancel(ryk_engine* h, int id, int taps, int delay_frames) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = fresh_session(e, id, "echo cancellation can only be enabled on a fresh session (no chunk pushed): the wave slides are captured at the first steps");
  if (!s) return -2;
  RYK_CHECK(!s->aec.on, "echo cancellation is already enabled for this session");
  if (int rc = echo_check(taps, delay_frames, 0.0)) return rc;
  if (frame_stage_alloc(e, s)) return -1;
  BufferSet& m = s->mem;
  EchoWork& a = s->aec.w;
  a.taps = taps; a.delay = delay_frames;
  // the filters start at zero; the residual suppression at 0 dB (gain 1)
  if (host_block_alloc(m, s->aec.block, &a.params, EchoParams{1.0}) || m.device(&a.filter, 1) ||
      m.device(&a.ring, (size_t)kDnBins * (taps + delay_frames)) || m.device(&a.far_spec, (size_t)kDnBins * s->frame.w.max_frames))
    return -1;
  for (ParitySet& p : s->par) if (m.device(&p.input[kFar].dn, 1)) return -1;     // zero: in_end 0, an empty history
  if (input_alloc(s, kFar, s->n_in, s->in.rate != 0)) return -1;
  RYK_CUDA(cudaStreamSynchronize(e->stream));      // the zero-fills: the session's streams do not wait for the engine stream
  s->aec.on = true;
  return 0;
}

int ryk_session_echo_reference(ryk_engine* h, int id, const float* far, int n) {
  Session* s = stage_session(&h->impl, id, &Session::aec);
  if (!s) return -2;
  RYK_CHECK(far != nullptr, "null argument");
  RYK_CHECK(n == s->n_in, "the far end of a step must be one chunk at the session's input rate (ryk_session_io_geometry n_in)");
  memcpy(s->aec.far_next.data(), far, sizeof(float) * n);
  s->aec.far_set = true;
  return 0;
}

int ryk_session_set_echo_suppression(ryk_engine* h, int id, double db) {
  Session* s = stage_session(&h->impl, id, &Session::aec);
  if (!s) return -2;
  if (int rc = echo_check(1, 0, db)) return rc;
  s->aec.block.edit().gain_floor = pow(10.0, -db / 20.0);
  return 0;
}

int ryk_session_echo_stats(ryk_engine* h, int id, long long* frames, double* erle_db) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = stage_session(e, id, &Session::aec);
  if (!s) return -2;
  EchoStats f;
  if (read_back(e, &s->aec.w.filter->stats, s->sE, &f)) return -1;     // behind the wave slides of every submitted step
  double sd = 0.0, sz = 0.0;
  for (int k = 0; k < kDnBins; ++k) { sd += f.sum_d[k]; sz += f.sum_z[k]; }
  if (frames) *frames = f.frames;
  if (erle_db) *erle_db = sd > 0.0 ? 10.0 * log10(sd / sz) : 0.0;
  return 0;
}

// ---- output limiter (DESIGN.md §4i) ----
int ryk_session_limiter(ryk_engine* h, int id, double lookahead_ms, double hold_ms) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = fresh_session(e, id, "the output limiter can only be enabled on a fresh session (no chunk pushed): the synthesis graphs are captured at the first steps");
  if (!s) return -2;
  RYK_CHECK(!s->lim.on, "the output limiter is already enabled for this session");
  if (int rc = limiter_check_shape(lookahead_ms, hold_ms)) return rc;
  s->lim.lookahead_ms = lookahead_ms;
  s->lim.hold_ms = hold_ms;
  // the ceiling starts at -1 dB of the samples as returned (gain 1)
  s->lim.ceiling_db = -1.0;
  if (limiter_alloc(s, limiter_params(-1.0, 1.0))) return -1;
  RYK_CUDA(cudaStreamSynchronize(e->stream));      // the zero-fills: the session's streams do not wait for the engine stream
  s->lim.on = true;
  return 0;
}

int ryk_session_set_limiter(ryk_engine* h, int id, double ceiling_db, double gain) {
  Session* s = stage_session(&h->impl, id, &Session::lim);
  if (!s) return -2;
  if (int rc = limiter_check_settings(ceiling_db, gain)) return rc;
  s->lim.ceiling_db = ceiling_db;
  s->lim.block.edit() = limiter_params(ceiling_db, gain);
  return 0;
}

int ryk_session_get_limiter(ryk_engine* h, int id, double* ceiling_db, double* gain, int* lookahead, int* hold) {
  Session* s = stage_session(&h->impl, id, &Session::lim);
  if (!s) return -2;
  if (ceiling_db) *ceiling_db = s->lim.ceiling_db;
  if (gain) *gain = s->lim.block.next.gain;
  if (lookahead) *lookahead = s->lim.w.L;
  if (hold) *hold = s->lim.w.R;
  return 0;
}

int ryk_session_limiter_stats(ryk_engine* h, int id, double* reduction_db, long long* limited) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = stage_session(e, id, &Session::lim);
  if (!s) return -2;
  LimMeter mt;
  if (read_back(e, s->lim.w.meter, s->sD, &mt)) return -1;       // behind the synthesis of every submitted step
  double g = 1.0;
  memcpy(&g, &mt.min_bits, sizeof(double));
  if (reduction_db) *reduction_db = mt.limited ? -20.0 * log10(g) : 0.0;
  if (limited) *limited = (long long)mt.limited;
  return 0;
}

// ---- automatic gain control (DESIGN.md §4j) ----
// The AGC runs on the model-rate chunk, whose length n_wave no device rate changes: nothing here depends on ryk_session_set_input_rate.
int ryk_session_agc(ryk_engine* h, int id, double target_db, double max_gain_db, double gate_db) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = fresh_session(e, id, "the automatic gain control can only be enabled on a fresh session (no chunk pushed): the wave slides are captured at the first steps");
  if (!s) return -2;
  RYK_CHECK(!s->agc.on, "the automatic gain control is already enabled for this session");
  if (int rc = agc_check(target_db, max_gain_db, gate_db)) return rc;
  BufferSet& m = s->mem;
  AgcWork& w = s->agc.w;
  if (host_block_alloc(m, s->agc.block, &w.params, AgcParams{}) || m.device(&w.meter, 1) ||
      m.device(&s->agc.d_chunk, s->n_wave))
    return -1;
  for (ParitySet& p : s->par) if (m.device(&p.agc, 1)) return -1;
  // step 0 reads par[0]: position 0, gains 1, no level yet
  AgcState st;
  AgcMeter mt;
  agc_state_init(&st);
  agc_meter_init(&mt);
  if (upload_wait(e, s->par[0].agc, &st) || upload_wait(e, w.meter, &mt)) return -1;
  agc_set_next(s, target_db, max_gain_db, gate_db);      // the first settings
  s->agc.on = true;
  return 0;
}

int ryk_session_set_agc(ryk_engine* h, int id, double target_db, double max_gain_db, double gate_db) {
  Session* s = stage_session(&h->impl, id, &Session::agc);
  if (!s) return -2;
  if (int rc = agc_check(target_db, max_gain_db, gate_db)) return rc;
  agc_set_next(s, target_db, max_gain_db, gate_db);
  return 0;
}

int ryk_session_get_agc(ryk_engine* h, int id, double* target_db, double* max_gain_db, double* gate_db, double* linear) {
  Session* s = stage_session(&h->impl, id, &Session::agc);
  if (!s) return -2;
  if (target_db) *target_db = s->agc.db[0];
  if (max_gain_db) *max_gain_db = s->agc.db[1];
  if (gate_db) *gate_db = s->agc.db[2];
  if (linear) {
    const AgcParams& P = s->agc.block.next;
    const double v[7] = {P.target, P.gate, P.gmax, P.ginv, P.a, P.s_up, P.s_dn};
    memcpy(linear, v, sizeof(v));
  }
  return 0;
}

int ryk_session_agc_stats(ryk_engine* h, int id, double* level_db, double* gain_db, int* active) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = stage_session(e, id, &Session::agc);
  if (!s) return -2;
  AgcMeter mt;
  if (read_back(e, s->agc.w.meter, s->sE, &mt)) return -1;       // behind the wave slides of every submitted step
  if (level_db) *level_db = mt.started ? 10.0 * log10(mt.level) : -HUGE_VAL;
  if (gain_db) *gain_db = 20.0 * log10(mt.gain);
  if (active) *active = mt.active;
  return 0;
}

// ---- pitch correction (DESIGN.md §4m) ----
int ryk_session_pitch_correct(ryk_engine* h, int id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = fresh_session(e, id, "pitch correction can only be enabled on a fresh session (no chunk pushed): the decode slides are captured at the first steps");
  if (!s) return -2;
  RYK_CHECK(!s->pitch.on, "pitch correction is already enabled for this session");
  PitchWork& w = s->pitch.w;
  // amount 0 changes nothing until the caller sets the correction
  const PitchParams first = pitch_params(s->cfg.frame_period_ms, 0, 0xfff, 440.0, 50.0, 0.0);
  if (host_block_alloc(s->mem, s->pitch.block, &w.params, first) || s->mem.device(&w.state, 1)) return -1;
  PitchState st;
  pitch_state_init(&st);
  if (upload_wait(e, w.state, &st)) return -1;
  s->pitch.on = true;
  return 0;
}

int ryk_session_set_pitch_correct(ryk_engine* h, int id, int key, int scale_mask, double a4_hz, double retune_ms, double amount) {
  Session* s = stage_session(&h->impl, id, &Session::pitch);
  if (!s) return -2;
  if (int rc = pitch_check(key, scale_mask, a4_hz, retune_ms, amount)) return rc;
  s->pitch.block.edit() = pitch_params(s->cfg.frame_period_ms, key, scale_mask, a4_hz, retune_ms, amount);
  return 0;
}

int ryk_session_get_pitch_correct(ryk_engine* h, int id, int* key, int* scale_mask, double* a4_hz, double* retune_ms, double* amount) {
  Session* s = stage_session(&h->impl, id, &Session::pitch);
  if (!s) return -2;
  const PitchParams& P = s->pitch.block.next;
  if (key) *key = P.key;
  if (scale_mask) *scale_mask = P.scale;
  if (a4_hz) *a4_hz = P.a4;
  if (retune_ms) *retune_ms = P.retune_ms;
  if (amount) *amount = P.amount;
  return 0;
}

int ryk_session_pitch_stats(ryk_engine* h, int id, long long* voiced, double* mean_cents, double* max_cents) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = stage_session(e, id, &Session::pitch);
  if (!s) return -2;
  PitchState st;
  if (read_back(e, s->pitch.w.state, s->sD, &st)) return -1;      // behind the decode slides of every submitted step
  if (voiced) *voiced = st.voiced;
  if (mean_cents) *mean_cents = st.voiced ? st.sum_cents / (double)st.voiced : 0.0;
  if (max_cents) *max_cents = st.max_cents;
  return 0;
}

}  // extern "C"
