// session_snapshot.cu -- moving a session: its snapshot and restore (DESIGN.md §4k).
#include <string.h>
#include <chrono>
#include <string>
#include <vector>

#include "../../include/ryk.h"
#include "session.h"
#include "snapshot.h"

namespace ryk {

// The host side of the stream state: every host block's next value and dirty flag, the f0 reset and far-end flags, the limiter's and
// AGC's dB settings and the synthesizer's host counters.
struct SnapHost {
  long long step;
  F0Map f0_next; DenoiseParams dn_next; EchoParams aec_next; LimParams lim_next; AgcParams agc_next;
  double lim_ceiling_db, agc_db[3];
  long long host_cum_frames, host_noise_generated;
  int f0_dirty, dn_dirty, aec_dirty, lim_dirty, agc_dirty, f0_reset, far_set, host_noise_slot;
};
static_assert(sizeof(SnapHost) == 2320, "snapshot layout: bump kSnapVersion (snapshot.h)");

// The one list of SnapHost's fields: copies s's host state into h when `save`, else h's into s.
static void snap_host(Session* s, SnapHost& h, bool save) {
  auto x = [save](auto& field, auto& value) { if (save) value = field; else field = value; };
  x(s->step, h.step);
  x(s->f0.block.next, h.f0_next); x(s->f0.block.dirty, h.f0_dirty); x(s->f0.reset, h.f0_reset);
  x(s->dn.block.next, h.dn_next); x(s->dn.block.dirty, h.dn_dirty);
  x(s->aec.block.next, h.aec_next); x(s->aec.block.dirty, h.aec_dirty); x(s->aec.far_set, h.far_set);
  x(s->lim.block.next, h.lim_next); x(s->lim.block.dirty, h.lim_dirty); x(s->lim.ceiling_db, h.lim_ceiling_db);
  x(s->agc.block.next, h.agc_next); x(s->agc.block.dirty, h.agc_dirty);
  for (int i = 0; i < 3; ++i) x(s->agc.db[i], h.agc_db[i]);
  x(s->synth->host_cum_frames, h.host_cum_frames); x(s->synth->host_noise_generated, h.host_noise_generated);
  x(s->synth->host_noise_slot, h.host_noise_slot);
}

// The host side of the pitch correction, in a section of its own that only a session with the correction writes (PTCH), so that
// SnapHost and the blobs of every other session stay as they were.
struct SnapPitch {
  PitchParams next;
  long long dirty;
};
static_assert(sizeof(SnapPitch) == 56, "snapshot layout: bump kSnapVersion (snapshot.h)");

// One section's payload: its tag, where it lies and its size.
struct SnapRegion { uint32_t tag; void* p; size_t bytes; };

// The device regions that carry stream state, in blob order: both parities of every double-buffered one.  Everything else a session
// owns is scratch, derived or configuration, and goes in no section (DESIGN.md §4k).
static std::vector<SnapRegion> session_regions(const Session* s) {
  std::vector<SnapRegion> r;
  auto add = [&](const char (&t)[5], const void* p, size_t bytes) { r.push_back({snap_tag(t), (void*)p, bytes}); };
  const size_t Lw = s->Lw, Tw = s->Tw, Td = s->Td, nb = s->nb, C = s->C, hop = s->hop;
  for (const ParitySet& p : s->par) {
    add("WAVE", p.wave_win, sizeof(float) * Lw);
    add("CWF0", p.cw_f0, sizeof(float) * Tw);
    add("CWAP", p.cw_ap, sizeof(float) * Tw * nb);
    add("CWMC", p.cw_mc, sizeof(float) * Tw * C);
    add("CWVO", p.cw_voiced, Tw);
    add("CWWV", p.cw_wave, sizeof(float) * Tw * hop);
    add("DWF0", p.dw_f0, sizeof(float) * Td);
    add("DWAP", p.dw_ap, sizeof(float) * Td * nb);
    add("DWSP", p.dw_sp, sizeof(float) * Td * nb);
    for (int i = 0; i < kInputs; ++i) {
      const InputState& x = p.input[i];
      if (x.win) {
        add(i == kMic ? "MWIN" : "FWIN", x.win, sizeof(float) * s->in.hist);
        add(i == kMic ? "MRES" : "FRES", x.rs, sizeof(ResampleState));
      }
      if (x.dn) add(i == kMic ? "MFRM" : "FFRM", x.dn, sizeof(DenoiseState));
    }
    if (p.out_hist) {
      add("OHIS", p.out_hist, sizeof(double) * s->out.hist);
      add("ORES", p.out_st, sizeof(ResampleState));
    }
    if (s->lim.on) {
      add("LG0H", p.lim.g0, sizeof(double) * (s->lim.w.R + 2 * s->lim.w.L - 1));
      add("LYH ", p.lim.y, sizeof(double) * s->lim.w.L);
      add("LPOS", p.lim.st, sizeof(LimState));
    }
    if (s->agc.on) add("AGCS", p.agc, sizeof(AgcState));
  }
  add("F0MP", s->f0.d_map, sizeof(F0Map));
  add("F0ST", s->f0.d_stats, sizeof(F0Stats));
  if (s->dn.on) {
    add("DNPA", s->frame.w.params, sizeof(DenoiseParams));
    add("DNLE", s->frame.w.learn, sizeof(DenoiseLearn));
  }
  if (s->aec.on) {
    const EchoWork& a = s->aec.w;
    add("AECP", a.params, sizeof(EchoParams));
    add("AECF", a.filter, sizeof(EchoFilter));
    add("AECR", a.ring, sizeof(double2) * kDnBins * (a.taps + a.delay));
  }
  if (s->lim.on) {
    add("LIMP", s->lim.w.params, sizeof(LimParams));
    add("LIMM", s->lim.w.meter, sizeof(LimMeter));
  }
  if (s->agc.on) {
    add("AGCP", s->agc.w.params, sizeof(AgcParams));
    add("AGCM", s->agc.w.meter, sizeof(AgcMeter));
  }
  if (s->pitch.on) {
    add("PTCP", s->pitch.w.params, sizeof(PitchParams));
    add("PTCS", s->pitch.w.state, sizeof(PitchState));
  }
  const SynthDev& D = s->synth->dev;
  const size_t sb = D.fft_size / 2 + 1;
  add("SYST", D.state, sizeof(SynthState));
  add("SYF0", D.f0, sizeof(double) * D.cap_frames);
  add("SYSP", D.sp, sizeof(float) * D.cap_frames * sb);
  add("SYAP", D.ap, sizeof(float) * D.cap_frames * sb);
  add("SYPI", D.p_index, sizeof(long long) * D.cap_pulses);
  add("SYPT", D.p_time, sizeof(double) * D.cap_pulses);
  add("SYPV", D.p_vuv, sizeof(int) * D.cap_pulses);
  add("SYNZ", D.noise, sizeof(uint32_t) * D.cap_noise);
  add("SYC0", D.carry[0], sizeof(double) * D.carry_len);
  add("SYC1", D.carry[1], sizeof(double) * D.carry_len);
  return r;
}

static void unet_channels(const UNet* n, int* c) { c[0] = n->in_ch; c[1] = n->out_ch; c[2] = n->base; }

// What a session's blob records, in order: CONF (ryk_snapshot_session), TAPI / TAPO (the device rates' taps, when set), HOST (SnapHost),
// FARN (the far end of the next step, with echo cancellation), PTCH (SnapPitch, with pitch correction), all in host memory, then the
// device regions of session_regions.
struct SessionBlob {
  ryk_snapshot_session conf;
  std::vector<double> taps_in, taps_out;
  SnapHost host;
  SnapPitch pitch;
  std::vector<SnapRegion> head, regions;
  std::vector<size_t> payloads() const {
    std::vector<size_t> p;
    for (const auto* list : {&head, &regions}) for (const SnapRegion& x : *list) p.push_back(x.bytes);
    return p;
  }
};

// The blob of session id when a snapshot may be taken, else the refusal (the taps are read from the device: this waits for the session's
// streams).
static int session_blob(Engine* e, int id, Session** out, SessionBlob* b) {
  Session* s = get_session(e, id);
  if (!s) { set_error("no such session"); return -2; }
  if (!session_idle(s)) { set_error("the session has steps in flight: collect every submitted chunk before a snapshot"); return -2; }
  if (s->group && s->group->collected != s->group->step) {
    set_error("the session's group has steps in flight: collect every submitted group chunk before a snapshot");
    return -2;
  }
  for (cudaStream_t st : s->streams()) RYK_CUDA(cudaStreamSynchronize(st));
  ryk_snapshot_session& c = b->conf;
  memset(&c, 0, sizeof(c));
  c.cfg = s->cfg;
  c.voice_id = s->voice_id;
  c.precision = s->precision; c.stage1_fused = s->s1_fused; c.f0_method = s->par[0].crepe ? 2 : dio_plan_harvest(s->par[0].dio) ? 1 : 0;
  unet_channels(s->voice->stage1, c.stage1_channels);
  unet_channels(s->voice->stage2, c.stage2_channels);
  c.in_rate = s->in.rate; c.in_up = s->in.up; c.in_down = s->in.down; c.in_taps = s->in.n_taps;
  c.out_rate = s->out.rate; c.out_up = s->out.up; c.out_down = s->out.down; c.out_taps = s->out.n_taps;
  c.denoise = s->dn.on; c.echo = s->aec.on; c.echo_taps = s->aec.w.taps; c.echo_delay_frames = s->aec.w.delay;
  c.limiter = s->lim.on; c.agc = s->agc.on; c.f0_measure = s->f0.on;
  c.limiter_lookahead_ms = s->lim.lookahead_ms; c.limiter_hold_ms = s->lim.hold_ms;
  c.step = s->step;
  b->taps_in.assign(c.in_taps, 0.0);
  b->taps_out.assign(c.out_taps, 0.0);
  if (c.in_rate) RYK_CUDA(cudaMemcpy(b->taps_in.data(), s->in.d_h, sizeof(double) * c.in_taps, cudaMemcpyDeviceToHost));
  if (c.out_rate) RYK_CUDA(cudaMemcpy(b->taps_out.data(), s->out.d_h, sizeof(double) * c.out_taps, cudaMemcpyDeviceToHost));
  memset(&b->host, 0, sizeof(b->host));
  snap_host(s, b->host, true);
  b->head = {{snap_tag("CONF"), &c, sizeof(c)}};
  if (c.in_rate) b->head.push_back({snap_tag("TAPI"), b->taps_in.data(), sizeof(double) * c.in_taps});
  if (c.out_rate) b->head.push_back({snap_tag("TAPO"), b->taps_out.data(), sizeof(double) * c.out_taps});
  b->head.push_back({snap_tag("HOST"), &b->host, sizeof(b->host)});
  if (c.echo) b->head.push_back({snap_tag("FARN"), s->aec.far_next.data(), sizeof(float) * s->n_in});
  if (s->pitch.on) {
    memset(&b->pitch, 0, sizeof(b->pitch));
    b->pitch.next = s->pitch.block.next;
    b->pitch.dirty = s->pitch.block.dirty;
    b->head.push_back({snap_tag("PTCH"), &b->pitch, sizeof(b->pitch)});
  }
  b->regions = session_regions(s);
  *out = s;
  return 0;
}

using Clock = std::chrono::steady_clock;
static double ms_since(Clock::time_point t) { return std::chrono::duration<double, std::milli>(Clock::now() - t).count(); }

// The sections of a session blob in front of its device regions, as restore_check found them.
struct BlobSections {
  const SnapSection *taps_in = nullptr, *taps_out = nullptr, *host = nullptr, *far = nullptr;
  const SnapSection* pitch = nullptr;    // present when the session had pitch correction
  size_t regions = 0;              // index of the first device region
};

// The checks of a session blob that need no allocation: its configuration and sections, against engine e and voice voice_id.
static int restore_check(Engine* e, int voice_id, const void* buf, size_t bytes, ryk_snapshot_session* c, std::vector<SnapSection>* sec,
                         BlobSections* w) {
  uint32_t kind = 0, version = 0;
  if (const char* refusal = snap_parse(buf, bytes, &kind, &version, sec)) { set_error(refusal); return -2; }
  RYK_CHECK(kind == kSnapSession, "not a session snapshot");
  RYK_CHECK(!sec->empty() && (*sec)[0].tag == snap_tag("CONF") && (*sec)[0].bytes == sizeof(*c), "malformed session snapshot: no configuration");
  memcpy(c, (*sec)[0].data, sizeof(*c));
  RYK_CHECK(c->precision == e->precision && c->stage1_fused == (int)e->s1_fused,
            "the engine's precision or stage-1 mode differ from those the snapshot records: a session keeps the numerics it was created with");
  Voice* v = engine_voice(e, voice_id);
  RYK_CHECK(v != nullptr, "no such voice");
  RYK_CHECK(v->stage1 && v->stage2, "load both models before restoring a session");
  int c1[3], c2[3];
  unet_channels(v->stage1, c1);
  unet_channels(v->stage2, c2);
  RYK_CHECK(memcmp(c1, c->stage1_channels, sizeof(c1)) == 0 && memcmp(c2, c->stage2_channels, sizeof(c2)) == 0,
            "the voice's stage-1 or stage-2 (in, out, base) channels differ from those the snapshot records");
  RYK_CHECK(c->f0_method >= 0 && c->f0_method <= 2, "malformed session snapshot: unknown f0 method");
  if (c->f0_method == 2) {
    const char* refusal = crepe_plan_refusal(c->cfg.fs);
    if (refusal) { set_error(refusal); return -2; }
  }
  // CONF, then TAPI / TAPO as the configuration says, HOST and FARN, and PTCH when present
  size_t i = 1;
  auto next = [&](const char (&t)[5]) { return i < sec->size() && (*sec)[i].tag == snap_tag(t) ? &(*sec)[i++] : nullptr; };
  auto sized = [&](const char (&t)[5], size_t n) { const SnapSection* x = next(t); return x && x->bytes == n ? x : nullptr; };
  RYK_CHECK(!c->in_rate || (w->taps_in = sized("TAPI", sizeof(double) * c->in_taps)), "malformed session snapshot: input resampler taps");
  RYK_CHECK(!c->out_rate || (w->taps_out = sized("TAPO", sizeof(double) * c->out_taps)), "malformed session snapshot: output resampler taps");
  RYK_CHECK((w->host = sized("HOST", sizeof(SnapHost))), "malformed session snapshot: host state");
  RYK_CHECK(!c->echo || (w->far = next("FARN")), "malformed session snapshot: far end");   // its size is checked against the session
  if (i < sec->size() && (*sec)[i].tag == snap_tag("PTCH"))
    RYK_CHECK((w->pitch = sized("PTCH", sizeof(SnapPitch))), "malformed session snapshot: pitch correction");
  w->regions = i;
  return 0;
}

// Enables on session id what the blob records, through the public calls; the settings given here are replaced by the recorded ones.
static int restore_enable(ryk_engine* h, int id, const ryk_snapshot_session& c, const BlobSections& w) {
  if (c.in_rate && ryk_session_set_input_rate(h, id, c.in_rate, c.in_up, c.in_down, (const double*)w.taps_in->data, c.in_taps)) return -1;
  if (c.out_rate && ryk_session_set_output_rate(h, id, c.out_rate, c.out_up, c.out_down, (const double*)w.taps_out->data, c.out_taps)) return -1;
  if (c.denoise && ryk_session_denoise(h, id)) return -1;
  if (c.echo && ryk_session_echo_cancel(h, id, c.echo_taps, c.echo_delay_frames)) return -1;
  if (c.limiter && ryk_session_limiter(h, id, c.limiter_lookahead_ms, c.limiter_hold_ms)) return -1;
  if (c.agc && ryk_session_agc(h, id, -26.0, 20.0, -50.0)) return -1;
  if (c.f0_measure && ryk_session_f0_measure(h, id, 1)) return -1;
  if (w.pitch && ryk_session_pitch_correct(h, id)) return -1;
  return 0;
}

// Copies the blob's state into the new session s: its device regions through the engine's pinned staging, then its host state.
static int restore_state(Engine* e, Session* s, const std::vector<SnapSection>& sec, const BlobSections& w, double* device_ms) {
  RYK_CHECK(!w.far || w.far->bytes == sizeof(float) * s->n_in, "malformed session snapshot: far end");
  const std::vector<SnapRegion> regions = session_regions(s);
  const size_t i = w.regions;
  RYK_CHECK(sec.size() - i == regions.size(), "the snapshot's state sections do not match the session its configuration makes");
  size_t dev_bytes = 0;
  for (size_t r = 0; r < regions.size(); ++r) {
    RYK_CHECK(sec[i + r].tag == regions[r].tag && sec[i + r].bytes == regions[r].bytes,
              "the snapshot's state sections do not match the session its configuration makes");
    dev_bytes += regions[r].bytes;
  }
  void* hp = nullptr;
  if (engine_pinned(e, dev_bytes, &hp)) return -1;
  size_t off = 0;
  for (size_t r = 0; r < regions.size(); ++r) { memcpy((uint8_t*)hp + off, sec[i + r].data, regions[r].bytes); off += regions[r].bytes; }
  // on the engine stream, behind the zero-fills of the new buffers; the session's streams do not wait for it, so wait here
  const Clock::time_point t1 = Clock::now();
  off = 0;
  for (const SnapRegion& x : regions) {
    RYK_CUDA(cudaMemcpyAsync(x.p, (const uint8_t*)hp + off, x.bytes, cudaMemcpyHostToDevice, e->stream));
    off += x.bytes;
  }
  RYK_CUDA(cudaStreamSynchronize(e->stream));
  *device_ms = ms_since(t1);
  SnapHost hs;
  memcpy(&hs, w.host->data, sizeof(hs));
  snap_host(s, hs, false);
  s->collected = s->step;
  if (w.far) memcpy(s->aec.far_next.data(), w.far->data, w.far->bytes);
  if (w.pitch) {
    SnapPitch sp;
    memcpy(&sp, w.pitch->data, sizeof(sp));
    s->pitch.block.next = sp.next;
    s->pitch.block.dirty = sp.dirty != 0;
  }
  return 0;
}

}  // namespace ryk

using namespace ryk;

extern "C" {

int ryk_session_snapshot_size(ryk_engine* h, int id, size_t* bytes) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(bytes != nullptr, "null argument");
  Session* s = nullptr;
  SessionBlob b;
  if (int rc = session_blob(e, id, &s, &b)) return rc;
  *bytes = snap_size(b.payloads());
  return 0;
}

int ryk_session_snapshot(ryk_engine* h, int id, void* buf, size_t bytes) {
  Engine* e = &h->impl;
  const Clock::time_point t0 = Clock::now();
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(buf != nullptr, "null argument");
  Session* s = nullptr;
  SessionBlob b;
  if (int rc = session_blob(e, id, &s, &b)) return rc;
  const size_t total = snap_size(b.payloads());
  RYK_CHECK(bytes == total, "the buffer must be exactly ryk_session_snapshot_size bytes");
  size_t dev_bytes = 0;
  for (const SnapRegion& x : b.regions) dev_bytes += x.bytes;
  void* hp = nullptr;
  if (engine_pinned(e, dev_bytes, &hp)) return -1;
  const Clock::time_point t1 = Clock::now();
  size_t off = 0;
  for (const SnapRegion& x : b.regions) {
    RYK_CUDA(cudaMemcpyAsync((uint8_t*)hp + off, x.p, x.bytes, cudaMemcpyDeviceToHost, s->sE));
    off += x.bytes;
  }
  RYK_CUDA(cudaStreamSynchronize(s->sE));
  const double device_ms = ms_since(t1);
  uint8_t* cur = snap_begin(buf, kSnapSession);
  for (const SnapRegion& x : b.head) memcpy(snap_section(&cur, x.tag, x.bytes), x.p, x.bytes);
  off = 0;
  for (const SnapRegion& x : b.regions) {
    memcpy(snap_section(&cur, x.tag, x.bytes), (const uint8_t*)hp + off, x.bytes);
    off += x.bytes;
  }
  snap_finish(buf, total);
  e->snap_device_ms = device_ms;
  e->snap_host_ms = ms_since(t0) - device_ms;
  return 0;
}

int ryk_session_restore(ryk_engine* h, int voice_id, const void* buf, size_t bytes, int* session_id) {
  Engine* e = &h->impl;
  const Clock::time_point t0 = Clock::now();
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(session_id != nullptr, "null argument");
  ryk_snapshot_session c;
  std::vector<SnapSection> sec;
  BlobSections w;
  if (int rc = restore_check(e, voice_id, buf, bytes, &c, &sec, &w)) return rc;
  int id = -1;
  if (int rc = session_create(e, &c.cfg, voice_id, c.f0_method, &id)) return rc;
  double device_ms = 0.0;
  if (int rc = restore_enable(h, id, c, w) ? -1 : restore_state(e, e->sessions[id], sec, w, &device_ms)) {
    const std::string cause = ryk_last_error();
    ryk_session_destroy(h, id);
    set_error(cause);
    return rc;
  }
  *session_id = id;
  e->snap_device_ms = device_ms;
  e->snap_host_ms = ms_since(t0) - device_ms;
  return 0;
}

int ryk_snapshot_last_times(ryk_engine* h, double* host_ms, double* device_ms) {
  if (host_ms) *host_ms = h->impl.snap_host_ms;
  if (device_ms) *device_ms = h->impl.snap_device_ms;
  return 0;
}

}  // extern "C"
