// session_group.cu -- session groups (several sessions of one GPU sharing one batched stage-2 forward per step) and the voice switch.
#include <algorithm>

#include "../../include/ryk.h"
#include "session.h"

using namespace ryk;

extern "C" {

static Group* get_group(Engine* e, int id) { return (id >= 0 && id < (int)e->groups.size()) ? e->groups[id] : nullptr; }

// The conditions on a group's member list (create, add and remove all end in one); nullptr when it may form a group.
static const char* group_refusal(Engine* e, const std::vector<Session*>& members) {
  if (members.empty() || (int)members.size() > kMaxGroupBatch) return "a group holds 1..64 sessions";
  const Session* s0 = members[0];
  for (const Session* s : members)
    if (s->Tw != s0->Tw) return "group members must be distinct sessions with the same window length";
  // one chunk length serves every member in ryk_group_submit / ryk_group_push_device
  for (const Session* s : members)
    if (s->n_in != s0->n_in || s->in.rate != s0->in.rate || s->out.rate != s0->out.rate)
      return "group members must have the same device input and output rates";
  std::vector<const Voice*> voices;
  for (const Session* s : members)
    if (std::find(voices.begin(), voices.end(), s->voice) == voices.end()) voices.push_back(s->voice);
  if (voices.size() > 1 && e->precision != 1) return "a group of several voices needs precision 1 (FP16 tensor cores)";
  if ((int)voices.size() > kMaxGroupVoices) return "a group holds at most 8 distinct voices";
  const UNet* n0 = voices[0]->stage2;
  for (const Voice* v : voices)
    if (v->stage2->in_ch != n0->in_ch || v->stage2->out_ch != n0->out_ch || v->stage2->base != n0->base)
      return "the members' stage-2 models must have the same (in, out, base) channels";
  return nullptr;
}

// The one way a group's batched stage 2 is built: around `members` (slot i = members[i]), for ryk_group_create, _add and _remove.  It
// builds first and releases the old plan after; on failure the group and every session are left as they were (DESIGN.md §4a, "Group
// membership", also for why a member's stream state survives the change).
static int group_rebuild(Engine* e, Group* G, const std::vector<Session*>& members) {
  const char* refusal = group_refusal(e, members);
  if (refusal) { set_error(refusal); return -1; }
  RYK_CUDA(cudaDeviceSynchronize());
  // Members of different voices share the forward: each batch item reads its voice's weights (unet_plan_set_voices).
  std::vector<Voice*> voices;
  std::vector<int> voice_of;
  for (Session* m : members) {
    const auto it = std::find(voices.begin(), voices.end(), m->voice);
    voice_of.push_back((int)(it - voices.begin()));
    if (it == voices.end()) voices.push_back(m->voice);
  }
  std::vector<const UNet*> nets;
  for (const Voice* v : voices) nets.push_back(v->stage2);
  // the batched forward computes the decoder rows of the hull of the members' kept frames (their e_conv may differ); the members
  // share Tw, so their padded tails start at the same row
  std::vector<int> kb, kl;
  for (Session* m : members) { kb.push_back(m->e_conv); kl.push_back(m->n_feat); }
  int keep_begin = 0, keep_len = 0;
  keep_hull((int)members.size(), kb.data(), kl.data(), &keep_begin, &keep_len);
  const int owner = ++e->plan_owners;
  UNetPlan* p2 = nullptr;
  if (unet_get_plan(e, voices[0]->stage2, (int)members.size(), members[0]->Tp, 512, e->precision, &p2, owner, keep_begin, keep_len, false,
                    members[0]->Tw) ||
      unet_plan_set_voices(p2, nets, voice_of)) {
    unet_release_owner(voices[0]->stage2, owner);
    return -1;
  }
  if (G->p2) unet_release_owner(G->voices[0]->stage2, G->owner);
  for (Voice* v : G->voices) v->users--;
  for (Voice* v : voices) v->users++;
  G->voices = voices; G->owner = owner; G->p2 = p2;
  G->fwd_graph.reset();
  for (size_t i = 0; i < members.size(); ++i) {
    Session* m = members[i];
    if (m->group != G) lanes_release(m);
    m->group = G; m->slot = (int)i;
    for (HandoffGraphs& hg : m->hgraphs) { hg.s2_pro.reset(); hg.s2_epi.reset(); }
  }
  G->members = members;
  return 0;
}

int ryk_group_create(ryk_engine* h, const int* session_ids, int n_sessions, int* group_id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  RYK_CHECK(session_ids && group_id && n_sessions >= 1 && n_sessions <= kMaxGroupBatch, "a group holds 1..64 sessions");
  std::vector<Session*> members;
  for (int i = 0; i < n_sessions; ++i) {
    Session* s = get_session(e, session_ids[i]);
    RYK_CHECK(s && !s->group && std::find(members.begin(), members.end(), s) == members.end(),
              "group members must be distinct sessions with the same window length, none of them in a group");
    RYK_CHECK(session_idle(s), "collect every submitted chunk of a session before it joins a group");
    members.push_back(s);
  }
  Group* G = new Group();
  if (group_rebuild(e, G, members)) { delete G; return -1; }
  { int lo = 0, hi = 0; RYK_CUDA(cudaDeviceGetStreamPriorityRange(&lo, &hi)); RYK_CUDA(cudaStreamCreateWithPriority(&G->sG, cudaStreamNonBlocking, lo)); }
  for (int i = 0; i < kRing; ++i) RYK_CUDA(cudaEventCreateWithFlags(&G->ev_fwd[i], cudaEventDisableTiming));
  RYK_CUDA(cudaDeviceSynchronize());
  e->groups.push_back(G);
  *group_id = (int)e->groups.size() - 1;
  return 0;
}

int ryk_group_add(ryk_engine* h, int group_id, int session_id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Group* G = get_group(e, group_id);
  RYK_CHECK(G != nullptr, "no such group");
  Session* s = get_session(e, session_id);
  RYK_CHECK(s != nullptr, "no such session");
  RYK_CHECK(s->group == nullptr, "the session is already in a group");
  RYK_CHECK(G->collected == G->step, "collect every submitted chunk of the group before changing its members");
  RYK_CHECK(session_idle(s), "collect every submitted chunk of a session before it joins a group");
  std::vector<Session*> members = G->members;
  members.push_back(s);
  return group_rebuild(e, G, members);
}

int ryk_group_remove(ryk_engine* h, int group_id, int session_id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Group* G = get_group(e, group_id);
  RYK_CHECK(G != nullptr, "no such group");
  Session* s = get_session(e, session_id);
  RYK_CHECK(s != nullptr && s->group == G, "the session is not a member of this group");
  RYK_CHECK(G->members.size() > 1, "the session is the group's last member: destroy the group instead");
  RYK_CHECK(G->collected == G->step, "collect every submitted chunk of the group before changing its members");
  std::vector<Session*> members = G->members;
  members.erase(members.begin() + s->slot);
  RYK_CUDA(cudaDeviceSynchronize());
  // the session's own stage-2 plans, as session_build makes its stage-1 plans: its next step (alone) allocates nothing
  auto build = [&]() -> int {
    UNetPlan* p = nullptr;
    for (const Stage2Lane& L : s->lane) if (s2_plan(e, s, s->voice, L.owner, &p)) return -1;
    return group_rebuild(e, G, members);
  };
  if (build()) {
    lanes_release(s);
    return -1;
  }
  s->group = nullptr; s->slot = 0;
  for (Stage2Lane& L : s->lane) L.s2_layers.reset();
  for (HandoffGraphs& hg : s->hgraphs) { hg.s2_pro.reset(); hg.s2_epi.reset(); }
  return 0;
}

// ---- voice switch: the session converts into another voice from its next submitted step on (DESIGN.md §4a, "Voice switch") ----
// What depends on the voice is built under fresh owner ids, then swapped in: a failure leaves the session on its old voice.
int ryk_session_set_voice(ryk_engine* h, int id, int voice_id) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Session* s = get_session(e, id);
  RYK_CHECK(s != nullptr, "no such session");
  Voice* v = engine_voice(e, voice_id);
  RYK_CHECK(v != nullptr, "no such voice");
  if (v == s->voice) return 0;
  RYK_CHECK(voice_models_loaded(v), "load every layer of both of the voice's models before switching a session to it");
  RYK_CHECK(v->stage1->in_ch == s->C, "the voice's stage-1 model does not take the session's mel-cepstrum order");
  RYK_CHECK(session_idle(s) && (!s->group || s->group->collected == s->group->step),
            "collect every submitted chunk of the session and of its group before switching its voice");
  RYK_CHECK(e->precision == s->precision && e->s1_fused == s->s1_fused,
            "the engine's precision or stage-1 mode changed since the session was created: a session keeps the numerics it was created with");
  RYK_CHECK(!s->f0.block.next.follow || v->has_f0_stats, "follow mode needs an f0 map: the voice has no f0 statistics (turn follow mode off first)");
  Group* G = s->group;
  Voice* const old = s->voice;
  if (G) {
    s->voice = v;                                  // the member list as the switch would leave it
    const char* refusal = group_refusal(e, G->members);
    s->voice = old;
    if (refusal) { set_error(refusal); return -1; }
  }
  if (voice_id >= 1 && voice_default_stage1_stats(v, s->C)) return -1;
  RYK_CUDA(cudaDeviceSynchronize());
  const int s1_owner = ++e->plan_owners;
  int lane_owner[2];
  for (int& o : lane_owner) o = ++e->plan_owners;
  StageGraph s1[kHandoffGraphs];
  auto build = [&]() -> int {
    UNetPlan* p = nullptr;
    for (int Tp = 128; Tp <= s->Tp; Tp += 128) if (unet_get_plan(e, v->stage1, 1, 1, Tp, e->precision, &p, s1_owner)) return -1;
    if (!G) for (int o : lane_owner) if (s2_plan(e, s, v, o, &p)) return -1;     // a member runs the group's plan
    for (int j = 0; j < kHandoffGraphs; ++j) if (stage1_build_switch(e, s, v, s1_owner, j, s1[j])) return -1;
    if (G) {
      s->voice = v;
      const int rc = group_rebuild(e, G, G->members);     // commits the group's new plan only on success
      s->voice = old;
      if (rc) return rc;
    }
    return 0;
  };
  if (int rc = build()) {
    for (StageGraph& g : s1) g.reset();
    unet_release_owner(v->stage1, s1_owner);
    for (int o : lane_owner) unet_release_owner(v->stage2, o);
    return rc;
  }
  // swap: nothing below fails
  unet_release_owner(old->stage1, s->s1_owner);
  lanes_release(s);                                // the old lane plans and s2_layers (a group member has none)
  old->users--; v->users++;
  s->voice = v; s->voice_id = voice_id; s->s1_owner = s1_owner;
  for (int i = 0; i < 2; ++i) s->lane[i].owner = lane_owner[i];
  for (int j = 0; j < kHandoffGraphs; ++j) {
    HandoffGraphs& hg = s->hgraphs[j];
    std::swap(hg.s1.exec, s1[j].exec); std::swap(hg.s1.launches, s1[j].launches);     // s1[j] drops the old graph
    hg.s2_pro.reset(); hg.s2_epi.reset();
  }
  // the new voice's f0 map, as a session created on it starts; the speaker statistics, follow mode and formant ratio stay
  const F0Map vm = voice_f0_map(v);
  F0Map& f = s->f0.block.edit();
  f.mu_in = vm.mu_in; f.sd_in = vm.sd_in; f.mu_tgt = vm.mu_tgt; f.sd_tgt = vm.sd_tgt;
  f.has_stats = vm.has_stats;
  return 0;
}

int ryk_group_members(ryk_engine* h, int group_id, int* session_ids, int capacity) {
  Engine* e = &h->impl;
  Group* G = get_group(e, group_id);
  RYK_CHECK(G != nullptr, "no such group");
  const int n = (int)G->members.size();
  for (int i = 0; i < n && i < capacity && session_ids; ++i) {
    const auto it = std::find(e->sessions.begin(), e->sessions.end(), G->members[i]);
    session_ids[i] = (int)(it - e->sessions.begin());
  }
  return n;
}

int ryk_group_destroy(ryk_engine* h, int group_id) {
  Engine* e = &h->impl;
  Group* G = get_group(e, group_id);
  RYK_CHECK(G != nullptr, "no such group");
  RYK_CUDA(cudaDeviceSynchronize());
  const int owner = G->owner;
  const std::vector<Voice*> voices = G->voices;
  group_free(G);                     // the member sessions survive (ungrouped) and are destroyed separately
  unet_release_owner(voices[0]->stage2, owner);
  for (Voice* v : voices) v->users--;
  e->groups[group_id] = nullptr;
  return 0;
}

int ryk_group_size(ryk_engine* h, int group_id) {
  Group* G = get_group(&h->impl, group_id);
  return G ? (int)G->members.size() : -1;
}

// Queue one chunk per member (host samples; waves[i] belongs to the member in slot i, see ryk_group_members).
int ryk_group_submit(ryk_engine* h, int group_id, const float* const* waves, int n, long long* ticket) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Group* G = get_group(e, group_id);
  RYK_CHECK(G != nullptr, "no such group");
  if (int rc = check_in_flight(G->step - G->collected)) return rc;
  for (Session* s : G->members) if (int rc = check_chunk(s, n)) return rc;
  const long long k = G->step;
  for (size_t i = 0; i < G->members.size(); ++i)
    if (stage_in(G->members[i], host_slot(G->members[i], k), waves[i])) return -1;
  if (group_enqueue(e, G, nullptr)) return -1;
  for (Session* s : G->members) {
    HostSlot& io = host_slot(s, k);
    if (stage_out(s, io, io.h_out, io.h_n, cudaMemcpyDeviceToHost)) return -1;
  }
  if (ticket) *ticket = k;
  return 0;
}

// Wait for step `ticket` of every member; outs[i] receives member i's samples, n_outs[i] their count.
int ryk_group_collect(ryk_engine* h, int group_id, long long ticket, double* const* outs, int out_capacity, int* n_outs) {
  Engine* e = &h->impl;
  Group* G = get_group(e, group_id);
  RYK_CHECK(G != nullptr, "no such group");
  RYK_CHECK(ticket == G->collected && ticket < G->step, "tickets are collected in submission order");
  for (size_t i = 0; i < G->members.size(); ++i)
    if (collect_out(G->members[i], host_slot(G->members[i], ticket), outs[i], out_capacity, &n_outs[i])) return -1;
  G->collected++;
  return 0;
}

// Device-resident group step, asynchronous (see ryk_session_push_device).
int ryk_group_push_device(ryk_engine* h, int group_id, const float* const* waves_dev, int n, double* const* outs_dev, int out_capacity,
                          int* const* n_outs_dev) {
  Engine* e = &h->impl;
  RYK_CUDA(cudaSetDevice(e->device));
  Group* G = get_group(e, group_id);
  RYK_CHECK(G != nullptr, "no such group");
  RYK_CHECK(waves_dev != nullptr, "null argument");
  for (size_t i = 0; i < G->members.size(); ++i) {
    RYK_CHECK(waves_dev[i] != nullptr, "null argument");
    if (int rc = check_chunk(G->members[i], n)) return rc;
    if (int rc = check_out_capacity(G->members[i], out_capacity)) return rc;
  }
  const long long k = G->step;
  if (group_enqueue(e, G, waves_dev)) return -1;
  for (size_t i = 0; i < G->members.size(); ++i) {
    Session* s = G->members[i];
    if (stage_out(s, host_slot(s, k), outs_dev[i], n_outs_dev[i], cudaMemcpyDeviceToDevice)) return -1;
    s->collected = s->step;
  }
  G->collected = G->step;
  return 0;
}

}  // extern "C"
