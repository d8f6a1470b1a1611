// snapshot.cu -- the container of session and re-blocker snapshots (snapshot.h; DESIGN.md §4k) and ryk_snapshot_describe, which
// reads one without an engine or a device.
#include <string.h>

#include "../../include/ryk.h"
#include "common.cuh"
#include "snapshot.h"

namespace ryk {

uint64_t fnv1a64(const void* p, size_t n) {
  const uint8_t* b = (const uint8_t*)p;
  uint64_t h = 0xcbf29ce484222325ull;
  for (size_t i = 0; i < n; ++i) { h ^= b[i]; h *= 0x100000001b3ull; }
  return h;
}

size_t snap_size(const std::vector<size_t>& payloads) {
  size_t total = sizeof(SnapHeader);
  for (size_t b : payloads) total += sizeof(SnapSectionHeader) + snap_padded(b);
  return total;
}

uint8_t* snap_begin(void* buf, uint32_t kind) {
  SnapHeader h = {kSnapMagic, kSnapVersion, kind, 0, 0};
  memcpy(buf, &h, sizeof(h));
  return (uint8_t*)buf + sizeof(h);
}

uint8_t* snap_section(uint8_t** cursor, uint32_t tag, size_t bytes) {
  SnapSectionHeader sh = {tag, 0, (uint64_t)bytes};
  memcpy(*cursor, &sh, sizeof(sh));
  uint8_t* data = *cursor + sizeof(sh);
  memset(data + bytes, 0, snap_padded(bytes) - bytes);
  *cursor = data + snap_padded(bytes);
  return data;
}

void snap_finish(void* buf, size_t total) {
  SnapHeader h;
  memcpy(&h, buf, sizeof(h));
  h.total = total;
  h.checksum = fnv1a64((const uint8_t*)buf + sizeof(h), total - sizeof(h));
  memcpy(buf, &h, sizeof(h));
}

const char* snap_parse(const void* buf, size_t bytes, uint32_t* kind, uint32_t* version, std::vector<SnapSection>* sections) {
  if (!buf || bytes < sizeof(SnapHeader)) return "snapshot blob truncated: shorter than its header";
  SnapHeader h;
  memcpy(&h, buf, sizeof(h));
  if (h.magic != kSnapMagic) return "not a snapshot blob (bad magic)";
  if (h.version != kSnapVersion) return "snapshot blob of an unknown format version";
  if (h.total > bytes) return "snapshot blob truncated: shorter than the size its header records";
  if (h.total < bytes) return "snapshot blob longer than the size its header records";
  const uint8_t* p = (const uint8_t*)buf;
  if (fnv1a64(p + sizeof(h), h.total - sizeof(h)) != h.checksum) return "snapshot blob fails its checksum";
  std::vector<SnapSection> out;
  size_t at = sizeof(h);
  while (at < h.total) {
    SnapSectionHeader sh;
    if (h.total - at < sizeof(sh)) return "malformed snapshot blob: a section header runs past the end";
    memcpy(&sh, p + at, sizeof(sh));
    at += sizeof(sh);
    if (sh.zero != 0 || sh.bytes > h.total - at || snap_padded(sh.bytes) > h.total - at)
      return "malformed snapshot blob: a section runs past the end";
    out.push_back({sh.tag, (size_t)sh.bytes, p + at});
    at += snap_padded(sh.bytes);
  }
  *kind = h.kind;
  *version = h.version;
  if (sections) *sections = out;
  return nullptr;
}

}  // namespace ryk

using namespace ryk;

extern "C" {

int ryk_snapshot_describe(const void* buf, size_t bytes, int* kind, int* version, ryk_snapshot_session* session,
                          ryk_snapshot_reblock* reblock, unsigned* tags, unsigned long long* sizes, int capacity) {
  uint32_t k = 0, v = 0;
  std::vector<SnapSection> sec;
  if (const char* refusal = snap_parse(buf, bytes, &k, &v, &sec)) { set_error(refusal); return -2; }
  RYK_CHECK(!sec.empty(), "malformed snapshot blob: no section");
  if (kind) *kind = (int)k;
  if (version) *version = (int)v;
  // the recorded configuration is the first section of a session or re-blocker blob
  if (k == kSnapSession && session) {
    RYK_CHECK(sec[0].tag == snap_tag("CONF") && sec[0].bytes == sizeof(ryk_snapshot_session), "malformed session snapshot: no configuration");
    memcpy(session, sec[0].data, sizeof(*session));
  }
  if (k == kSnapReblock && reblock) {
    RYK_CHECK(sec[0].tag == snap_tag("RCNF") && sec[0].bytes == sizeof(ryk_snapshot_reblock), "malformed re-blocker snapshot: no configuration");
    memcpy(reblock, sec[0].data, sizeof(*reblock));
  }
  for (int i = 0; i < (int)sec.size() && i < capacity; ++i) {
    if (tags) tags[i] = sec[i].tag;
    if (sizes) sizes[i] = sec[i].bytes;
  }
  return (int)sec.size();
}

int ryk_snapshot_seal(void* buf, size_t bytes) {
  RYK_CHECK(buf != nullptr && bytes >= sizeof(SnapHeader), "snapshot blob shorter than its header");
  snap_finish(buf, bytes);
  return 0;
}

}  // extern "C"
