// snapshot.h -- the self-describing container of session and re-blocker snapshots (snapshot.cu; DESIGN.md §4k).
//
// A blob is a 32-byte header followed by tagged sections:
//   header   {magic "RYKSNAP\0", format version, kind, total bytes, FNV-1a-64 of bytes [32, total)}
//   section  {tag (four characters), 0, payload bytes} then the payload, zero-padded to a multiple of 8 bytes
// Every field is little-endian.  Payloads hold values only, never device or host pointers.
#pragma once
#include <stddef.h>
#include <stdint.h>

#include <vector>

#include "../../include/ryk.h"
#include "agc.h"
#include "echo.h"
#include "features.h"
#include "limiter.h"
#include "pitch.h"
#include "synth.h"

namespace ryk {

constexpr uint64_t kSnapMagic = 0x0050414e534b5952ull;     // "RYKSNAP\0"
constexpr uint32_t kSnapVersion = 1;
// The payloads are these structs as they lie in memory (and SnapHost in session_snapshot.cu, ReblockState in reblock.cu, DriftSnap in drift.cu).  A change to any of them
// changes what a blob means: bump kSnapVersion with it, so that an older blob is refused before anything is allocated, and the sizes here.
static_assert(sizeof(ryk_snapshot_session) == 224 && sizeof(ryk_snapshot_reblock) == 32, "snapshot layout: bump kSnapVersion");
static_assert(sizeof(F0Map) == 64 && sizeof(F0Stats) == 24 && sizeof(ResampleState) == 16, "snapshot layout: bump kSnapVersion");
static_assert(sizeof(DenoiseParams) == 2088 && sizeof(DenoiseLearn) == 4144 && sizeof(DenoiseState) == 10256, "snapshot layout: bump kSnapVersion");
static_assert(sizeof(EchoParams) == 8 && sizeof(EchoFilter) == 541776, "snapshot layout: bump kSnapVersion");
static_assert(sizeof(LimParams) == 16 && sizeof(LimState) == 8 && sizeof(LimMeter) == 16, "snapshot layout: bump kSnapVersion");
static_assert(sizeof(AgcParams) == 56 && sizeof(AgcState) == 1064 && sizeof(AgcMeter) == 24, "snapshot layout: bump kSnapVersion");
static_assert(sizeof(PitchParams) == 48 && sizeof(PitchState) == 40, "snapshot layout: bump kSnapVersion");
static_assert(sizeof(SynthState) == 136, "snapshot layout: bump kSnapVersion");
enum : uint32_t { kSnapSession = 1, kSnapReblock = 2, kSnapPipeline = 3, kSnapDrift = 4 };   // kinds (a pipeline blob is written by worker.py)

struct SnapHeader { uint64_t magic; uint32_t version, kind; uint64_t total, checksum; };
struct SnapSectionHeader { uint32_t tag, zero; uint64_t bytes; };
static_assert(sizeof(SnapHeader) == 32 && sizeof(SnapSectionHeader) == 16, "blob layout");

constexpr uint32_t snap_tag(const char (&t)[5]) {
  return (uint32_t)(uint8_t)t[0] | (uint32_t)(uint8_t)t[1] << 8 | (uint32_t)(uint8_t)t[2] << 16 | (uint32_t)(uint8_t)t[3] << 24;
}
inline size_t snap_padded(size_t bytes) { return (bytes + 7) & ~(size_t)7; }

uint64_t fnv1a64(const void* p, size_t n);

// One section of a parsed blob
struct SnapSection { uint32_t tag; size_t bytes; const uint8_t* data; };

// Writing: snap_size gives the blob size of sections of these payload sizes; snap_begin writes the header's fixed fields, each
// snap_section its section header and returns where its payload goes, and snap_finish the total and the checksum.
size_t snap_size(const std::vector<size_t>& payloads);
uint8_t* snap_begin(void* buf, uint32_t kind);
uint8_t* snap_section(uint8_t** cursor, uint32_t tag, size_t bytes);
void snap_finish(void* buf, size_t total);

// Reading: verifies the header, the total, the checksum and the section walk.  Returns null and fills kind / version / sections, or
// the refusal (a malformed, truncated or corrupt blob, an unknown format version).
const char* snap_parse(const void* buf, size_t bytes, uint32_t* kind, uint32_t* version, std::vector<SnapSection>* sections);

}  // namespace ryk
