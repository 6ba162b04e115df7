// Host planning of the multi-version Confluent decode (rv_decode_*_versions, DESIGN.md §7 "Several writer schemas"):
// which writer buffer feeds which output buffer, the output batches' sizes from the writers' parts, and the job tables of
// the take (take.cuh).  Shared by the CUDA engine and the tests' host emulation; no CUDA calls.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "plan.hpp"
#include "result.hpp"
#include "take.cuh"

namespace rv {

// A writer's resolved plan next to the reader's plan: both build the reader's Arrow tree (the §7 identity), so every
// OutArray of the reader has one at the same tree position in the writer's plan.
//   slot[s]   the writer's slot of reader slot s; -1 only for a Validity slot the writer never needs (a writer non-union
//             read as a reader ["null", T] is never null)
//   space[p]  the writer's row space of reader row space p
struct VersionPairing {
    std::vector<int> slot;
    std::vector<int> space;
};

// Throws std::runtime_error when the two output trees differ in shape, type or buffers.
VersionPairing pair_plans(const Plan& reader, const Plan& writer);

// Writer w's part of one output chunk: its one-chunk batch (c == nullptr: no message of the chunk has its id) and the
// base address of the arena that batch lives in.
struct VersionPart {
    const ChunkOut* c = nullptr;
    const uint8_t* base = nullptr;
};

// The take permutes rows inside a chunk, so the chunk's row counts, stream totals and null counts are the sums over its
// parts.  tot: the chunk's row of compute_layout's chunk_tot ([max(S, 1)] reader streams).  null_rows: the chunk's bad
// group of a permissive registry, rows of space 0 that add to no stream and are null in every space-0 validity bitmap.
void versions_chunk_totals(const Plan& reader, const std::vector<VersionPairing>& pairs, const std::vector<VersionPart>& parts,
                           unsigned long long* tot);
void versions_null_counts(const Plan& reader, const std::vector<VersionPairing>& pairs, const std::vector<VersionPart>& parts, ChunkOut& out,
                          int64_t null_rows = 0);

// The job tables of one take, laid out for a scratch block at `base` (device memory, or host memory in the emulation):
// [header: spaces, jobs, scans, pointer tables][block sums][child row maps].  `header` is the image of the first
// header_bytes, to be copied to `base`; the rest is written by the take itself.
struct TakePlan {
    std::vector<uint8_t> header;
    size_t header_bytes = 0, total_bytes = 0;
    std::vector<int> level_first;       // [levels + 1] ranges of TakeSpace entries, parents before children
    std::vector<int> scan_first;        // [levels + 1] ranges of TakeScan entries
    std::vector<long long> level_blocks;  // [levels] most blocks of kTakeBlock rows of an entry of the level
    const TakeSpace* spaces = nullptr;  // addresses inside `base`
    const TakeScan* scans = nullptr;
    const TakeJob* jobs = nullptr;
};

// parts: [k][W]; chunks: the output layout (compute_layout over the summed totals); out_base: the output arena;
// map0[j]: the space-0 row map of chunk j (the partition's).
TakePlan plan_take(const Plan& reader, const std::vector<VersionPairing>& pairs, const std::vector<std::vector<VersionPart>>& parts,
                   const std::vector<ChunkOut>& chunks, uint8_t* out_base, const std::vector<const unsigned long long*>& map0, uint8_t* base);

}  // namespace rv
