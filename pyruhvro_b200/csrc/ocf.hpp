// Avro Object Container Files as an input framing (SURVEY.md 8(f) rank 4): header (magic "Obj\x01", a metadata map with
// avro.schema / avro.codec, a 16-byte sync marker) followed by blocks [record count][byte size][datums...][sync].
// Inside a block the datums carry NO lengths, so record boundaries only exist after walking the records: the host walks
// the (few) block headers, the GPU walks every block's records in parallel (ocf_offsets_kernel, one lane per block) to
// produce the i64 offsets the decode kernel wants.  Host-only part: this file (no CUDA).  Not in the reference (its
// inputs are bare datums, README.md:93-94).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace rv {

struct OcfBlock {
    int64_t data_off;   // first datum byte, relative to the file
    int64_t size;       // bytes of datums
    int64_t count;      // records
    int64_t rec_base;   // records in earlier blocks
};

struct OcfIndex {
    std::string schema_json;
    std::string codec;          // "null" (or absent); anything else is rejected
    std::vector<OcfBlock> blocks;
    int64_t n_records = 0;
    int64_t end_off = 0;        // one past the last block's datums
};

// Throws std::runtime_error on a malformed container (bad magic, truncated block, sync mismatch, compressed blocks, a
// block that claims more records than it has bytes).
OcfIndex ocf_index(const uint8_t* file, int64_t len);

}  // namespace rv
