// Decode plan: the GPU analogue of the reference's FieldDecoder tree
// (ruhvro/src/fast_decode.rs:73-167, built by make_* at :176-414).
//
// The tree is flattened in pre-order into `DNode`s that every lane of a warp
// steps through in lock step.  Three derived notions drive the kernels:
//
//   row space   space 0 = the records of a chunk; every list/map node opens a new
//               space whose rows are its items.  A node's rows live in one space.
//   stream      a quantity that needs a prefix sum across records: the row count a
//               record contributes to a space (>0), or the bytes a record contributes
//               to one Utf8 column.  Per-record counts are scanned to get each
//               record's first row / first byte in the Arrow buffers.
//   slot        one Arrow buffer of one node (validity / values / offsets / data /
//               type_ids); the kernels address output memory as bufs[slot].
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "dev_types.h"
#include "schema.hpp"

namespace rv {

// ---- host-side description ----------------------------------------------------
enum class SlotRole : uint8_t { Validity, Bits, Values32, Values64, Offsets, Data, TypeIds, ValuesW };  // ValuesW: `width` bytes per row

struct Slot {
    SlotRole role;
    int node;      // owning DNode index
    int space;     // row space whose row count sizes this buffer (Data: unused)
    int stream;    // Data: the byte stream that sizes it
    bool zero_init;  // written with atomicOr (bit buffers in spaces > 0): must start zeroed
    int width = 0;   // ValuesW: bytes per row (FixedSizeBinary(N): N, Decimal128: 16)
};

struct Stream {
    bool is_rows;  // true: rows of `space`; false: bytes of Utf8 node `node`
    int space;
    int node;
};

// One Arrow array of the output tree (what finish() returns, fast_decode.rs:536-567).
struct OutArray {
    AT type;
    int width = 0;     // FixedSizeBinary
    int node;          // DNode that owns the buffers (-1 for a map's synthetic entries struct)
    int space;         // row space giving its length
    bool always_validity;  // nullable record/list/map: bitmap always exported (:629,739,790)
    int slot_v, slot_a, slot_b;
    std::vector<int> children;  // indices into Plan::arrays
};

struct Plan {
    std::vector<DNode> nodes;
    std::vector<Slot> slots;
    std::vector<Stream> streams;
    std::vector<int> space_stream;   // space -> its row stream (space 0: -1)
    std::vector<int> space_depth;    // space -> list nesting depth (space 0: 0)
    std::vector<int32_t> sym_off;    // concatenated per-enum prefix offsets into sym_bytes (n+1 entries per enum)
    std::vector<uint8_t> sym_bytes;
    std::vector<OutArray> arrays;
    std::vector<int> top_arrays;     // one per top-level column
    std::vector<int> validity_slots; // slots with role Validity (null counts are computed for these)
    int n_spaces = 1;
    int max_depth = 0;
};

// Throws std::runtime_error when the schema exceeds a documented limit.
// `keep` (a column projection, select_columns in schema.hpp): the top-level fields that become columns, in output
// order; every other field is still walked as NF_SKIP nodes.  nullptr: every field, in schema order.
Plan build_plan(const AvroNode& top, const std::vector<ArrowField>& fields, const std::vector<int>* keep = nullptr);

// A resolved plan (rv_schema_resolve): the walk follows the writer's schema as `res` (resolve_schemas) pairs it with the
// reader's, and the output tree is the reader's, in the reader's field order at every depth (`fields`: the reader's
// to_arrow_fields).  Writer-only fields become NF_SKIP subtrees, reader-only fields NK_DEFAULT leaves placed after their
// record's writer fields, promotions NK_PROMOTE leaves.  `keep`: the reader's top-level fields that become columns, in
// output order (nullptr: all); the writer fields behind the others are skipped.
Plan build_resolved_plan(const Resolution& res, const std::vector<ArrowField>& fields, const std::vector<int>* keep = nullptr);

}  // namespace rv
