// Per-message and per-row steps of the multi-version Confluent decode (rv_decode_*_versions, DESIGN.md §7): the
// partition of the messages by schema id and the take that interleaves the per-writer batches back into message order.
// The kernels of versions.cu call them one lane per message / output row; the host emulation of the tests
// (tests/emu/versions.cpp) calls the same functions in a loop.
//
// Compiles for: nvcc (device) and g++ (tests/emu host emulation; test infra only).
#pragma once
#include "dev_types.h"

#if defined(__CUDACC__)
#define RV_HD __host__ __device__ __forceinline__
#else
#ifndef RV_HD
#define RV_HD inline
#endif
#endif

namespace rv {

constexpr int kMaxVersions = 256;   // registered writer schemas of one rv_versions handle (the partition's id table)
constexpr uint32_t E_FRAME_ID = 14; // framed message whose schema id / fingerprint is not registered (reported as RV_ERR_FRAME)
constexpr unsigned long long kNoRow = ~0ull;  // row-map entry of a message that failed its header check (permissive
                                              // registries: a null row, rv_versions_permissive)

// A row-map entry: output row -> (writer index, row within that writer's part of the chunk).
RV_HD unsigned long long take_pack(uint32_t writer, uint64_t row) { return (static_cast<unsigned long long>(writer) << 40) | row; }
RV_HD uint32_t take_writer(unsigned long long e) { return uint32_t(e >> 40); }
RV_HD int64_t take_row(unsigned long long e) { return int64_t(e & ((1ull << 40) - 1)); }

// The Confluent header of message [m, m + len): 0x00, then the big-endian u32 schema id, looked up in the sorted
// table ids[0 .. n_ids).  Returns E_OK with *writer set, E_FRAME (short message / wrong magic byte) or E_FRAME_ID.
RV_HD uint32_t vp_header(const uint8_t* m, int64_t len, const uint32_t* ids, int n_ids, int* writer) {
    if (len < 5 || m[0] != 0) return E_FRAME;
    const uint32_t id = (uint32_t(m[1]) << 24) | (uint32_t(m[2]) << 16) | (uint32_t(m[3]) << 8) | uint32_t(m[4]);
    int lo = 0, hi = n_ids;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (ids[mid] < id) lo = mid + 1; else hi = mid;
    }
    if (lo == n_ids || ids[lo] != id) return E_FRAME_ID;
    *writer = lo;
    return E_OK;
}

// The single-object header of message [m, m + len): C3 01, then the little-endian CRC-64-AVRO fingerprint of the
// writer's schema, looked up in the sorted table fps[0 .. n_fps).  Returns like the Confluent vp_header.
RV_HD uint32_t vp_header(const uint8_t* m, int64_t len, const unsigned long long* fps, int n_fps, int* writer) {
    if (len < int64_t(kSingleObjectHeader) || m[0] != 0xC3u || m[1] != 0x01u) return E_FRAME;
    unsigned long long fp = 0;
    for (int b = 0; b < 8; ++b) fp |= static_cast<unsigned long long>(m[2 + b]) << (8 * b);
    int lo = 0, hi = n_fps;
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (fps[mid] < fp) lo = mid + 1; else hi = mid;
    }
    if (lo == n_fps || fps[lo] != fp) return E_FRAME_ID;
    *writer = lo;
    return E_OK;
}

// One output slot of one output chunk: the take writes `dst` from the same slot of every writer's part.
//   role       SlotRole (plan.hpp) of the reader's slot
//   width      bytes per row for the value roles (Values32: 4, Values64: 8, ValuesW: the slot's width, TypeIds: 1)
//   src[w]     writer w's buffer of the paired slot; null for a Validity slot the writer's plan does not have (its rows
//              are all valid) or a writer absent from the chunk
// Offsets (Utf8 / Binary / List / Map) carry what their rows open:
//   dst_data / src_data[w]   the Utf8 / Binary bytes (null for a list / map)
//   child_map                list / map: the row map of the child row space, written by the offsets pass
//   block_base               [blocks] the rows' lengths summed per block of kTakeBlock rows, scanned in place
struct TakeJob {
    uint8_t* dst;
    const uint8_t* const* src;
    int32_t role;
    int32_t width;
    uint8_t* dst_data;
    const uint8_t* const* src_data;
    unsigned long long* child_map;
    long long* block_base;
};

// One (output chunk, row space): `map` holds one entry per row.
struct TakeSpace {
    const unsigned long long* map;
    long long rows;
    int32_t first_job, n_jobs;
};

constexpr int kTakeBlock = 256;

// One offsets slot's block sums, scanned in place into block bases.
struct TakeScan {
    long long* base;  // a TakeJob's block_base
    long long n;      // its blocks
};

// Kernel parameters of the partition.  Tiles of kTakeBlock messages never span two output chunks (tile_of of the
// decode).  W = n_ids writers; group g = chunk * W + writer.
struct VersionsParams {
    const uint8_t* data;
    const int64_t* offsets;
    int64_t n;
    int64_t chunk_rows;
    int32_t k, tiles_per_chunk, n_tiles, n_ids;
    const uint32_t* ids;                 // [W] registered schema ids, ascending
    unsigned long long* err;             // min over (message << 8 | code); ~0 = none
    uint32_t* tile_cnt;                  // [n_tiles][W] messages per writer; scanned into the tile's first rank
    unsigned long long* tile_bytes;      // [n_tiles][W] bytes per writer; scanned into the tile's first byte
    unsigned long long* group_tot;       // [k][W][2] messages and bytes of every group
    uint16_t* msg_w;                     // [n] writer of every message (0xFFFF: failed its header check)
    // scatter
    uint8_t* gdata;                      // the groups' packed messages
    const unsigned long long* gdata_off; // [k][W] where group g's bytes start in gdata (16-byte aligned)
    int64_t* goffs;                      // the groups' offsets
    const unsigned long long* goff_base; // [k][W] where group g's rows + 1 offsets start in goffs
    unsigned long long* map0;            // [n] space-0 row map (take_pack)
    const unsigned long long* fps;       // [W] single-object registries: the writers' fingerprints, ascending (instead of ids)
    // permissive registries only: the tables above have W + 1 columns (n_ids = W + 1), the last being every chunk's
    // bad group (framing errors and unregistered keys: no bytes, no sub-decode, a kNoRow row-map entry)
    unsigned long long* bad;             // [n] (message << 8 | code) of the bad-group messages
    unsigned long long* n_bad;           // their count
    int64_t* inv;                        // [goffs entries] group row -> message (the inverse of the row map)
};

// Validity / Bits: the source row's bit (a missing validity buffer counts as all valid).
RV_HD uint32_t take_bit(const TakeJob& j, uint32_t w, int64_t s) {
    const uint8_t* b = j.src[w];
    if (!b) return 1u;
    return (uint32_t(b[s >> 3]) >> (s & 7)) & 1u;
}

// Fixed-width slots: row r's value is the source row's.
RV_HD void take_value(const TakeJob& j, uint32_t w, int64_t s, int64_t r) {
    const uint8_t* src = j.src[w] + s * j.width;
    uint8_t* dst = j.dst + r * j.width;
    switch (j.width) {
        case 1: *dst = *src; break;
        case 4: *reinterpret_cast<uint32_t*>(dst) = *reinterpret_cast<const uint32_t*>(src); break;
        case 8: *reinterpret_cast<unsigned long long*>(dst) = *reinterpret_cast<const unsigned long long*>(src); break;
        default:
            if ((j.width & 7) == 0)
                for (int i = 0; i < j.width; i += 8)
                    *reinterpret_cast<unsigned long long*>(dst + i) = *reinterpret_cast<const unsigned long long*>(src + i);
            else
                for (int i = 0; i < j.width; ++i) dst[i] = src[i];
    }
}

// Offsets: the source row's item count / byte length, and where it starts in the writer's child space / data.
RV_HD int32_t take_len(const TakeJob& j, uint32_t w, int64_t s) {
    const int32_t* o = reinterpret_cast<const int32_t*>(j.src[w]);
    return o[s + 1] - o[s];
}
RV_HD int32_t take_start(const TakeJob& j, uint32_t w, int64_t s) { return reinterpret_cast<const int32_t*>(j.src[w])[s]; }

// Row r of an offsets slot once its start `pos` in the output is known: the end offset, and either the child rows'
// map entries or (take_copy) the bytes.
RV_HD void take_offsets_row(const TakeJob& j, uint32_t w, int64_t s, int64_t r, int32_t pos, int32_t len) {
    int32_t* o = reinterpret_cast<int32_t*>(j.dst);
    o[r + 1] = pos + len;
    if (r == 0) o[0] = 0;
    if (j.child_map) {
        const int64_t first = take_start(j, w, s);
        for (int32_t q = 0; q < len; ++q) j.child_map[pos + q] = take_pack(w, uint64_t(first + q));
    }
}

// A null row of a permissive registry (row-map entry kNoRow): what a permissive decode writes for a bad record.  Bits
// and validity are 0 (take_rows_kernel), fixed-width values and N-variant union type ids 0, offsets open no items or
// bytes and start no rows in any child row space.
RV_HD void take_null_value(const TakeJob& j, int64_t r) {
    uint8_t* dst = j.dst + r * j.width;
    for (int i = 0; i < j.width; ++i) dst[i] = 0;
}
RV_HD void take_null_offsets_row(const TakeJob& j, int64_t r, int32_t pos) {
    int32_t* o = reinterpret_cast<int32_t*>(j.dst);
    o[r + 1] = pos;
    if (r == 0) o[0] = 0;
}

// Per-lane copy of one row's bytes: 8-byte words where source and destination agree mod 8, else bytes.
RV_HD void take_copy(uint8_t* dst, const uint8_t* src, int32_t len) {
    int32_t i = 0;
    if (((reinterpret_cast<uintptr_t>(dst) ^ reinterpret_cast<uintptr_t>(src)) & 7) == 0) {
        for (; i < len && (reinterpret_cast<uintptr_t>(dst + i) & 7); ++i) dst[i] = src[i];
        for (; i + 8 <= len; i += 8)
            *reinterpret_cast<unsigned long long*>(dst + i) = *reinterpret_cast<const unsigned long long*>(src + i);
    }
    for (; i < len; ++i) dst[i] = src[i];
}

}  // namespace rv
