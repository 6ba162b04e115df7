// Types shared by the host planner, the statically compiled kernels, the NVRTC-compiled
// schema-specialised kernels and the tests-only host emulation.  Must stay free of standard
// library includes when compiled by NVRTC (__CUDACC_RTC__).
#pragma once

#if defined(__CUDACC_RTC__)
typedef signed char int8_t;
typedef unsigned char uint8_t;
typedef short int16_t;
typedef unsigned short uint16_t;
typedef int int32_t;
typedef unsigned int uint32_t;
typedef long long int64_t;
typedef unsigned long long uint64_t;
typedef unsigned long long uintptr_t;
typedef unsigned long size_t;
#else
#include <cstddef>
#include <cstdint>
#endif

namespace rv {

// ---- device-visible node of the generic (interpreted) walker ------------------------------
enum NodeKind : uint8_t {
    NK_I32 = 0,   // int, date            (varint -> i32, `as i32` truncation, fast_decode.rs:424,430)
    NK_I64 = 1,   // long, timestamp-*    (varint -> i64)
    NK_F32 = 2,   // float   (4 raw LE bytes, :871-879)
    NK_F64 = 3,   // double  (8 raw LE bytes, :881-891)
    NK_BOOL = 4,  // boolean (:893-900), LSB-first bit column
    NK_STR = 5,   // string  (:902-922)
    NK_ENUM = 6,  // enum -> Utf8 symbol text (:570-578)
    NK_NULL = 7,  // null (:480)
    NK_REC = 8,   // record (:597-616)
    NK_UNION = 9, // N-variant sparse union (:643-668)
    NK_LIST = 10, // array (:703-727)
    NK_MAP = 11,  // map (:745-770); children = [keys (NK_STR), values]
    // wider subset (SURVEY.md 8(f) rank 3; Arrow types per schema_translate.rs:58,133-143)
    NK_BYTES = 12,     // bytes -> Binary (same wire form and buffers as NK_STR)
    NK_FIXED = 13,     // fixed(N) -> FixedSizeBinary(N): N raw bytes, aux = N
    NK_DEC_BYTES = 14, // decimal on bytes -> Decimal128: varint length + big-endian two's complement
    NK_DEC_FIXED = 15, // decimal on fixed(N) -> Decimal128: N big-endian bytes, aux = N
    NK_UUID = 16,      // uuid (string logical type) -> FixedSizeBinary(16): 36-char hyphenated hex text
    // schema resolution (rv_schema_resolve)
    NK_PROMOTE = 17,   // a writer int / long / float read as a reader long / float / double: aux = writer kind (NK_I32, NK_I64,
                       // NK_F32), aux2 = reader kind (NK_I64, NK_F32, NK_F64)
    NK_DEFAULT = 18    // a reader field the writer does not have: reads nothing, writes its (non-null) default on every row.
                       // pad0 = the column's kind (NK_I32, NK_I64, NK_F32, NK_F64, NK_BOOL; NK_STR for string / bytes / enum
                       // text); aux / aux2 = the low / high 32 bits of the value, or (NK_STR) aux = the first of the two
                       // symbol-table entries that bound its bytes.  (A null default is an NF_ABSENT subtree.)
};

enum NodeFlags : uint8_t {
    NF_NULLABLE = 1,     // wrapped in a 2-variant null union (Nullable* variants, :94-119)
    NF_NULL_FIRST = 2,   // which branch index is null (:404-414)
    NF_VALIDITY = 4,     // a validity bitmap is written for this node
    NF_ZERO_ITEMS = 8,   // list/map whose items occupy zero bytes and own no buffers
    // Part of a top-level field outside a column projection: walked with the skip ops (dev_core.cuh), which read and
    // check what the decoding op's COUNT path does and store nothing.  Such a node has no slots (-1), no stream (-1),
    // opens no row space (space 0) and backs no OutArray; a skipped list/map keeps no row count.
    NF_SKIP = 16,
    // NK_ENUM of a resolved plan whose writer has symbols the reader cannot map: the symbol table holds, after the n + 1
    // offsets, n words that are non-zero for those symbols.  A record that has one fails with E_ENUM_MAP.
    NF_ENUM_MAP = 32,
    // The root of a subtree that is never present: a reader-only field of a nullable type whose default is null (resolved
    // plans).  The walkers treat it like a node whose parent is absent -- the append_null path of every op, reading
    // nothing -- so its buffers are those of a null of the reader's own type: a cleared validity bit, zeroed values, an
    // unchanged offset, type id 0, and the same for every descendant.
    NF_ABSENT = 64
};

struct DNode {
    uint8_t kind;
    uint8_t flags;
    uint8_t level;     // depth in the node tree (root record's children are level 1)
    uint8_t ulevel;    // number of NK_UNION ancestors
    uint8_t variant;   // index within the parent union, 0xFF otherwise
    uint8_t space;     // row space of this node's rows
    uint8_t pad0, pad1;
    int32_t end;       // one past the last node of this subtree (pre-order)
    int16_t slot_v;    // validity bitmap slot (-1: none)
    int16_t slot_a;    // values / offsets / type_ids slot (-1: none)
    int16_t slot_b;    // Utf8 data slot (-1: none)
    int16_t stream;    // NK_STR/NK_ENUM: byte stream; NK_LIST/NK_MAP: child-row stream; else -1
    int32_t aux;       // NK_ENUM: first entry in the symbol-offset table; NK_UNION: variant count
    int32_t aux2;      // NK_ENUM: symbol count
    int32_t pad2;
};
static_assert(sizeof(DNode) == 32, "DNode layout is shared with the kernels");

constexpr int kMaxListDepth = 3;   // row-space nesting the kernels are instantiated for
constexpr int kMaxLevel = 31;      // per-lane presence mask is 32 bits
constexpr int kMaxUnionLevel = 8;  // per-lane union selections packed 8 x 8 bits
constexpr int kMaxStreams = 120;
constexpr int kMaxNodes = 1024;

// Per-record error categories (the bail!/anyhow! sites of fast_decode.rs); values match rv_status.
enum ErrCode : uint32_t {
    E_OK = 0,
    E_EOF = 1,       // "unexpected end of buffer" (:849,874,884,910)
    E_VARINT = 2,    // "zigzag varint too long" (:866)
    E_BOOL = 3,      // "invalid boolean byte" (:898)
    E_NEG_LEN = 4,   // "negative string length" (:906)
    E_BRANCH = 5,    // "invalid union branch index" / "out of range" (:591,646)
    E_ENUM = 6,      // "enum index out of range" (:575)
    E_SCHEMA = 7,
    E_OVERFLOW = 8,  // i32 Arrow offset overflow (arrow-rs panics; reported as an error)
    E_FRAME = 12,    // framed input (SURVEY.md 8(f) rank 4): message shorter than its header / wrong magic byte / wrong schema id
    E_ENUM_MAP = 13, // resolved plans: a writer enum symbol with neither a reader symbol nor a reader default (reported as RV_ERR_ENUM)
    E_VALUE = 11     // wider subset: a value its logical type cannot hold (uuid text that is not a UUID, decimal wider than 128 bits)
};

#ifndef RV_KBLOCK
#define RV_KBLOCK 256
#endif
// Records per tile == threads per CTA (one record per lane).  The static library (interpreter, encoder) is built at
// 256; a generated walker is compiled at its plan's tile (jit.cpp generate_kernel_source): 256, or kWideTile for
// plans of more than kWideStreams streams, where every stream then gets a warp of its own for the scan and look-back.
constexpr int kBlock = RV_KBLOCK;
static_assert(kBlock % 32 == 0 && kBlock >= 64 && kBlock <= 1024, "tiles are whole warps");
constexpr int kWarps = kBlock / 32;
constexpr int kWideTile = 384;
constexpr int kWideStreams = 8;

// Device control block of one decode call, in 64-bit words.
enum CtrlWord : int {
    CW_ERR = 0,         // min over (record << 8 | code); ~0 = none
    CW_MAX_SPAN = 1,    // largest tile input span seen (bytes): sizes the shared-memory window of later calls
    CW_MAX_UTF8 = 2,    // largest staging need of a tile seen (bytes)
    CW_OVER = 3,        // != 0: some tile's output range exceeded the capacity the host planned (p.caps)
    CW_SLOW_TILES = 4,  // tiles that did not fit shared memory and were walked in global memory
    CW_IN_FIRST = 5,    // offsets[0]
    CW_IN_LAST = 6,     // offsets[n]: the input's byte span sizes later calls' windows
    CW_CHUNK_TOT = 8    // [k][n_streams] exact stream totals per chunk
};

// Kernel parameter block of the fused decode pass.
struct DecodeParams {
    // input: packed Avro records (BinaryArray layout, deserialize.rs:90) with i64 offsets
    const uint8_t* data;
    const int64_t* offsets;
    int64_t n;            // records
    int64_t chunk_rows;   // n / k (last chunk takes the remainder, deserialize.rs:57-68)
    int32_t k;            // chunks (= output batches)
    int32_t tiles_per_chunk;
    int32_t n_tiles;
    // plan
    const DNode* nodes;
    int32_t n_nodes;
    int32_t n_streams;
    int32_t n_slots;
    const int32_t* sym_off;
    const uint8_t* sym_bytes;
    const int16_t* stream_slot;  // [n_streams] Utf8 data slot of a byte stream, -1 for a row stream
    // scan
    unsigned long long* tile_state;  // [n_streams][n_tiles] look-back status words {flag:2, value:62}; zero before the launch
    unsigned long long* ctrl;        // control block (CtrlWord)
    const uint32_t* caps;            // [k][n_streams] rows / bytes the planned buffers can take per chunk
    // output
    void* const* bufs;     // [k][n_slots]
    int32_t n_utf8;            // Utf8 byte streams in the plan
    int32_t prefetch_dist;    // CTAs resident on the device: a CTA prefetches (into L2) the tile that far ahead
    uint32_t smem_data_cap;   // bytes of shared memory for staging a tile's input bytes
    uint32_t smem_stage_cap;  // bytes of shared memory for staging a tile's Utf8 output bytes
    int32_t count_only;       // 1: validate + totals only (no buffers yet)
    // framed input: every message starts with `frame_skip` header bytes that are not part of the datum (Confluent wire
    // format: magic 0x00 + big-endian u32 schema id).  frame_check: 0 skip only, 1 check the magic byte, 2 also the id
    uint32_t frame_skip;
    int32_t frame_check;
    uint32_t frame_id;
};

// Object container files: where every record of every block starts (ocf.hpp, ocf_walk.cuh).
struct OcfBlockDev { long long data_off, size, count, rec_base; };
struct OcfParams {
    const uint8_t* data;          // the file's bytes on the device
    const OcfBlockDev* blocks;
    int32_t n_blocks;
    const DNode* nodes;
    int32_t n_nodes;
    int32_t n_streams;            // counters of the walk, zeroed before every record
    const int32_t* sym_off;
    const uint8_t* sym_bytes;
    int64_t* offsets;             // [n_records + 1], relative to `data`
    int64_t n_records;
    long long end_off;
    unsigned long long* err;      // min over (record << 8 | code); ~0 = none
};

// Readers may run a few tokens past a record's end before the deferred end-of-buffer check notices (dev_core.cuh):
// the staged window is followed by this many readable bytes.
constexpr uint32_t kWindowPad = 64;

// Item-position table of the item-parallel list/map emit (generated walkers, jit.cpp).  For each top-level list/map
// whose items are walked (list index L) and each lane, the FAST count walk stores kItemEntries bytes, as offsets from
// where the list starts in the record: the starts of its first kItemSlots items, the position after the terminating
// block, and the item count — kItemSeq when the lane has more than kItemSlots items or the list spans more than 255
// bytes, which makes its warp emit that list with the per-lane loop.  Entry (L, j) of lane t is byte
// (L * kItemEntries + j) * kBlock + t.  (One byte per entry: 1.5 KiB per list at 256 rows keeps the Kafka plan at three
// CTAs per SM.)  `tile`: the tile the table is laid out for (the host sizes a generated kernel's tile, not its own kBlock).
constexpr int kItemSlots = 4;
constexpr int kItemEntries = kItemSlots + 2;
constexpr uint32_t kItemSeq = 0xFFu;
#if defined(__CUDACC__)
__host__ __device__
#endif
constexpr uint32_t item_table_bytes(int n_lists, int tile = kBlock) { return uint32_t(n_lists) * uint32_t(kItemEntries) * uint32_t(tile); }

// Dynamic shared-memory map of a decode CTA (byte offsets inside the CTA's shared memory):
//   [nodes n_nodes*32][ttot (S+1)*4][tbase S*4][adj S*4][flags 16][mbar 8][ptrs n_slots*8][items item_bytes]
//   [cur S*tile*4][in: data_cap+pad][stage: stage_cap]
// alias_cur (walkers that keep their cursors in registers): the scan area `cur` overlays the Utf8 staging area
// (it is dead before the first staged byte is written) and costs no extra shared memory.
struct SmemMap {
    uint32_t nodes, ttot, tbase, adj, flags, mbar, ptrs, items, cur, in, stage, total;
};

#if defined(__CUDACC__)
__host__ __device__
#endif
inline SmemMap smem_map(int n_nodes, int n_streams, int n_slots, uint32_t data_cap, uint32_t stage_cap, bool alias_cur, uint32_t item_bytes,
                        int tile = kBlock) {
    SmemMap m;
    m.nodes = 0;
    m.ttot = uint32_t(n_nodes) * 32u;
    m.tbase = m.ttot + uint32_t(n_streams + 1) * 4u;
    m.adj = m.tbase + uint32_t(n_streams) * 4u;
    m.flags = (m.adj + uint32_t(n_streams) * 4u + 15u) & ~15u;
    m.mbar = m.flags + 16u;  // mbarrier of the bulk-copy staging (8 bytes)
    m.ptrs = m.mbar + 16u;
    m.items = (m.ptrs + uint32_t(n_slots) * 8u + 15u) & ~15u;
    m.cur = (m.items + item_bytes + 15u) & ~15u;
    const uint32_t cur_bytes = uint32_t(n_streams) * uint32_t(tile) * 4u;
    m.in = alias_cur ? m.cur : ((m.cur + cur_bytes + 15u) & ~15u);
    m.stage = (m.in + data_cap + kWindowPad + 15u) & ~15u;
    if (alias_cur) {
        m.cur = m.stage;
        m.total = m.stage + (stage_cap > cur_bytes ? stage_cap : cur_bytes);
    } else {
        m.total = m.stage + stage_cap;
    }
    return m;
}

}  // namespace rv
