// GPU Arrow -> Avro direct encode behind serialize_record_batch (SURVEY.md 8(f) rank 1).
//
// Replaces, for the direct-encode subset:
//   ruhvro/src/serialize.rs:38-67     serialize_record_batch (clamp_chunks, slice_struct, one BinaryArray per chunk)
//   ruhvro/src/fast_encode.rs:27-53   serialize_chunk
//   ruhvro/src/fast_encode.rs:153-381 encoder-tree construction (Arrow columns matched to Avro fields BY NAME)
//   ruhvro/src/fast_encode.rs:397-599 per-row write + wire writers
//
// Shape: the (Avro schema x Arrow array tree) pair is flattened into ENodes whose buffers are uploaded to
// the device; one lane per top-level row walks the nodes in lock step twice — SIZE (bytes this row encodes
// to; CTA-reduced into per-tile totals), a per-chunk scan (offsets restart at 0 in every output chunk),
// then WRITE (datum bytes + the BinaryArray's i32 offsets).  Integer/byte work; HBM-bound in principle.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <array>
#include <chrono>
#include <mutex>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <system_error>
#include <thread>
#include <vector>

#include "../../include/ruhvro_b200.h"
#include "arrow_c.h"
#include "dev_types.h"
#include "result.hpp"
#include "schema.hpp"

namespace rv {

// ------------------------------------------------------------------------------------------------
// device-visible encode node
// ------------------------------------------------------------------------------------------------
struct ENode {
    uint8_t kind;      // NodeKind
    uint8_t flags;     // NF_NULLABLE | NF_NULL_FIRST
    uint8_t level, ulevel, variant, pad0, pad1, pad2;
    int32_t end;       // one past the subtree
    int32_t n_sym;     // enum
    int32_t sym_base;  // enum: first entry in sym_off
    int32_t n_variants;
    const uint8_t* validity;  // may be null: no null buffer => never null
    const uint8_t* buf_a;     // values / offsets / type_ids
    const uint8_t* buf_b;     // Utf8 data
    int64_t row_add;          // logical row -> index into this array's buffers (accumulated slice offsets)
};

struct EncParams {
    const ENode* nodes;
    int32_t n_nodes;
    const int32_t* sym_off;
    const uint8_t* sym_bytes;
    int64_t n;            // rows of this launch (a row group of the batch)
    int64_t row_base;     // first row of the group inside the batch
    int64_t chunk_rows;
    int32_t k, tiles_per_chunk, n_tiles;
    uint32_t* row_size;   // [n]
    uint32_t* tile_agg;   // [n_tiles]
    uint32_t* tile_base;  // [n_tiles]
    unsigned long long* err;
    uint8_t* const* out_data;   // [k]
    int32_t* const* out_offsets;  // [k]
    uint32_t stage_cap;   // bytes of dynamic shared memory in which a tile's datums are assembled
};

namespace {

enum EncErr : uint32_t { EE_ENUM = RV_ERR_ENUM, EE_BRANCH = RV_ERR_BRANCH, EE_OVERFLOW = RV_ERR_OVERFLOW };

struct EncCtx {
    const ENode* nodes;
    const int32_t* sym_off;
    const uint8_t* sym_bytes;
    uint32_t pm;
    uint64_t usel;
    uint32_t err;
    uint32_t size;   // SIZE: bytes so far
    uint8_t* out;    // WRITE: cursor
};

__device__ __forceinline__ bool bit_at(const uint8_t* p, int64_t i) { return (p[i >> 3] >> (i & 7)) & 1; }

// write_zigzag_long, fast_encode.rs:585-593
template <int MODE>
__device__ __forceinline__ void put_long(EncCtx& c, int64_t v) {
    unsigned long long zz = (static_cast<unsigned long long>(v) << 1) ^ static_cast<unsigned long long>(v >> 63);
    if (MODE == 0) {
        c.size += zz ? uint32_t((64 - __clzll(zz) + 6) / 7) : 1u;
    } else {
        while (zz & ~0x7Full) { *c.out++ = uint8_t((zz & 0x7F) | 0x80); zz >>= 7; }
        *c.out++ = uint8_t(zz);
    }
}

// WRITE mode: n bytes from a global Arrow buffer to the lane's output cursor (shared-memory staging or global).
// Destination words are written whole: bytes up to the destination's 4-byte boundary and the tail go bytewise,
// every word in between is one aligned 32-bit load (two when source and destination disagree in alignment,
// the second carried over to the next word) + funnel shift + one 32-bit store — a quarter of the memory
// instructions of a byte loop, which is what the write kernel spends its time on for string columns.
template <int MODE>
__device__ __forceinline__ void put_bytes(EncCtx& c, const uint8_t* src, uint32_t n) {
    if (MODE == 0) { c.size += n; return; }
    uint8_t* dst = c.out;
    uint32_t i = 0;
    while (i < n && (reinterpret_cast<uintptr_t>(dst + i) & 3u)) { dst[i] = src[i]; ++i; }
    if (i + 4 <= n) {
        const uintptr_t sa = reinterpret_cast<uintptr_t>(src + i);
        const uint32_t sh = uint32_t(sa & 3u) * 8u;
        const uint32_t* sw = reinterpret_cast<const uint32_t*>(sa & ~uintptr_t(3));
        uint32_t lo = __ldg(sw);
        if (sh == 0) {
            for (;;) {
                *reinterpret_cast<uint32_t*>(dst + i) = lo;
                i += 4; ++sw;
                if (i + 4 > n) break;
                lo = __ldg(sw);
            }
        } else {
            for (;;) {
                const uint32_t hi = __ldg(sw + 1);  // holds source bytes of this destination word: always in bounds
                *reinterpret_cast<uint32_t*>(dst + i) = __funnelshift_r(lo, hi, sh);
                i += 4; ++sw; lo = hi;
                if (i + 4 > n) break;
            }
        }
    }
    for (; i < n; ++i) dst[i] = src[i];
    c.out += n;
}

template <int MODE, int D>
__device__ __forceinline__ void enc_range(EncCtx& c, int pc, const int end, const int64_t row) {
    while (pc < end) {
        const ENode nd = c.nodes[pc];
        bool present = (c.pm >> (nd.level - 1)) & 1u;
        if (nd.variant != 0xFF) present = present && (uint32_t((c.usel >> (8 * (nd.ulevel - 1))) & 0xFF) == nd.variant);
        bool valid = present;
        const int64_t r = row + nd.row_add;
        if ((nd.flags & NF_NULLABLE) && present) {  // write_nullable, :556-569
            const bool is_null = nd.validity && !bit_at(nd.validity, r);
            const bool nf = (nd.flags & NF_NULL_FIRST) != 0;
            put_long<MODE>(c, is_null ? (nf ? 0 : 1) : (nf ? 1 : 0));
            valid = !is_null;
        }
        switch (nd.kind) {
            case NK_I32: if (valid) put_long<MODE>(c, int64_t(reinterpret_cast<const int32_t*>(nd.buf_a)[r])); break;
            case NK_I64: if (valid) put_long<MODE>(c, reinterpret_cast<const int64_t*>(nd.buf_a)[r]); break;
            case NK_F32: if (valid) put_bytes<MODE>(c, nd.buf_a + 4 * r, 4); break;
            case NK_F64: if (valid) put_bytes<MODE>(c, nd.buf_a + 8 * r, 8); break;
            case NK_BOOL:
                if (valid) { if (MODE == 0) c.size += 1; else *c.out++ = bit_at(nd.buf_a, r) ? 1 : 0; }
                break;
            case NK_STR:
                if (valid) {  // write_string :595-599
                    const int32_t s0 = reinterpret_cast<const int32_t*>(nd.buf_a)[r], s1 = reinterpret_cast<const int32_t*>(nd.buf_a)[r + 1];
                    const uint32_t len = uint32_t(s1 - s0);
                    put_long<MODE>(c, int64_t(len));
                    put_bytes<MODE>(c, nd.buf_b + s0, len);
                }
                break;
            case NK_ENUM:
                if (valid) {  // write_enum_idx :571-579: the Arrow column holds the symbol TEXT
                    const int32_t s0 = reinterpret_cast<const int32_t*>(nd.buf_a)[r], s1 = reinterpret_cast<const int32_t*>(nd.buf_a)[r + 1];
                    const int32_t len = s1 - s0;
                    int found = -1;
                    for (int k = 0; k < nd.n_sym && found < 0; ++k) {
                        const int32_t b0 = c.sym_off[nd.sym_base + k], b1 = c.sym_off[nd.sym_base + k + 1];
                        if (b1 - b0 != len) continue;
                        bool eq = true;
                        for (int32_t q = 0; q < len && eq; ++q) eq = c.sym_bytes[b0 + q] == nd.buf_b[s0 + q];
                        if (eq) found = k;
                    }
                    if (found < 0) { if (!c.err) c.err = EE_ENUM; }
                    else put_long<MODE>(c, found);
                }
                break;
            case NK_NULL: break;
            case NK_REC:
                c.pm = (c.pm & ~(1u << nd.level)) | (uint32_t(valid) << nd.level);
                ++pc;
                continue;
            case NK_UNION: {  // UnionEncoder::write :504-516
                uint32_t sel = 0xFE;
                if (valid) {
                    const int tid = reinterpret_cast<const int8_t*>(nd.buf_a)[r];
                    if (tid < 0 || tid >= nd.n_variants) { if (!c.err) c.err = EE_BRANCH; valid = false; }
                    else { put_long<MODE>(c, tid); sel = uint32_t(tid); }
                }
                c.pm = (c.pm & ~(1u << nd.level)) | (uint32_t(valid) << nd.level);
                c.usel = (c.usel & ~(uint64_t(0xFF) << (8 * nd.ulevel))) | (uint64_t(sel) << (8 * nd.ulevel));
                ++pc;
                continue;
            }
            case NK_LIST:
            case NK_MAP: {  // ListEncoder / MapEncoder :518-554
                if (valid) {
                    const int32_t s0 = reinterpret_cast<const int32_t*>(nd.buf_a)[r], s1 = reinterpret_cast<const int32_t*>(nd.buf_a)[r + 1];
                    if (s1 > s0) {
                        put_long<MODE>(c, int64_t(s1 - s0));
                        c.pm |= (1u << nd.level);
                        if constexpr (D < kMaxListDepth)
                            for (int32_t j = s0; j < s1; ++j) enc_range<MODE, D + 1>(c, pc + 1, nd.end, int64_t(j));
                    }
                    put_long<MODE>(c, 0);
                }
                pc = nd.end;
                continue;
            }
            default: break;
        }
        ++pc;
    }
}

__device__ __forceinline__ void enc_tile(const EncParams& p, int tile, int* chunk, int64_t* r0, int* nrec, int* local) {
    int j = 0;
    if (p.k > 1) { j = tile / p.tiles_per_chunk; if (j > p.k - 1) j = p.k - 1; }
    const int lt = tile - j * p.tiles_per_chunk;
    const int64_t cs = int64_t(j) * p.chunk_rows, ce = (j == p.k - 1) ? p.n : cs + p.chunk_rows;
    *chunk = j; *local = lt; *r0 = cs + int64_t(lt) * kBlock;
    const int64_t left = ce - *r0;
    *nrec = left < kBlock ? int(left) : kBlock;
}

__device__ __forceinline__ void enc_init(EncCtx& c, const EncParams& p) {
    c.nodes = p.nodes; c.sym_off = p.sym_off; c.sym_bytes = p.sym_bytes;
    c.pm = 1u; c.usel = 0; c.err = 0; c.size = 0; c.out = nullptr;
}

__global__ void __launch_bounds__(kBlock) encode_size_kernel(const EncParams p) {
    int chunk, nrec, local; int64_t r0;
    enc_tile(p, blockIdx.x, &chunk, &r0, &nrec, &local);
    const int tid = threadIdx.x;
    EncCtx c;
    enc_init(c, p);
    if (tid < nrec) {
        enc_range<0, 0>(c, 0, p.n_nodes, p.row_base + r0 + tid);
        if (c.err) atomicMin(p.err, (static_cast<unsigned long long>(p.row_base + r0 + tid) << 8) | c.err);
        p.row_size[r0 + tid] = c.size;
    }
    unsigned long long sum = (tid < nrec) ? c.size : 0u;
    for (int d = 16; d; d >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, d);
    __shared__ unsigned long long s_w[kWarps];
    if ((tid & 31) == 0) s_w[tid >> 5] = sum;
    __syncthreads();
    if (tid == 0) {
        unsigned long long t = 0;
        for (int w = 0; w < kWarps; ++w) t += s_w[w];
        if (t > 0x7FFFFFFFull) { atomicMin(p.err, (static_cast<unsigned long long>(p.row_base + r0) << 8) | EE_OVERFLOW); t = 0x7FFFFFFFull; }
        p.tile_agg[blockIdx.x] = uint32_t(t);
    }
}

__global__ void __launch_bounds__(kBlock) encode_write_kernel(const EncParams p) {
    int chunk, nrec, local; int64_t r0;
    enc_tile(p, blockIdx.x, &chunk, &r0, &nrec, &local);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t sz = tid < nrec ? p.row_size[r0 + tid] : 0u;
    uint32_t incl = sz;
    for (int d = 1; d < 32; d <<= 1) { const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= d) incl += u; }
    __shared__ uint32_t s_w[kWarps];
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    uint32_t base = p.tile_base[blockIdx.x];
    for (int w = 0; w < warp; ++w) base += s_w[w];
    const uint32_t off = base + incl - sz;
    // The tile's datums are contiguous in the output ([tile_base, tile_base + tile_total)): assemble them in
    // shared memory (per-lane byte stores are cheap there) and write the tile out with coalesced 128-bit stores.
    extern __shared__ __align__(16) uint8_t enc_smem[];
    const uint32_t tile_base = p.tile_base[blockIdx.x];
    const uint32_t tile_total = p.tile_agg[blockIdx.x];
    uint8_t* gout = p.out_data[chunk] + tile_base;
    const uint32_t galign = uint32_t(reinterpret_cast<uintptr_t>(gout) & 15u);
    const bool staged = tile_total + galign <= p.stage_cap;
    if (tid < nrec) {
        int32_t* offs = p.out_offsets[chunk];
        const int64_t i = int64_t(local) * kBlock + tid;  // row inside the chunk
        if (i == 0) offs[0] = 0;
        offs[i + 1] = int32_t(off + sz);
        EncCtx c;
        enc_init(c, p);
        c.out = staged ? enc_smem + galign + (off - tile_base) : p.out_data[chunk] + off;
        enc_range<1, 0>(c, 0, p.n_nodes, p.row_base + r0 + tid);
    }
    if (staged) {
        __syncthreads();
        const uint32_t head = min(tile_total, (16u - galign) & 15u);
        for (uint32_t i = tid; i < head; i += kBlock) gout[i] = enc_smem[galign + i];
        const uint32_t nvec = (tile_total - head) >> 4;
        const uint4* sv = reinterpret_cast<const uint4*>(enc_smem + galign + head);
        uint4* gv = reinterpret_cast<uint4*>(gout + head);
        for (uint32_t i = tid; i < nvec; i += kBlock) gv[i] = sv[i];
        for (uint32_t i = head + (nvec << 4) + tid; i < tile_total; i += kBlock) gout[i] = enc_smem[galign + i];
    }
}

// max over tiles of the tile's output bytes (sizes the staging area)
__global__ void encode_tile_max_kernel(const EncParams p, unsigned long long* out_max) {
    unsigned long long m = 0;
    for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < p.n_tiles; t += gridDim.x * blockDim.x) m = max(m, (unsigned long long)p.tile_agg[t]);
    for (int d = 16; d; d >>= 1) { const unsigned long long o = __shfl_xor_sync(0xFFFFFFFFu, m, d); if (o > m) m = o; }
    if ((threadIdx.x & 31) == 0 && m) atomicMax(out_max, m);
}

// per-chunk exclusive scan of the tile totals (one CTA per chunk)
__global__ void encode_scan_kernel(const EncParams p, unsigned long long* chunk_tot) {
    __shared__ unsigned long long s_part[32];
    const int j = blockIdx.x;
    const int t_begin = j * p.tiles_per_chunk, t_end = (j == p.k - 1) ? p.n_tiles : t_begin + p.tiles_per_chunk;
    const int T = t_end - t_begin, nthr = blockDim.x, per = (T + nthr - 1) / nthr;
    const int a = t_begin + min(T, int(threadIdx.x) * per), b = t_begin + min(T, (int(threadIdx.x) + 1) * per);
    unsigned long long local = 0;
    for (int i = a; i < b; ++i) local += p.tile_agg[i];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long incl = local;
    for (int d = 1; d < 32; d <<= 1) { unsigned long long v = __shfl_up_sync(0xFFFFFFFFu, incl, d); if (lane >= d) incl += v; }
    if (lane == 31) s_part[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        unsigned long long v = (lane < (nthr + 31) / 32) ? s_part[lane] : 0ull, w = v;
        for (int d = 1; d < 32; d <<= 1) { unsigned long long u = __shfl_up_sync(0xFFFFFFFFu, w, d); if (lane >= d) w += u; }
        s_part[lane] = w - v;
        if (lane == 31) {
            chunk_tot[j] = w;
            if (w > 0x7FFFFFFFull) atomicMin(p.err, (static_cast<unsigned long long>(p.row_base + int64_t(j) * p.chunk_rows) << 8) | EE_OVERFLOW);
        }
    }
    __syncthreads();
    unsigned long long run = s_part[warp] + (incl - local);
    for (int i = a; i < b; ++i) { p.tile_base[i] = uint32_t(run); run += p.tile_agg[i]; }
}

// ------------------------------------------------------------------------------------------------
// host: plan building from the Arrow C Data structs
// ------------------------------------------------------------------------------------------------
// A host buffer the plan touches, and the byte window [lo, hi) of it that the rows of this launch can address.
struct HostBuf { const void* ptr; size_t lo, hi; };

// Builds the encode plan for the logical rows [lo, hi) of the batch: every node indexes its Arrow buffers absolutely
// (row_add), but only the window of each buffer that those rows can reach is recorded for upload — the rows' slice of
// fixed-width columns, their offsets and the string bytes / child rows between the first and the last offset.  That is
// what lets a batch be encoded as a few row groups whose uploads, kernels and downloads overlap.
struct EncBuilder {
    std::vector<ENode> nodes;
    std::vector<int32_t> sym_off;
    std::vector<uint8_t> sym_bytes;
    std::vector<HostBuf> bufs;                 // host buffers to upload
    std::map<const void*, size_t> buf_index;   // ptr -> index in bufs (windows are merged)
    // per node: indices into bufs for validity / a / b (-1: none)
    std::vector<int> ref_v, ref_a, ref_b;

    int add_buf(const void* p, size_t lo, size_t hi) {
        if (!p) return -1;
        if (hi < lo) hi = lo;
        auto it = buf_index.find(p);
        if (it != buf_index.end()) {
            HostBuf& b = bufs[it->second];
            if (b.hi == b.lo) { b.lo = lo; b.hi = hi; }
            else if (hi > lo) { b.lo = std::min(b.lo, lo); b.hi = std::max(b.hi, hi); }
            return int(it->second);
        }
        buf_index[p] = bufs.size();
        bufs.push_back(HostBuf{p, lo, hi});
        return int(bufs.size()) - 1;
    }
    int add_bits(const void* p, int64_t i0, int64_t i1) { return add_buf(p, size_t(i0 >> 3), size_t((i1 + 7) >> 3)); }
    [[noreturn]] static void bad(const std::string& m) { throw std::runtime_error(m); }

    static bool fmt_is(const ArrowSchema* s, const char* f) { return std::strcmp(s->format, f) == 0; }
    static bool fmt_starts(const ArrowSchema* s, const char* f) { return std::strncmp(s->format, f, std::strlen(f)) == 0; }

    int new_node(NodeKind k, bool nullable, bool null_first, int level, int ulevel, int variant) {
        ENode n{};
        n.kind = k; n.flags = uint8_t((nullable ? NF_NULLABLE : 0) | (null_first ? NF_NULL_FIRST : 0));
        n.level = uint8_t(level); n.ulevel = uint8_t(ulevel); n.variant = uint8_t(variant);
        nodes.push_back(n);
        ref_v.push_back(-1); ref_a.push_back(-1); ref_b.push_back(-1);
        if (level > kMaxLevel) bad("schema nested too deeply");
        return int(nodes.size()) - 1;
    }

    // build_field_encoder / build_union_encoder / build_nullable_encoder (fast_encode.rs:191-354).
    // `base` = slice offset inherited from struct/union ancestors (children of a struct share its rows);
    // [lo, hi) = the logical rows (of the enclosing row space) this launch encodes.
    void field(const AvroNode& s, const ArrowArray* a, const ArrowSchema* as, int64_t base, int level, int ulevel, int variant, int depth,
               int64_t lo, int64_t hi) {
        if (s.k == AK::Union) {
            const bool two = s.sub.size() == 2 && (s.sub[0]->k == AK::Null || s.sub[1]->k == AK::Null);
            if (two) {
                const bool nf = s.sub[0]->k == AK::Null;
                const AvroNode& inner = nf ? *s.sub[1] : *s.sub[0];
                if (inner.k == AK::Null || inner.k == AK::Union) bad("fast_encode: unsupported nullable inner type");
                value(inner, a, as, base, true, nf, level, ulevel, variant, depth, lo, hi);
                return;
            }
            if (!fmt_starts(as, "+us:")) bad("fast_encode: expected (sparse) UnionArray for multi-variant union");
            if (size_t(a->n_children) != s.sub.size()) bad("fast_encode: union variant count mismatch");
            if (ulevel >= kMaxUnionLevel) bad("unions nested too deeply");
            // Avro variant i is the Arrow child whose type code is i (`ua.child(i as i8)`, fast_encode.rs:276), so a row's
            // type id is its Avro branch index whatever the order of the children.  Codes must be a permutation of 0..N-1.
            std::vector<int> child_of(s.sub.size(), -1);
            {
                const char* f = as->format + 4;
                bool ok = true;
                for (size_t c = 0; c < s.sub.size() && ok; ++c) {
                    char* e = nullptr;
                    const long code = std::strtol(f, &e, 10);
                    ok = e != f && (*e == ',' || (*e == '\0' && c + 1 == s.sub.size())) && code >= 0 && code < long(s.sub.size()) &&
                         child_of[size_t(code)] < 0;
                    if (ok) { child_of[size_t(code)] = int(c); f = *e ? e + 1 : e; }
                }
                if (!ok) bad(std::string("fast_encode: union type codes '") + (as->format + 4) + "' are not a permutation of 0.." +
                             std::to_string(s.sub.size() - 1));
            }
            const int id = new_node(NK_UNION, false, false, level, ulevel, variant);
            nodes[size_t(id)].n_variants = int32_t(s.sub.size());
            const int64_t off = base + a->offset;
            nodes[size_t(id)].row_add = off;
            // sparse union: one buffer (type ids); tolerate the legacy layout with a leading null validity slot
            const void* tids = (a->n_buffers >= 2 && a->buffers[0] == nullptr) ? a->buffers[1] : a->buffers[0];
            ref_a[size_t(id)] = add_buf(tids, size_t(off + lo), size_t(off + hi));
            for (size_t i = 0; i < s.sub.size(); ++i) {
                const size_t c = size_t(child_of[i]);
                field(*s.sub[i], a->children[c], as->children[c], off, level + 1, ulevel + 1, int(i), depth, lo, hi);
            }
            nodes[size_t(id)].end = int32_t(nodes.size());
            return;
        }
        value(s, a, as, base, false, false, level, ulevel, variant, depth, lo, hi);
    }

    void value(const AvroNode& s, const ArrowArray* a, const ArrowSchema* as, int64_t base, bool nullable, bool nf, int level, int ulevel,
               int variant, int depth, int64_t lo, int64_t hi) {
        const int64_t off = base + a->offset;
        const int64_t i0 = off + lo, i1 = off + hi;  // elements of this array's buffers the rows can address
        auto leaf = [&](NodeKind k, const char* what, bool ok, size_t width) {
            if (!ok) bad(std::string("fast_encode: arrow array downcast failed (expected ") + what + ", got format '" + as->format + "')");
            const int id = new_node(k, nullable, nf, level, ulevel, variant);
            nodes[size_t(id)].row_add = off;
            nodes[size_t(id)].end = id + 1;
            if (nullable) ref_v[size_t(id)] = add_bits(a->buffers[0], i0, i1);
            if (width) ref_a[size_t(id)] = k == NK_BOOL ? add_bits(a->buffers[1], i0, i1) : add_buf(a->buffers[1], size_t(i0) * width, size_t(i1) * width);
            return id;
        };
        auto utf8 = [&](NodeKind k) {
            const int id = leaf(k, "Utf8", fmt_is(as, "u"), 0);
            const int32_t* offs = static_cast<const int32_t*>(a->buffers[1]);
            ref_a[size_t(id)] = add_buf(offs, size_t(i0) * 4, size_t(i1 + 1) * 4);
            const size_t d0 = offs ? size_t(offs[i0]) : 0, d1 = offs ? size_t(offs[i1]) : 0;
            ref_b[size_t(id)] = add_buf(a->buffers[2], d0, d1);
            return id;
        };
        switch (s.k) {
            case AK::Int: leaf(NK_I32, "Int32", fmt_is(as, "i"), 4); break;
            case AK::Date: leaf(NK_I32, "Date32", fmt_is(as, "tdD"), 4); break;
            case AK::Long: leaf(NK_I64, "Int64", fmt_is(as, "l"), 8); break;
            case AK::TsMillis: leaf(NK_I64, "Timestamp(ms)", fmt_starts(as, "tsm:"), 8); break;
            case AK::TsMicros: leaf(NK_I64, "Timestamp(us)", fmt_starts(as, "tsu:"), 8); break;
            case AK::Float: leaf(NK_F32, "Float32", fmt_is(as, "f"), 4); break;
            case AK::Double: leaf(NK_F64, "Float64", fmt_is(as, "g"), 8); break;
            case AK::Bool: leaf(NK_BOOL, "Boolean", fmt_is(as, "b"), 1); break;
            case AK::String: utf8(NK_STR); break;
            case AK::Enum: {
                const int id = utf8(NK_ENUM);
                nodes[size_t(id)].sym_base = int32_t(sym_off.size());
                nodes[size_t(id)].n_sym = int32_t(s.symbols.size());
                for (auto& sym : s.symbols) { sym_off.push_back(int32_t(sym_bytes.size())); sym_bytes.insert(sym_bytes.end(), sym.begin(), sym.end()); }
                sym_off.push_back(int32_t(sym_bytes.size()));
                break;
            }
            case AK::Null: { const int id = new_node(NK_NULL, false, false, level, ulevel, variant); nodes[size_t(id)].end = id + 1; break; }
            case AK::Record: {
                if (!fmt_is(as, "+s")) bad("fast_encode: expected StructArray for record");
                const int id = new_node(NK_REC, nullable, nf, level, ulevel, variant);
                nodes[size_t(id)].row_add = off;
                if (nullable) ref_v[size_t(id)] = add_bits(a->buffers[0], i0, i1);
                record_children(s, a, as, off, level + 1, ulevel, depth, lo, hi);
                nodes[size_t(id)].end = int32_t(nodes.size());
                break;
            }
            case AK::Array: case AK::Map: {
                const bool is_map = s.k == AK::Map;
                if (!fmt_is(as, is_map ? "+m" : "+l")) bad(is_map ? "fast_encode: expected MapArray for map schema" : "fast_encode: expected ListArray for array schema");
                if (depth + 1 > kMaxListDepth) bad("arrays/maps nested deeper than " + std::to_string(kMaxListDepth) + " levels are not supported");
                const int id = new_node(is_map ? NK_MAP : NK_LIST, nullable, nf, level, ulevel, variant);
                nodes[size_t(id)].row_add = off;
                if (nullable) ref_v[size_t(id)] = add_bits(a->buffers[0], i0, i1);
                const int32_t* offs = static_cast<const int32_t*>(a->buffers[1]);
                ref_a[size_t(id)] = add_buf(offs, size_t(i0) * 4, size_t(i1 + 1) * 4);
                if (a->n_children != 1) bad("fast_encode: list/map without a child");
                const int64_t c0 = offs ? int64_t(offs[i0]) : 0, c1 = offs ? int64_t(offs[i1]) : 0;  // the rows' items
                if (is_map) {
                    const ArrowArray* en = a->children[0];
                    const ArrowSchema* ens = as->children[0];
                    if (!fmt_is(ens, "+s") || en->n_children != 2) bad("fast_encode: map entries must be a 2-field struct");
                    if (!fmt_is(ens->children[0], "u")) bad("fast_encode: map keys must be StringArray");
                    AvroNode key;
                    key.k = AK::String;
                    value(key, en->children[0], ens->children[0], en->offset, false, false, level + 1, ulevel, 0xFF, depth + 1, c0, c1);
                    field(*s.sub[0], en->children[1], ens->children[1], en->offset, level + 1, ulevel, 0xFF, depth + 1, c0, c1);
                } else {
                    field(*s.sub[0], a->children[0], as->children[0], 0, level + 1, ulevel, 0xFF, depth + 1, c0, c1);
                }
                nodes[size_t(id)].end = int32_t(nodes.size());
                break;
            }
            default: bad("fast_encode: unsupported schema");
        }
    }

    // build_record_encoder (:153-189): Arrow columns are matched to Avro fields BY NAME
    void record_children(const AvroNode& rs, const ArrowArray* a, const ArrowSchema* as, int64_t base, int level, int ulevel, int depth,
                         int64_t lo, int64_t hi) {
        for (auto& f : rs.fields) {
            int idx = -1;
            for (int64_t i = 0; i < as->n_children; ++i)
                if (as->children[i]->name && f.name == as->children[i]->name) idx = int(i);  // later duplicates win, like HashMap::collect
            if (idx < 0) {
                std::string avail = "[";
                for (int64_t i = 0; i < as->n_children; ++i) { if (i) avail += ", "; avail += std::string("\"") + (as->children[i]->name ? as->children[i]->name : "") + "\""; }
                avail += "]";
                bad("Arrow struct missing column '" + f.name + "' required by Avro schema. Available columns: " + avail);
            }
            field(*f.type, a->children[idx], as->children[idx], base, level, ulevel, 0xFF, depth, lo, hi);
        }
    }
};

}  // namespace
}  // namespace rv
extern "C" void* rv_internal_dev_get(size_t bytes, int device, size_t* actual);
extern "C" void rv_internal_dev_put(void* p, size_t actual, int device);
namespace rv {
namespace {

struct DevMem {  // from the library's device-memory cache (blocks return after the stream was synchronised)
    void* p = nullptr;
    size_t actual = 0;
    int device = 0;
    ~DevMem() { if (p) rv_internal_dev_put(p, actual, device); }
    cudaError_t alloc(size_t n) {
        if (cudaGetDevice(&device) != cudaSuccess) return cudaErrorInvalidDevice;
        p = rv_internal_dev_get(n ? n : 1, device, &actual);
        return p ? cudaSuccess : cudaErrorMemoryAllocation;
    }
};

}  // namespace
}  // namespace rv

using namespace rv;

// Access to the schema internals lives in engine.cu.
extern "C" const void* rv_schema_avro_root(const rv_schema* s);
extern "C" int rv_schema_is_projection(const rv_schema* s);
extern "C" void rv_set_last_error(const char* msg);

struct rv_encoded {
    struct Chunk { void* host = nullptr; int64_t rows = 0, data_bytes = 0; };
    std::vector<Chunk> chunks;  // host: [offsets (rows+1)*4, padded to 64][data]
    std::vector<std::shared_ptr<void>> keep;
};

namespace {

struct EncExport {
    std::shared_ptr<void> keep;
    const void* buffers[3];
};
void release_encoded_array(ArrowArray* a) {
    if (!a || !a->release) return;
    delete static_cast<EncExport*>(a->private_data);
    a->release = nullptr;
}
void release_static_schema(ArrowSchema* s) { s->release = nullptr; }

#define ENC_CUDA(expr)                                                                                               \
    do {                                                                                                             \
        cudaError_t e_ = (expr);                                                                                     \
        if (e_ != cudaSuccess) { rv_set_last_error((std::string(#expr) + ": " + cudaGetErrorString(e_)).c_str()); return RV_ERR_CUDA; } \
    } while (0)

}  // namespace

extern "C" {

// Replaces ruhvro::serialize::serialize_record_batch (ruhvro/src/serialize.rs:38-67).
static thread_local float t_enc_timings[5] = {0, 0, 0, 0, 0};
extern "C" int rv_last_encode_timings(float* out_ms, int cap) {
    const int n = cap < 5 ? cap : 5;
    for (int i = 0; i < n; ++i) out_ms[i] = t_enc_timings[i];
    return n;
}

// One row group of the batch — chunks [c0, c1), rows [g0, g1) — on its own stream: upload of the buffer windows its rows
// reach, size -> scan -> write, download of its chunks.  Returns a status; the message goes to *msg (worker threads have
// their own thread-local error string).
static rv_status encode_group(const AvroNode* top, const ArrowArray* batch, const ArrowSchema* batch_schema, int64_t g0, int64_t g1,
                              int c0, int c1, int64_t chunk_rows, cudaStream_t stream, rv_encoded* res, float* ms5,
                              std::string* msg) {
#define GRP_CUDA(expr)                                                                                   \
    do {                                                                                                 \
        cudaError_t e_ = (expr);                                                                         \
        if (e_ != cudaSuccess) { *msg = std::string(#expr) + ": " + cudaGetErrorString(e_); cudaStreamSynchronize(stream); (void)cudaGetLastError(); return RV_ERR_CUDA; } \
    } while (0)
    EncBuilder b;
    try {
        b.record_children(*top, batch, batch_schema, batch->offset, 1, 0, 0, g0, g1);
    } catch (const std::exception& e) {
        *msg = e.what();
        return RV_ERR_INVALID;
    }
    const int64_t n = g1 - g0;
    const int k = c1 - c0;
    struct Ev {
        cudaEvent_t e[8] = {};
        Ev() { for (auto& x : e) if (cudaEventCreate(&x) != cudaSuccess) x = nullptr; }
        ~Ev() { for (auto& x : e) if (x) cudaEventDestroy(x); (void)cudaGetLastError(); }
        void rec(int i, cudaStream_t st) { if (e[i]) cudaEventRecord(e[i], st); }
        float ms(int a, int b_) { float t = 0; if (e[a] && e[b_] && cudaEventElapsedTime(&t, e[a], e[b_]) == cudaSuccess) return t; (void)cudaGetLastError(); return 0; }
    } ev;

    // ---- upload the windows of the Arrow buffers this group's rows reach (one device arena) ----
    size_t total = 0;
    std::vector<size_t> boff(b.bufs.size()), blo(b.bufs.size());
    for (size_t i = 0; i < b.bufs.size(); ++i) {
        blo[i] = b.bufs[i].lo & ~size_t(63);                 // windows start on a 64-byte boundary of the source buffer
        boff[i] = total;
        total += (b.bufs[i].hi - blo[i] + 8 + 63) & ~size_t(63);
    }
    DevMem d_in, d_nodes, d_symoff, d_symbytes, d_rowsize, d_agg, d_base, d_err, d_tot, d_ptrs;
    GRP_CUDA(d_in.alloc(total));
    ev.rec(0, stream);
    // Buffers in ordinary pageable memory are staged through a pinned arena in 16 MiB pieces (a direct copy runs at a
    // fraction of PCIe speed); pinned / registered buffers — e.g. batches this library decoded — go direct.
    bool pageable = false;
    for (size_t i = 0; i < b.bufs.size() && !pageable; ++i) {
        if (b.bufs[i].hi - blo[i] < (size_t(1) << 20)) continue;
        cudaPointerAttributes at{};
        if (cudaPointerGetAttributes(&at, b.bufs[i].ptr) != cudaSuccess) { (void)cudaGetLastError(); pageable = true; }
        else pageable = at.type == cudaMemoryTypeUnregistered;
    }
    std::shared_ptr<void> h_in_keep;
    uint8_t* h_in = nullptr;
    if (pageable && total >= (size_t(4) << 20)) {
        h_in = static_cast<uint8_t*>(rv_host_alloc(total));
        if (!h_in) { *msg = "pinned staging allocation failed"; return RV_ERR_CUDA; }
        h_in_keep = std::shared_ptr<void>(h_in, [](void* q) { rv_host_free(q); });
    }
    const size_t kPiece = size_t(16) << 20;
    for (size_t i = 0; i < b.bufs.size(); ++i) {
        const uint8_t* src = static_cast<const uint8_t*>(b.bufs[i].ptr) + blo[i];
        const size_t bytes = b.bufs[i].hi - blo[i];
        uint8_t* dst = static_cast<uint8_t*>(d_in.p) + boff[i];
        for (size_t o = 0; o < bytes; o += kPiece) {
            const size_t len = std::min(kPiece, bytes - o);
            const uint8_t* from = src + o;
            if (h_in) { std::memcpy(h_in + boff[i] + o, from, len); from = h_in + boff[i] + o; }
            GRP_CUDA(cudaMemcpyAsync(dst + o, from, len, cudaMemcpyHostToDevice, stream));
        }
    }
    for (size_t i = 0; i < b.nodes.size(); ++i) {
        // device address of the buffer's byte 0 (the window starts at byte blo): nodes keep indexing absolutely
        auto fix = [&](int ref) -> const uint8_t* { return ref < 0 ? nullptr : static_cast<const uint8_t*>(d_in.p) + boff[size_t(ref)] - blo[size_t(ref)]; };
        b.nodes[i].validity = fix(b.ref_v[i]);
        b.nodes[i].buf_a = fix(b.ref_a[i]);
        b.nodes[i].buf_b = fix(b.ref_b[i]);
    }
    GRP_CUDA(d_nodes.alloc(b.nodes.size() * sizeof(ENode)));
    GRP_CUDA(cudaMemcpyAsync(d_nodes.p, b.nodes.data(), b.nodes.size() * sizeof(ENode), cudaMemcpyHostToDevice, stream));
    GRP_CUDA(d_symoff.alloc(b.sym_off.size() * 4));
    GRP_CUDA(d_symbytes.alloc(b.sym_bytes.size()));
    if (!b.sym_off.empty()) GRP_CUDA(cudaMemcpyAsync(d_symoff.p, b.sym_off.data(), b.sym_off.size() * 4, cudaMemcpyHostToDevice, stream));
    if (!b.sym_bytes.empty()) GRP_CUDA(cudaMemcpyAsync(d_symbytes.p, b.sym_bytes.data(), b.sym_bytes.size(), cudaMemcpyHostToDevice, stream));
    ev.rec(1, stream);

    EncParams p{};
    p.nodes = static_cast<const ENode*>(d_nodes.p); p.n_nodes = int32_t(b.nodes.size());
    p.sym_off = static_cast<const int32_t*>(d_symoff.p); p.sym_bytes = static_cast<const uint8_t*>(d_symbytes.p);
    p.n = n; p.row_base = g0; p.chunk_rows = chunk_rows; p.k = k;
    const int64_t tpc = std::max<int64_t>(1, (chunk_rows + kBlock - 1) / kBlock);
    const int64_t last_rows = n - chunk_rows * (k - 1);
    const int64_t n_tiles = n > 0 ? tpc * (k - 1) + (last_rows + kBlock - 1) / kBlock : 0;
    p.tiles_per_chunk = int32_t(tpc); p.n_tiles = int32_t(n_tiles);
    std::vector<unsigned long long> chunk_tot(static_cast<size_t>(k), 0ull);
    unsigned long long max_tile = 0;
    if (n > 0) {
        GRP_CUDA(d_rowsize.alloc(size_t(n) * 4));
        GRP_CUDA(d_agg.alloc(size_t(n_tiles) * 4));
        GRP_CUDA(d_base.alloc(size_t(n_tiles) * 4));
        GRP_CUDA(d_err.alloc(16));
        GRP_CUDA(d_tot.alloc(size_t(k) * 8));
        GRP_CUDA(cudaMemsetAsync(d_err.p, 0xFF, 8, stream));
        p.row_size = static_cast<uint32_t*>(d_rowsize.p); p.tile_agg = static_cast<uint32_t*>(d_agg.p);
        p.tile_base = static_cast<uint32_t*>(d_base.p); p.err = static_cast<unsigned long long*>(d_err.p);
        encode_size_kernel<<<unsigned(n_tiles), kBlock, 0, stream>>>(p);
        ev.rec(2, stream);
        int thr = 32;
        while (thr < 1024 && thr < tpc) thr <<= 1;
        encode_scan_kernel<<<unsigned(k), thr, 0, stream>>>(p, static_cast<unsigned long long*>(d_tot.p));
        GRP_CUDA(cudaMemsetAsync(static_cast<uint8_t*>(d_err.p) + 8, 0, 8, stream));
        encode_tile_max_kernel<<<std::max(1, std::min(int((n_tiles + 255) / 256), 592)), 256, 0, stream>>>(p, static_cast<unsigned long long*>(d_err.p) + 1);
        GRP_CUDA(cudaGetLastError());
        ev.rec(3, stream);
        unsigned long long err_word = ~0ull;
        GRP_CUDA(cudaMemcpyAsync(&max_tile, static_cast<uint8_t*>(d_err.p) + 8, 8, cudaMemcpyDeviceToHost, stream));
        GRP_CUDA(cudaMemcpyAsync(&err_word, d_err.p, 8, cudaMemcpyDeviceToHost, stream));
        GRP_CUDA(cudaMemcpyAsync(chunk_tot.data(), d_tot.p, size_t(k) * 8, cudaMemcpyDeviceToHost, stream));
        GRP_CUDA(cudaStreamSynchronize(stream));
        if (err_word != ~0ull) {
            const uint32_t code = uint32_t(err_word & 0xFF);
            const std::string what = code == EE_ENUM ? "fast_encode: enum symbol not in schema"
                                     : code == EE_BRANCH ? "fast_encode: union type_id out of range"
                                                         : "Arrow i32 offset overflow: a chunk's datums exceed 2 GiB";
            *msg = what + " (row " + std::to_string(err_word >> 8) + ")";
            return rv_status(code);
        }
    }
    // ---- outputs: per chunk [offsets][data] on the device, then one D2H per chunk into pinned memory ----
    std::vector<DevMem> d_out(static_cast<size_t>(k));
    std::vector<uint8_t*> h_data(static_cast<size_t>(k), nullptr);
    std::vector<int32_t*> h_offs(static_cast<size_t>(k), nullptr);
    std::vector<size_t> off_bytes(static_cast<size_t>(k), 0);
    for (int j = 0; j < k; ++j) {
        auto& c = res->chunks[size_t(c0 + j)];
        c.data_bytes = int64_t(chunk_tot[size_t(j)]);
        off_bytes[size_t(j)] = (size_t(c.rows + 1) * 4 + 63) & ~size_t(63);
        GRP_CUDA(d_out[size_t(j)].alloc(off_bytes[size_t(j)] + size_t(c.data_bytes) + 64));
        h_offs[size_t(j)] = static_cast<int32_t*>(d_out[size_t(j)].p);
        h_data[size_t(j)] = static_cast<uint8_t*>(d_out[size_t(j)].p) + off_bytes[size_t(j)];
        if (c.rows == 0) GRP_CUDA(cudaMemsetAsync(d_out[size_t(j)].p, 0, 64, stream));
    }
    if (n > 0) {
        GRP_CUDA(d_ptrs.alloc(size_t(k) * 16));
        GRP_CUDA(cudaMemcpyAsync(d_ptrs.p, h_data.data(), size_t(k) * 8, cudaMemcpyHostToDevice, stream));
        GRP_CUDA(cudaMemcpyAsync(static_cast<uint8_t*>(d_ptrs.p) + size_t(k) * 8, h_offs.data(), size_t(k) * 8, cudaMemcpyHostToDevice, stream));
        p.out_data = static_cast<uint8_t* const*>(d_ptrs.p);
        p.out_offsets = reinterpret_cast<int32_t* const*>(static_cast<uint8_t*>(d_ptrs.p) + size_t(k) * 8);
        // staging area: the largest tile (+ alignment), capped so at least two CTAs share an SM
        size_t stage = std::min<size_t>(size_t(max_tile) + 32, 100 * 1024);
        stage = (stage + 63) & ~size_t(63);
        {   // function attributes are per device
            static std::mutex attr_mu;
            static std::vector<char> attr_set;
            int dev_now = 0;
            GRP_CUDA(cudaGetDevice(&dev_now));
            std::lock_guard<std::mutex> g(attr_mu);
            if (attr_set.size() <= size_t(dev_now)) attr_set.resize(size_t(dev_now) + 1, 0);
            if (!attr_set[size_t(dev_now)]) {
                GRP_CUDA(cudaFuncSetAttribute(encode_write_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024));
                GRP_CUDA(cudaFuncSetAttribute(encode_write_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
                attr_set[size_t(dev_now)] = 1;
            }
        }
        p.stage_cap = uint32_t(stage);
        ev.rec(4, stream);
        encode_write_kernel<<<unsigned(n_tiles), kBlock, stage, stream>>>(p);
        ev.rec(5, stream);
        GRP_CUDA(cudaGetLastError());
    }
    ev.rec(6, stream);
    for (int j = 0; j < k; ++j) {
        auto& c = res->chunks[size_t(c0 + j)];
        const size_t bytes = off_bytes[size_t(j)] + size_t(c.data_bytes);
        void* h = rv_host_alloc(bytes + 64);
        if (!h) { *msg = "pinned allocation of an output chunk failed"; cudaStreamSynchronize(stream); return RV_ERR_CUDA; }
        res->keep[size_t(c0 + j)] = std::shared_ptr<void>(h, [](void* q) { rv_host_free(q); });  // slot per chunk: rv_encoded_export(i) holds keep[i]
        c.host = h;
        GRP_CUDA(cudaMemcpyAsync(h, d_out[size_t(j)].p, bytes, cudaMemcpyDeviceToHost, stream));
    }
    ev.rec(7, stream);
    GRP_CUDA(cudaStreamSynchronize(stream));
    ms5[3] = ev.ms(0, 1);
    ms5[4] = ev.ms(6, 7);
    if (n > 0) { ms5[0] = ev.ms(1, 2); ms5[1] = ev.ms(2, 3); ms5[2] = ev.ms(4, 5); }
    return RV_OK;
#undef GRP_CUDA
}

rv_status rv_encode_host(const rv_schema* s, struct ArrowArray* batch, struct ArrowSchema* batch_schema, int64_t num_chunks, rv_encoded** out) {
    if (!s || !batch || !batch_schema || !out) { rv_set_last_error("null argument"); return RV_ERR_INVALID; }
    *out = nullptr;
    struct Releaser {  // ownership of the C structs moved to us
        ArrowArray* a; ArrowSchema* s;
        ~Releaser() { if (a && a->release) a->release(a); if (s && s->release) s->release(s); }
    } releaser{batch, batch_schema};
    if (rv_schema_is_projection(s)) {
        rv_set_last_error("fast_encode: a column projection (rv_schema_project) or a resolved handle (rv_schema_resolve) is not a schema to write with; encode with the full schema handle");
        return RV_ERR_INVALID;
    }
    if (!rv_schema_is_supported(s)) { rv_set_last_error("schema is outside the direct-encode subset; this library has no Value-tree CPU fallback"); return RV_ERR_SCHEMA; }
    const AvroNode* top = static_cast<const AvroNode*>(rv_schema_avro_root(s));
    if (std::strcmp(batch_schema->format, "+s") != 0) { rv_set_last_error("fast_encode: expected StructArray"); return RV_ERR_INVALID; }
    for (float& t : t_enc_timings) t = 0;
    {   // plan errors (missing column, wrong Arrow type, ...) surface before any GPU work, on the calling thread
        EncBuilder probe;
        try {
            probe.record_children(*top, batch, batch_schema, batch->offset, 1, 0, 0, 0, 0);
        } catch (const std::exception& e) {
            rv_set_last_error(e.what());
            return RV_ERR_INVALID;
        }
    }
    int ndev = 0, device = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { rv_set_last_error("no CUDA device available (this library has no CPU fallback)"); return RV_ERR_CUDA; }
    ENC_CUDA(cudaGetDevice(&device));
    const int64_t n = batch->length;
    const int64_t k64 = clamp_chunks(num_chunks, n);  // serialize.rs:15-17
    const int k = int(k64);
    const int64_t chunk_rows = n / k;                 // slice_struct :19-30
    auto res = std::make_unique<rv_encoded>();
    res->chunks.resize(size_t(k));
    res->keep.resize(size_t(k));
    for (int j = 0; j < k; ++j) res->chunks[size_t(j)].rows = (j == k - 1) ? n - chunk_rows * (k - 1) : chunk_rows;

    // Row groups of whole chunks, each on its own stream and host thread: the upload of group g+1 overlaps the kernels
    // and the download of group g (full-duplex PCIe), like the decode side's chunk pipeline.  Small batches: one group.
    int groups = 1;
    if (k >= 2 && n >= (int64_t(1) << 18)) groups = std::min(k, 4);
    if (const char* e = std::getenv("RV_ENC_GROUPS")) groups = std::max(1, std::min(k, std::atoi(e)));
    std::vector<rv_status> status(size_t(groups), RV_OK);
    std::vector<std::string> message(static_cast<size_t>(groups));
    std::vector<std::array<float, 5>> times(static_cast<size_t>(groups), std::array<float, 5>{0, 0, 0, 0, 0});
    auto run = [&](int g) {
        cudaSetDevice(device);
        const int c0 = int(int64_t(g) * k / groups), c1 = int(int64_t(g + 1) * k / groups);
        const int64_t g0 = int64_t(c0) * chunk_rows, g1 = (c1 == k) ? n : int64_t(c1) * chunk_rows;
        cudaStream_t stream = nullptr;
        if (groups > 1 && cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking) != cudaSuccess) { status[size_t(g)] = RV_ERR_CUDA; message[size_t(g)] = "stream creation failed"; return; }
        try {
            status[size_t(g)] = encode_group(top, batch, batch_schema, g0, g1, c0, c1, chunk_rows, stream, res.get(), times[size_t(g)].data(), &message[size_t(g)]);
        } catch (const std::exception& e) {  // bad_alloc on a group's own thread must not terminate the process
            cudaStreamSynchronize(stream);
            (void)cudaGetLastError();
            status[size_t(g)] = RV_ERR_INVALID;
            message[size_t(g)] = e.what();
        }
        if (stream) cudaStreamDestroy(stream);
    };
    if (groups == 1) run(0);
    else {
        std::vector<std::thread> pool;
        for (int g = 1; g < groups; ++g) {
            try { pool.emplace_back(run, g); }
            catch (const std::system_error&) { run(g); }   // no thread to be had: this group runs here
        }
        run(0);
        for (auto& t : pool) t.join();
    }
    for (int g = 0; g < groups; ++g) {
        if (status[size_t(g)] != RV_OK) { rv_set_last_error(message[size_t(g)].c_str()); return status[size_t(g)]; }  // lowest rows first
        for (int q = 0; q < 5; ++q) t_enc_timings[q] += times[size_t(g)][size_t(q)];
    }
    *out = res.release();
    return RV_OK;
}

int64_t rv_encoded_num_chunks(const rv_encoded* r) { return r ? int64_t(r->chunks.size()) : 0; }

// Exports chunk i as an Arrow Binary array (format "z": i32 offsets + bytes), like GenericBinaryArray<i32>.
rv_status rv_encoded_export(rv_encoded* r, int64_t i, struct ArrowArray* out_array, struct ArrowSchema* out_schema) {
    if (!r || !out_array || i < 0 || i >= int64_t(r->chunks.size())) { rv_set_last_error("bad argument"); return RV_ERR_INVALID; }
    const auto& c = r->chunks[size_t(i)];
    auto* ex = new EncExport();
    ex->keep = r->keep[size_t(i)];
    const size_t off_bytes = (size_t(c.rows + 1) * 4 + 63) & ~size_t(63);
    ex->buffers[0] = nullptr;
    ex->buffers[1] = c.host;
    ex->buffers[2] = static_cast<const uint8_t*>(c.host) + off_bytes;
    out_array->length = c.rows; out_array->null_count = 0; out_array->offset = 0;
    out_array->n_buffers = 3; out_array->n_children = 0; out_array->buffers = ex->buffers;
    out_array->children = nullptr; out_array->dictionary = nullptr;
    out_array->release = release_encoded_array; out_array->private_data = ex;
    if (out_schema) {
        out_schema->format = "z"; out_schema->name = ""; out_schema->metadata = nullptr; out_schema->flags = 0;
        out_schema->n_children = 0; out_schema->children = nullptr; out_schema->dictionary = nullptr;
        out_schema->release = release_static_schema; out_schema->private_data = nullptr;
    }
    return RV_OK;
}

void rv_encoded_free(rv_encoded* r) { delete r; }

}  // extern "C"
