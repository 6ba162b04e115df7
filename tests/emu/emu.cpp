// TEST INFRASTRUCTURE ONLY — host emulation of the GPU decode pipeline.
//
// Compiles the product's walker (pyruhvro_b200/csrc/walker.cuh), plan, layout and Arrow export
// for the CPU and steps through the same count -> per-chunk scan -> exact layout -> emit ->
// null-count sequence the kernels run, one 256-"lane" tile at a time.  It exists so the decode
// LOGIC can be checked against the oracle in the GPU-less build container; it is never loaded by
// the product (pyruhvro_b200 has no CPU path) and is not what the -m gpu tests exercise.
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <cstdio>
#include <stdexcept>
#include <algorithm>
#include <memory>
#include <string>
#include <vector>

#include "../../pyruhvro_b200/csrc/plan.hpp"
#include "../../pyruhvro_b200/csrc/result.hpp"
#include "../../pyruhvro_b200/csrc/gather.hpp"
#include "../../pyruhvro_b200/csrc/schema.hpp"
#include "../../pyruhvro_b200/csrc/interp.cuh"
#include "../../pyruhvro_b200/csrc/ocf.hpp"
#include "../../pyruhvro_b200/csrc/ocf_walk.cuh"
#ifdef EMU_GEN_WALKER
#include EMU_GEN_WALKER   // schema-specialised walker source produced by rv_schema_walker_source()
using EmuWalker = rv::gen::Walker;
#else
using EmuWalker = rv::InterpWalker;
#endif

using namespace rv;

namespace {
constexpr int kTile = rv::kBlock;

struct Tile { int chunk; int64_t r0; int nrec; int local; };

std::vector<Tile> make_tiles(int64_t n, int k) {
    std::vector<Tile> t;
    const int64_t cr = n / k;
    for (int j = 0; j < k; ++j) {
        const int64_t cs = int64_t(j) * cr, ce = (j == k - 1) ? n : cs + cr;
        int local = 0;
        for (int64_t r = cs; r < ce; r += kTile) t.push_back(Tile{j, r, int(std::min<int64_t>(kTile, ce - r)), local++});
    }
    return t;
}

using Ctx = WalkCtx<false>;      // PRECISE flavour: reads the record where it lies
using FastCtx = WalkCtx<true>;   // FAST flavour: reads a padded copy of the tile's byte window, like the staged shared-memory window

// register-cursor walkers exchange their cursors with the emulation's cur[stream][lane] table
template <class Q>
void store_cursors(const Q& q, uint32_t* cur_lane, int S) {
    if constexpr (EmuWalker::kRegCursors) for (int s = 0; s < S; ++s) cur_lane[size_t(s) * kTile] = q.v[s];
}
template <class Q>
void load_cursors(Q& q, const uint32_t* cur_lane, int S) {
    if constexpr (EmuWalker::kRegCursors) for (int s = 0; s < S; ++s) q.v[s] = cur_lane[size_t(s) * kTile];
}

template <class C>
void init_common(C& c, const Plan& plan, const Tile& t, int lane, uint32_t* cur, void* const* bufs) {
    std::memset(&c, 0, sizeof c);
    c.nodes = plan.nodes.data();
    c.cur = cur + lane;
    c.cur_stride = kTile;
    c.sym_off = plan.sym_off.data();
    c.sym_bytes = plan.sym_bytes.data();
    c.bufs = bufs;
    c.in_range = lane < t.nrec;
    c.row0 = uint32_t(t.local) * kTile + uint32_t(lane);
    c.store_word = false;
}

void init_ctx(Ctx& c, const Plan& plan, const uint8_t* data, const int64_t* off, const Tile& t, int lane,
              uint32_t* cur, int S, void* const* bufs) {
    init_common(c, plan, t, lane, cur, bufs);
    (void)S;
    if (c.in_range) {
        const int64_t r = t.r0 + lane;
        c.base = data + off[r];
        c.pos = 0;
        c.end = uint32_t(off[r + 1] - off[r]);
    }
}

// The tile's bytes followed by kWindowPad bytes of junk (the device leaves whatever was in shared memory there).
std::vector<uint8_t> make_window(const uint8_t* data, const int64_t* off, const Tile& t) {
    const int64_t t0 = off[t.r0], t1 = off[t.r0 + t.nrec];
    std::vector<uint8_t> w(size_t(t1 - t0) + kWindowPad, uint8_t(0xA5));
    if (t1 > t0) std::memcpy(w.data(), data + t0, size_t(t1 - t0));
    return w;
}

void init_fast(FastCtx& c, const Plan& plan, const std::vector<uint8_t>& window, const int64_t* off, const Tile& t, int lane,
               uint32_t* cur, void* const* bufs) {
    init_common(c, plan, t, lane, cur, bufs);
    c.base = window.data();
    if (c.in_range) {
        const int64_t r = t.r0 + lane, t0 = off[t.r0];
        c.pos = uint32_t(off[r] - t0);
        c.end = uint32_t(off[r + 1] - t0);
    }
}

// COUNT of one tile the way fused_body does it: every lane walks FAST; a lane whose record is not plain repeats it
// PRECISE (which alone decides errors); a 32-lane "warp" with any such lane is marked for the precise EMIT.
// Returns the first error's lane or -1.
int count_tile(const Plan& plan, const uint8_t* data, const int64_t* off, const Tile& t, int S, std::vector<uint32_t>& cur,
               bool* warp_precise, uint32_t* err_code, long long* fast_lanes, long long* precise_lanes) {
    std::fill(cur.begin(), cur.end(), 0u);
    const std::vector<uint8_t> window = make_window(data, off, t);
    for (int w = 0; w < kTile / 32; ++w) warp_precise[w] = false;
    for (int lane = 0; lane < kTile; ++lane) {
        FastCtx f;
        init_fast(f, plan, window, off, t, lane, cur.data(), nullptr);
        EmuWalker::Cur q{};
        EmuWalker::walk<WM_COUNT>(f, int(plan.nodes.size()), q);
        if (f.in_range && f.pos > f.end + kWindowPad) { std::fprintf(stderr, "emu: fast reader ran %u bytes past the record\n", f.pos - f.end); std::abort(); }
        if (f.in_range && f.err) {
            warp_precise[lane / 32] = true;
            for (int s = 0; s < S; ++s) cur[size_t(s) * kTile + lane] = 0;
            Ctx c;
            init_ctx(c, plan, data, off, t, lane, cur.data(), S, nullptr);
            q = EmuWalker::Cur{};
            EmuWalker::walk<WM_COUNT>(c, int(plan.nodes.size()), q);
            store_cursors(q, cur.data() + lane, S);
            if (precise_lanes) ++*precise_lanes;
            if (c.err) { *err_code = c.err; return lane; }
        } else {
            store_cursors(q, cur.data() + lane, S);
            if (fast_lanes && f.in_range) ++*fast_lanes;
        }
    }
    return -1;
}
struct Keep { std::shared_ptr<Plan> plan; std::vector<ChunkOut> chunks; uint8_t* arena; ~Keep() { std::free(arena); } };
struct Decoded {
    std::shared_ptr<Plan> plan;
    std::vector<ArrowField> fields;
    std::shared_ptr<Keep> keep;   // arena + final chunks (null counts filled)
    int k = 0;
};

// The emulated pipeline up to (and including) null counts.  Returns 0, or the error code of the first failing record.
int decode_core(const char* json, size_t len, const uint8_t* data, const int64_t* off, int64_t n, int64_t num_chunks, Decoded& out, int64_t* err_record) {
    auto avro = parse_avro_schema(json, len);
    std::string why;
    if (!is_supported(*avro, &why)) throw std::runtime_error("unsupported: " + why);
    out.fields = to_arrow_fields(*avro);
    auto plan_sp = std::make_shared<Plan>(build_plan(*avro, out.fields));
    out.plan = plan_sp;
    const Plan& plan = *plan_sp;
    const int S = int(plan.streams.size()), S1 = std::max(S, 1);
    const int k = int(clamp_chunks(num_chunks, n));
    out.k = k;
    auto tiles = make_tiles(n, k);
    std::vector<uint32_t> cur(size_t(S1) * kTile);
    std::vector<std::vector<uint32_t>> tile_agg(tiles.size(), std::vector<uint32_t>(size_t(S1), 0));
    // ---- count pass ----
    long long fast_lanes = 0, precise_lanes = 0;
    for (size_t ti = 0; ti < tiles.size(); ++ti) {
        bool wp[kTile / 32];
        uint32_t code = 0;
        const int bad = count_tile(plan, data, off, tiles[ti], S, cur, wp, &code, &fast_lanes, &precise_lanes);
        if (bad >= 0) { *err_record = tiles[ti].r0 + bad; return int(code); }
        for (int s = 0; s < S; ++s) {
            uint64_t sum = 0;
            for (int lane = 0; lane < kTile; ++lane) sum += cur[size_t(s) * kTile + lane];
            if (sum > 0x7FFFFFFFull) { *err_record = tiles[ti].r0; return int(E_OVERFLOW); }
            tile_agg[ti][size_t(s)] = uint32_t(sum);
        }
    }
    if (std::getenv("EMU_TRACE")) std::fprintf(stderr, "emu: %lld fast lanes, %lld precise lanes\n", fast_lanes, precise_lanes);
    // ---- per-chunk scan ----
    std::vector<unsigned long long> chunk_tot(size_t(k) * size_t(S1), 0ull);
    std::vector<std::vector<uint32_t>> tile_base(tiles.size(), std::vector<uint32_t>(size_t(S1), 0));
    for (size_t ti = 0; ti < tiles.size(); ++ti)
        for (int s = 0; s < S; ++s) {
            unsigned long long& tot = chunk_tot[size_t(tiles[ti].chunk) * size_t(S1) + size_t(s)];
            tile_base[ti][size_t(s)] = uint32_t(tot);
            tot += tile_agg[ti][size_t(s)];
            if (tot > 0x7FFFFFFFull) { *err_record = tiles[ti].r0; return int(E_OVERFLOW); }
        }
    // ---- layout + arena ----
    Layout L = compute_layout(plan, n, k, chunk_tot.data());
    auto keep = std::make_shared<Keep>();
    keep->plan = plan_sp;
    keep->arena = static_cast<uint8_t*>(std::calloc(std::max<size_t>(L.total_bytes, 64), 1));
    const int n_slots = int(plan.slots.size());
    std::vector<void*> bufs(size_t(k) * size_t(std::max(n_slots, 1)));
    for (int j = 0; j < k; ++j)
        for (int sl = 0; sl < n_slots; ++sl) bufs[size_t(j) * size_t(n_slots) + size_t(sl)] = keep->arena + L.chunks[size_t(j)].slot_off[size_t(sl)];
    // ---- emit pass ----
    for (size_t ti = 0; ti < tiles.size(); ++ti) {
        const Tile& t = tiles[ti];
        void* const* cb = bufs.data() + size_t(t.chunk) * size_t(n_slots);
        bool wp[kTile / 32];
        uint32_t code = 0;
        (void)count_tile(plan, data, off, t, S, cur, wp, &code, nullptr, nullptr);
        for (int s = 0; s < S; ++s) {  // exclusive scan across lanes + tile base
            uint32_t run = tile_base[ti][size_t(s)];
            for (int lane = 0; lane < kTile; ++lane) { uint32_t v = cur[size_t(s) * kTile + lane]; cur[size_t(s) * kTile + lane] = run; run += v; }
        }
        if (t.local == 0)
            for (const DNode& nd : plan.nodes)
                if (nd.kind == NK_STR || nd.kind == NK_ENUM || nd.kind == NK_LIST || nd.kind == NK_MAP || nd.kind == NK_BYTES) static_cast<int32_t*>(cb[nd.slot_a])[0] = 0;
        const std::vector<uint8_t> window = make_window(data, off, t);
        for (int lane = 0; lane < kTile; ++lane) {
            EmuWalker::Cur q{};
            load_cursors(q, cur.data() + lane, S);
            if (wp[lane / 32]) {  // a warp with a record that is not plain emits with the precise walker
                Ctx c;
                init_ctx(c, plan, data, off, t, lane, cur.data(), S, cb);
                EmuWalker::walk<WM_EMIT>(c, int(plan.nodes.size()), q);
            } else {
                FastCtx f;
                init_fast(f, plan, window, off, t, lane, cur.data(), cb);
                EmuWalker::walk<WM_EMIT>(f, int(plan.nodes.size()), q);
            }
        }
    }
    // ---- null counts ----
    for (int j = 0; j < k; ++j)
        for (int sl : plan.validity_slots) {
            ChunkOut& c = L.chunks[size_t(j)];
            const int64_t bits = c.space_rows[size_t(plan.slots[size_t(sl)].space)];
            const uint8_t* bm = keep->arena + c.slot_off[size_t(sl)];
            int64_t ones = 0;
            for (int64_t i = 0; i < bits; ++i) ones += (bm[i >> 3] >> (i & 7)) & 1;
            c.null_count[size_t(sl)] = bits - ones;
        }
    keep->chunks = L.chunks;
    out.keep = keep;
    return 0;
}

// Host execution of one gather job (what gather_push_kernel does on the device), into a zero-initialised arena.
void apply_job(const GatherJob& j, const uint8_t* src, uint8_t* dst_base) {
    uint8_t* dst = dst_base + j.dst_off;
    if (j.kind == GK_RAW) {
        std::memcpy(dst, src, size_t(j.count));
    } else if (j.kind == GK_OFFSETS) {
        const int32_t* s = reinterpret_cast<const int32_t*>(src);
        int32_t* d = reinterpret_cast<int32_t*>(dst);
        for (int64_t i = 0; i < j.count; ++i) d[1 + i] = s[1 + i] + int32_t(j.param);
    } else {
        for (int64_t i = 0; i < j.count; ++i)
            if ((src[i >> 3] >> (i & 7)) & 1) dst[(j.param + i) >> 3] |= uint8_t(1u << ((j.param + i) & 7));
    }
}
}  // namespace

extern "C" {

// Returns 0 on success; on a data error returns the error code and sets *err_record.
// out_batches must have room for clamp_chunks(num_chunks, n) ArrowArrays.
int emu_decode(const char* json, size_t len, const uint8_t* data, const int64_t* off, int64_t n, int64_t num_chunks,
               ArrowArray* out_batches, ArrowSchema* out_schema, int64_t* k_out, int64_t* err_record, char* msg, size_t msg_cap) {
    try {
        Decoded d;
        const int rc = decode_core(json, len, data, off, n, num_chunks, d, err_record);
        *k_out = d.k;
        if (rc) return rc;
        for (int j = 0; j < d.k; ++j) export_batch(*d.plan, d.keep->chunks[size_t(j)], d.keep->arena, d.keep, &out_batches[j]);
        if (out_schema) export_arrow_schema(d.fields, out_schema);
        return 0;
    } catch (const std::exception& e) {
        std::snprintf(msg, msg_cap, "%s", e.what());
        return -1;
    }
}

// ---- object container files: the product's container reader (ocf.cpp) and its per-block offsets walk (ocf_walk.cuh),
// run for every block in turn with the kernel's error rule (lowest record << 8 | code), then the emulated decode.
// Returns 0, a record error's code (*err_record set), -2 for a malformed container or -1 for anything else (msg set).
int emu_decode_ocf(const uint8_t* file, int64_t len, int64_t num_chunks, ArrowArray* out_batches, ArrowSchema* out_schema,
                   int64_t* k_out, int64_t* err_record, char* msg, size_t msg_cap) {
    OcfIndex ix;
    try {
        ix = ocf_index(file, len);
    } catch (const std::exception& e) {
        std::snprintf(msg, msg_cap, "%s", e.what());
        return -2;
    }
    try {
        auto avro = parse_avro_schema(ix.schema_json.data(), ix.schema_json.size());
        std::string why;
        if (!is_supported(*avro, &why)) throw std::runtime_error("unsupported: " + why);
        const Plan plan = build_plan(*avro, to_arrow_fields(*avro));
        const int64_t n = ix.n_records;
        std::vector<int64_t> off(size_t(n) + 1, ix.end_off);
        std::vector<OcfBlockDev> blocks;
        for (const OcfBlock& b : ix.blocks) blocks.push_back(OcfBlockDev{b.data_off, b.size, b.count, b.rec_base});
        unsigned long long err = ~0ull;
        OcfParams q{};
        q.data = file;
        q.blocks = blocks.data();
        q.n_blocks = int32_t(blocks.size());
        q.nodes = plan.nodes.data();
        q.n_nodes = int32_t(plan.nodes.size());
        q.n_streams = int32_t(plan.streams.size());
        q.sym_off = plan.sym_off.data();
        q.sym_bytes = plan.sym_bytes.data();
        q.offsets = off.data();
        q.n_records = n;
        q.end_off = ix.end_off;
        q.err = &err;
        for (int b = 0; b < q.n_blocks; ++b) ocf_walk_block(q, b);
        if (err != ~0ull) {
            *err_record = int64_t(err >> 8);
            *k_out = 0;
            return int(err & 0xFF);
        }
        Decoded d;
        const int rc = decode_core(ix.schema_json.data(), ix.schema_json.size(), file, off.data(), n, num_chunks, d, err_record);
        *k_out = d.k;
        if (rc) return rc;
        for (int j = 0; j < d.k; ++j) export_batch(*d.plan, d.keep->chunks[size_t(j)], d.keep->arena, d.keep, &out_batches[j]);
        if (out_schema) export_arrow_schema(d.fields, out_schema);
        return 0;
    } catch (const std::exception& e) {
        std::snprintf(msg, msg_cap, "%s", e.what());
        return -1;
    }
}

// ---- multi-rank gather on the host: the product's plan (gather.cpp), the kernel's job semantics restated ------------
// A decoded shard (one batch) kept for the gather steps.
void* emu_shard_decode(const char* json, size_t len, const uint8_t* data, const int64_t* off, int64_t n, char* msg, size_t msg_cap) {
    try {
        auto d = std::make_unique<Decoded>();
        int64_t rec = -1;
        if (decode_core(json, len, data, off, n, 1, *d, &rec) != 0) throw std::runtime_error("decode error in shard");
        return d.release();
    } catch (const std::exception& e) {
        std::snprintf(msg, msg_cap, "%s", e.what());
        return nullptr;
    }
}
void emu_shard_free(void* h) { delete static_cast<Decoded*>(h); }
int64_t emu_meta_len(void* h) { return gather_meta_len(*static_cast<Decoded*>(h)->plan); }
void emu_shard_meta(void* h, int64_t* out) {
    auto* d = static_cast<Decoded*>(h);
    gather_meta_of(*d->plan, d->keep->chunks[0], out);
}
// out[0] = groups; then per group: first rank, ranks, arena bytes, rows
int emu_gather_groups(void* h, const int64_t* metas, int world, int64_t* out, int cap) {
    auto* d = static_cast<Decoded*>(h);
    GatherPlan gp = plan_gather(*d->plan, metas, world);
    out[0] = int64_t(gp.groups.size());
    for (size_t i = 0; i < gp.groups.size() && int(1 + 4 * (i + 1)) <= cap; ++i) {
        out[1 + 4 * i] = gp.groups[i].first_rank; out[2 + 4 * i] = gp.groups[i].n_ranks;
        out[3 + 4 * i] = int64_t(gp.groups[i].arena_bytes); out[4 + 4 * i] = gp.groups[i].out.rows;
    }
    return 0;
}
// Applies `rank`'s jobs into `arena` (the arena of the rank's group, zero-initialised by the caller).
int emu_gather_apply(void* h, const int64_t* metas, int world, int rank, uint8_t* arena) {
    auto* d = static_cast<Decoded*>(h);
    GatherPlan gp = plan_gather(*d->plan, metas, world);
    const GatherGroup& g = gp.groups[size_t(gp.group_of_rank[size_t(rank)])];
    const ChunkOut& mine = d->keep->chunks[0];
    for (const GatherJob& j : g.jobs[size_t(rank - g.first_rank)]) apply_job(j, d->keep->arena + mine.slot_off[size_t(j.slot)], arena);
    return 0;
}
// Exports the gathered batch of `group` from a finished arena (copied).
int emu_gather_export(void* h, const int64_t* metas, int world, int group, const uint8_t* arena, ArrowArray* out, ArrowSchema* out_schema) {
    auto* d = static_cast<Decoded*>(h);
    GatherPlan gp = plan_gather(*d->plan, metas, world);
    const GatherGroup& g = gp.groups[size_t(group)];
    auto keep = std::make_shared<Keep>();
    keep->plan = d->plan;
    keep->arena = static_cast<uint8_t*>(std::malloc(std::max<size_t>(g.arena_bytes, 64)));
    std::memcpy(keep->arena, arena, g.arena_bytes);
    keep->chunks = {g.out};
    export_batch(*d->plan, keep->chunks[0], keep->arena, keep, out);
    if (out_schema) export_arrow_schema(d->fields, out_schema);
    return 0;
}

}  // extern "C"
