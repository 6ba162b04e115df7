// Kernel body of the decode: ONE fused pass per kBlock-record tile (256; 384 for generated walkers of plans with more
// than eight streams, engine.cu choose_tile), templated over the walker (InterpWalker or a generated,
// schema-specialised walker).  Device-only; compiled by nvcc (kernels.cu) and by NVRTC (jit.cpp).
//
//   fused_body  one CTA per tile, tiles taken in blockIdx order:
//     1. one TMA bulk copy (cp.async.bulk + mbarrier) stages the tile's contiguous byte window in shared memory;
//     2. every lane COUNT-walks its record (full validation) -> per-stream counts;
//     3. a warp-per-stream scan turns the lane counts into in-tile prefixes and the tile's totals;
//     4. the totals are chained across tiles with a decoupled look-back (Merrill & Garland): each (stream, tile) has a
//        64-bit status word {flag, value} in global memory; a tile publishes its aggregate, sums its predecessors'
//        aggregates back to the nearest published inclusive prefix, then publishes its own inclusive prefix.  Every
//        output batch (chunk) is its own chain, so Arrow offsets restart at 0 per batch;
//     5. the same CTA EMIT-walks the still-resident window: fixed-width values / offsets are stored row-aligned,
//        space-0 validity is one ballot word per warp, Utf8 bytes are assembled per column in a shared-memory staging
//        area and leave through TMA bulk stores (16-byte aligned body) plus a few head/tail bytes.
//   The input is read from HBM once and nothing but the Arrow buffers (and 8 bytes per stream per tile of scan
//   status) is written.
//
//   Output capacity.  Buffers whose size depends on the data (string bytes, list child rows) are sized by the host
//   from what earlier calls on the same schema needed (p.caps); a tile whose range would not fit raises CW_OVER,
//   skips its emit and still publishes, so the pass ends with exact totals and the host repeats it once with an
//   exact-size arena.  p.count_only (the first call on a schema) skips every emit.
//
// Shared-memory map (dynamic, rv_smem; smem_map() in dev_types.h):
//   [nodes n_nodes*32][ttot (S+1)*4][tbase S*4][adj S*4][flags 16][mbar 8][ptrs n_slots*8][item positions (generated walkers)]
//   [cur S*256*4 (interpreter)]
//   [in: smem_data_cap + pad][stage: smem_stage_cap]        (register-cursor walkers: the scan area overlays `stage`)
#pragma once
#include "dev_core.cuh"

namespace rv {

struct Tile {
    int chunk;
    int local_tile;
    int lin;             // chunk * tiles_per_chunk + local_tile: index of the tile's scan status words
    int64_t r0;          // first record of the tile
    int nrec;            // records in the tile
    int64_t chunk_len;   // rows in the chunk
};

// blockIdx -> tile.  CTAs are dispatched in blockIdx order and every chunk (output batch) is its own look-back
// chain, so consecutive CTAs take tiles of DIFFERENT chunks (id = local * k + chunk): the k chains advance side by
// side instead of one after the other, which multiplies the rate at which prefixes become known and divides how many
// running predecessors a tile can be held up by.  (The last chunk is the longest — it takes the remainder rows — and
// its surplus tiles come last.)
__device__ __forceinline__ Tile tile_of(const DecodeParams& p, int id) {
    Tile t;
    int j = 0, local = id;
    if (p.k > 1) {
        const int body = p.k * p.tiles_per_chunk;
        if (id < body) {  // id / k without the ~40-instruction integer division: estimate and correct
            local = int(__fdividef(float(id), float(p.k)));
            while (local > 0 && local * p.k > id) --local;
            while ((local + 1) * p.k <= id) ++local;
            j = id - local * p.k;
        } else {
            j = p.k - 1;
            local = p.tiles_per_chunk + (id - body);
        }
    }
    t.chunk = j;
    t.local_tile = local;
    t.lin = j * p.tiles_per_chunk + local;
    const int64_t cs = int64_t(j) * p.chunk_rows;
    const int64_t ce = (j == p.k - 1) ? p.n : cs + p.chunk_rows;
    t.chunk_len = ce - cs;
    t.r0 = cs + int64_t(t.local_tile) * kBlock;
    const int64_t left = ce - t.r0;
    t.nrec = left < kBlock ? int(left) : kBlock;
    return t;
}

struct TileWindow {
    bool staged;
    bool tma;         // the window is in flight on the copy engine: wait_window() before reading it
    int64_t t0, t1;   // byte range of the tile in `data`
    uint32_t mis;     // (data + t0) & 15: the window starts at the aligned-down address
    int64_t o0, o1;   // this lane's record: byte range in `data`
    int64_t f0, f1;   // (one lane) byte range of the tile `prefetch_dist` ahead, -1: none
};

// L2 prefetch: a CTA's first act is a dependent chain of DRAM round trips (offsets -> input window);
// the CTA that ran `prefetch_dist` tiles earlier has already pulled those lines into L2.
__device__ __forceinline__ void l2_prefetch_line(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
__device__ __forceinline__ void l2_prefetch_bulk(const void* p, uint32_t bytes) {
    asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
constexpr int kPrefetchLane = 32;  // the lane (first of warp 1) that carries the look-ahead

// ---- TMA (bulk async copy) staging of the input window -----------------------------------------------
// One thread hands the whole window to the copy engine (cp.async.bulk global -> shared, completion counted in
// bytes on an mbarrier) instead of every thread moving its share through registers (LDG.128 + STS.128).
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint32_t mbar, uint32_t arrivals) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(arrivals) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");  // visible to the async proxy
}
__device__ __forceinline__ void bulk_load(uint32_t dst, const void* src, uint32_t bytes, uint32_t mbar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst), "l"(src), "r"(bytes), "r"(mbar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t mbar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred P1;\n"
        "RV_WAIT:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n"
        "@P1 bra RV_DONE;\n"
        "bra RV_WAIT;\n"
        "RV_DONE:\n"
        "}" ::"r"(mbar), "r"(parity) : "memory");
}

// ---- scan status words (decoupled look-back) -----------------------------------------------------------
// {flag:2, value:62} in one 64-bit word, written and read with single relaxed gpu-scope accesses: flag and
// value can never be seen torn, so no fences are needed around them.
constexpr unsigned long long kStAgg = 1ull << 62;      // value = this tile's total
constexpr unsigned long long kStPrefix = 2ull << 62;   // value = total of this tile and every earlier tile of the chunk
constexpr unsigned long long kStMask = (1ull << 62) - 1ull;

__device__ __forceinline__ unsigned long long ld_state(const unsigned long long* p) {
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_state(unsigned long long* p, unsigned long long v) {
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}

// Whole warp: the sum of the totals of tiles [first, tile) of one stream.  Lane l inspects tile (t - l); the warp
// walks back 32 tiles at a time until it meets a published inclusive prefix (tiles before `first` count as one).
__device__ __forceinline__ unsigned long long look_back(const unsigned long long* st, const int tile, const int first) {
    const int lane = threadIdx.x & 31;
    unsigned long long excl = 0;
    int t = tile - 1;
    for (;;) {
        const int mine = t - lane;
        const bool real = mine >= first;  // tiles before the chain count as one virtual tile with inclusive prefix 0
        unsigned long long v;
        do { v = real ? ld_state(st + mine) : kStPrefix; } while (__any_sync(0xFFFFFFFFu, (v >> 62) == 0ull));
        const unsigned has = __ballot_sync(0xFFFFFFFFu, (v >> 62) == 2ull);
        const int pl = has ? __ffs(int(has)) - 1 : 32;  // nearest tile that already knows its prefix
        unsigned long long c = lane <= pl ? (v & kStMask) : 0ull;
#pragma unroll
        for (int d = 16; d; d >>= 1) c += __shfl_xor_sync(0xFFFFFFFFu, c, d);
        excl += c;
        if (has) break;
        t -= 32;
    }
    return excl;
}

// Loads the plan and the tile's byte window into shared memory.
template <class W>
__device__ __forceinline__ TileWindow stage_in(const DecodeParams& p, const Tile& t, const int tile_id, const SmemMap& m) {
    const int tid = threadIdx.x;
    if (tid == 0) mbar_init(smem_addr(rv_smem + m.mbar), 1);
    if (p.n_nodes) {
        uint4* dn = reinterpret_cast<uint4*>(rv_smem + m.nodes);
        for (int i = tid; i < p.n_nodes * 2; i += kBlock) dn[i] = __ldg(reinterpret_cast<const uint4*>(p.nodes) + i);
    }
    if (p.bufs) {  // this chunk's Arrow buffer pointers (see buf_ptr)
        void** sp = reinterpret_cast<void**>(rv_smem + m.ptrs);
        void* const* gp = p.bufs + size_t(t.chunk) * p.n_slots;
        for (int i = tid; i < p.n_slots; i += kBlock) sp[i] = gp[i];
    }
    if constexpr (!W::kRegCursors) {
        uint32_t* cur = reinterpret_cast<uint32_t*>(rv_smem + m.cur);
        for (int s = 0; s < p.n_streams; ++s) cur[s * kBlock + tid] = 0;
    }
    if (tid == 0) *reinterpret_cast<uint32_t*>(rv_smem + m.flags) = 0u;
    TileWindow w;
    // One round trip: the tile's bounds, this lane's record bounds and (one lane) the bounds of the tile a
    // later CTA will work on are all requested before anything waits.
    w.t0 = __ldg(p.offsets + t.r0);
    w.t1 = __ldg(p.offsets + t.r0 + t.nrec);
    w.o0 = w.o1 = 0;
    if (tid < t.nrec) {
        w.o0 = __ldg(p.offsets + t.r0 + tid);
        w.o1 = __ldg(p.offsets + t.r0 + tid + 1);
    }
    w.f0 = w.f1 = -1;
    const int64_t ft = int64_t(tile_id) + p.prefetch_dist;
    if (p.prefetch_dist > 0 && ft < p.n_tiles) {
        const Tile f = tile_of(p, int(ft));
        // the kBlock * 8 (+8) bytes of offsets of that tile: kBlock / 16 + 1 lines of 128 bytes
        if (tid <= kBlock / 16 && f.r0 + 16 * tid <= p.n) l2_prefetch_line(p.offsets + f.r0 + 16 * tid);
        if (tid == kPrefetchLane) {
            w.f0 = __ldg(p.offsets + f.r0);
            w.f1 = __ldg(p.offsets + f.r0 + f.nrec);
        }
    }
    const int64_t span = w.t1 - w.t0;
    w.mis = uint32_t(reinterpret_cast<uintptr_t>(p.data + w.t0) & 15u);
    w.staged = span >= 0 && uint64_t(span) + w.mis <= uint64_t(p.smem_data_cap);
    w.tma = false;
    if (w.staged) {
        // (the last vector may read up to 15 bytes past offsets[n]: rv_decode_device documents the padding)
        const uint4* g = reinterpret_cast<const uint4*>(p.data + w.t0 - w.mis);
        const int nvec = int((span + w.mis + 15) >> 4);
        w.tma = nvec > 0;
        if (w.tma && tid == 0) bulk_load(smem_addr(rv_smem + m.in), g, uint32_t(nvec) << 4, smem_addr(rv_smem + m.mbar));
    }
    if (tid == 0) {  // window sizing of later calls: the largest tile seen, the input's byte span
        if (span > 0 && static_cast<unsigned long long>(span) > p.ctrl[CW_MAX_SPAN]) atomicMax(p.ctrl + CW_MAX_SPAN, static_cast<unsigned long long>(span));
        if (t.lin == 0) p.ctrl[CW_IN_FIRST] = static_cast<unsigned long long>(w.t0);
        if (t.lin == p.n_tiles - 1) p.ctrl[CW_IN_LAST] = static_cast<unsigned long long>(w.t1);
    }
    return w;
}

// After the CTA barrier that follows stage_in (which also publishes the mbarrier's initialisation).
__device__ __forceinline__ void wait_window(const TileWindow& w, const SmemMap& m) {
    if (w.tma) mbar_wait(smem_addr(rv_smem + m.mbar), 0);
}

template <class C>
__device__ __forceinline__ int64_t init_ctx(C& c, const DecodeParams& p, const Tile& t, const SmemMap& m, const TileWindow& w) {
    const int tid = threadIdx.x;
    const uint32_t s0 = smem_addr(rv_smem);
    c.nodes = reinterpret_cast<const DNode*>(rv_smem + m.nodes);
    c.cur = reinterpret_cast<uint32_t*>(rv_smem + m.cur) + tid;
    c.cur_stride = kBlock;
    c.sym_off = p.sym_off;
    c.sym_bytes = p.sym_bytes;
    c.bufs = p.bufs ? p.bufs + size_t(t.chunk) * p.n_slots : nullptr;
    c.ptrs_saddr = p.bufs ? s0 + m.ptrs : 0u;
    c.err = 0;
    c.pm = 0;
    c.usel = 0;
    c.stage_on = false;
    c.stage_saddr = s0 + m.stage;
    c.adj_saddr = s0 + m.adj;
    c.items_saddr = s0 + m.items;
    c.in_range = tid < t.nrec;
    c.row0 = uint32_t(t.local_tile) * kBlock + tid;
    c.store_word = (tid & 31) == 0 && int64_t(c.row0) < t.chunk_len;
    c.base = p.data;
    c.sbase = s0 + m.in;
    c.pos = c.end = 0;
    const int64_t r = t.r0 + tid;
    if (c.in_range) {
        const int64_t o0 = w.o0, o1 = w.o1;
        if (o1 < o0 || o1 - o0 > int64_t(0xFFFFFFF0u)) c.err = E_OVERFLOW;  // malformed offsets / >4 GiB record
        else if (C::kShared) {
            if (o0 < w.t0 || o1 > w.t1) c.err = E_OVERFLOW;
            else { c.pos = uint32_t(o0 - w.t0) + w.mis; c.end = uint32_t(o1 - w.t0) + w.mis; }
        } else {
            c.base = p.data + o0;
            c.end = uint32_t(o1 - o0);
        }
        if (p.frame_skip && !c.err) {  // framed input: the datum starts behind the message's header
            if (c.end - c.pos < p.frame_skip) c.err = E_FRAME;
            else {
                if (p.frame_check == kFrameSingleObject) {
                    unsigned long long fp = 0;
                    for (uint32_t b = 0; b < 8; ++b) fp |= static_cast<unsigned long long>(ld_u8(c, c.pos + 2 + b)) << (8 * b);
                    if (ld_u8(c, c.pos) != 0xC3u || ld_u8(c, c.pos + 1) != 0x01u || fp != p.frame_fp) c.err = E_FRAME;
                } else if (p.frame_check) {
                    const uint32_t id = (ld_u8(c, c.pos + 1) << 24) | (ld_u8(c, c.pos + 2) << 16) | (ld_u8(c, c.pos + 3) << 8) | ld_u8(c, c.pos + 4);
                    if (ld_u8(c, c.pos) != 0u || (p.frame_check == 2 && id != p.frame_id)) c.err = E_FRAME;
                }
                c.pos += p.frame_skip;
            }
        }
    }
    return r;
}

__device__ __forceinline__ void report(const DecodeParams& p, int64_t record, uint32_t code) {
    atomicMin(p.ctrl + CW_ERR, (static_cast<unsigned long long>(record) << 8) | code);
}

// The look-ahead lane asks L2 for the input window of the tile `prefetch_dist` ahead (its bounds arrived
// long ago, with this tile's own offsets).
__device__ __forceinline__ void prefetch_window(const DecodeParams& p, const TileWindow& w) {
    if (threadIdx.x == kPrefetchLane && w.f0 >= 0 && w.f1 > w.f0 && w.f1 - w.f0 < (int64_t(1) << 20)) {
        const uintptr_t a = reinterpret_cast<uintptr_t>(p.data + w.f0) & ~uintptr_t(15);
        const uintptr_t e = (reinterpret_cast<uintptr_t>(p.data + w.f1) + 15) & ~uintptr_t(15);
        l2_prefetch_bulk(reinterpret_cast<const void*>(a), uint32_t(e - a));
    }
}

// ---- count ----------------------------------------------------------------------------------
// SM = true, the FAST flavour: returns != 0 when the record is not plain (dev_core.cuh) and reports nothing — the
// caller repeats the record with the precise flavour.  SM = false, PRECISE: reports the record's first error and
// returns its code.
template <class W, bool SM, bool PERM = false>
__device__ __forceinline__ uint32_t count_walk(const DecodeParams& p, const Tile& t, const SmemMap& m, const TileWindow& w, typename W::Cur& q) {
    WalkCtx<SM> c;
    const int64_t r = init_ctx(c, p, t, m, w);
    if constexpr (W::kRegCursors) {
#pragma unroll
        for (int s = 0; s < W::kStreams; ++s) q.v[s] = 0;
    } else {
        if (!SM) for (int s = 0; s < p.n_streams; ++s) c.cur[s * kBlock] = 0;  // (a fast walk may have left partial counts)
    }
#if !defined(RV_ABL_NOCOUNTWALK)
    W::template walk<WM_COUNT>(c, p.n_nodes, q);
#endif
    if (!SM && c.in_range && c.err && !(PERM && record_error(c.err))) report(p, r, c.err);
    return c.in_range ? c.err : 0u;
}
// Everything by value: a reference parameter of a function that is not inlined would force the caller's copy (the
// kernel parameters, the cursors) out of registers into local memory for the whole kernel.
template <class W>
struct CountOut { typename W::Cur q; uint32_t err; };
template <class W>
__device__ __noinline__ CountOut<W> count_walk_global(const DecodeParams p, const Tile t, const SmemMap m, const TileWindow w) {
    CountOut<W> o;
    o.err = count_walk<W, false>(p, t, m, w, o.q);
    return o;
}
// Permissive decodes: the same, except that a record error (record_error) is left to the caller instead of reported.
template <class W>
__device__ __noinline__ CountOut<W> count_walk_global_perm(const DecodeParams p, const Tile t, const SmemMap m, const TileWindow w) {
    CountOut<W> o;
    o.err = count_walk<W, false, true>(p, t, m, w, o.q);
    return o;
}

template <class W, bool PERM>
__device__ __forceinline__ CountOut<W> count_precise(const DecodeParams& p, const Tile& t, const SmemMap& m, const TileWindow& w) {
    if constexpr (PERM) return count_walk_global_perm<W>(p, t, m, w);
    else return count_walk_global<W>(p, t, m, w);
}

// ---- emit: staging map ------------------------------------------------------------------------
// Stream s's Utf8 bytes of this tile occupy [tbase, tbase + ttot) of its Arrow data buffer; in shared memory its
// region starts at a 16-byte boundary plus the destination's misalignment, so the write-out can use aligned 16-byte
// pieces.  Warp 0 computes the map with a shuffle scan once the look-back delivered the tile's bases.
// flags bit 1 <- the tile's strings fit the staging area.
__device__ __forceinline__ void stage_map(const DecodeParams& p, const Tile& t, const SmemMap& m) {
    const uint32_t* tbase = reinterpret_cast<const uint32_t*>(rv_smem + m.tbase);
    const uint32_t* ttot = reinterpret_cast<const uint32_t*>(rv_smem + m.ttot);
    uint32_t* adj = reinterpret_cast<uint32_t*>(rv_smem + m.adj);
    const int lane = threadIdx.x & 31;
    uint32_t carry = 0;
    for (int s0 = 0; s0 < p.n_streams; s0 += 32) {
        const int s = s0 + lane;
        uint32_t tb = 0, ga = 0, region = 0;
        int slot = -1;
        if (s < p.n_streams) {
            tb = tbase[s];
            slot = p.stream_slot[s];
            if (slot >= 0) {
                const uint8_t* b = *reinterpret_cast<uint8_t* const*>(rv_smem + m.ptrs + uint32_t(slot) * 8u);
                ga = uint32_t(reinterpret_cast<uintptr_t>(b + tb) & 15u);
                region = (ttot[s] + ga + 15u) & ~15u;
            }
        }
        uint32_t incl = region;
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, d);
            if (lane >= d) incl += u;
        }
        if (s < p.n_streams) adj[s] = slot >= 0 ? (carry + incl - region + ga) - tb : 0u;  // staging offset of chunk-relative byte o = adj + o
        carry += __shfl_sync(0xFFFFFFFFu, incl, 31);
    }
    if (lane == 0 && (p.n_utf8 == 0 || (p.smem_stage_cap > 0 && carry <= p.smem_stage_cap))) atomicOr(reinterpret_cast<uint32_t*>(rv_smem + m.flags), 2u);
    (void)t;
}

// ---- emit -----------------------------------------------------------------------------------
template <class W, bool SM>
__device__ __forceinline__ void emit_walk(const DecodeParams& p, const Tile& t, const SmemMap& m, const TileWindow& w, typename W::Cur& q, const bool stage_on,
                                          const uint32_t bad = 0u) {
    WalkCtx<SM> c;
    (void)init_ctx(c, p, t, m, w);
    c.stage_on = stage_on;
    // permissive decodes: the count walk's verdict on a bad record.  Its row is emitted absent -- the walkers' top-level
    // presence is false while c.err is set (interp.cuh; the permissive generated walker's vtop) -- and reads nothing.
    if (bad) c.err = bad;
    const int tid = threadIdx.x;
    // offsets[0] = 0 of every offsets buffer of this chunk (first tile of the chunk only)
    if (t.local_tile == 0) {
        if (p.n_nodes) {
            for (int i = tid & 31; i < p.n_nodes; i += 32) {  // (every warp: a warp may be alone on the precise path)
                const DNode nd = c.nodes[i];
                if (nd.flags & NF_SKIP) continue;  // owns no buffers
                if (nd.kind == NK_STR || nd.kind == NK_ENUM || nd.kind == NK_LIST || nd.kind == NK_MAP || nd.kind == NK_BYTES ||
                    (nd.kind == NK_DEFAULT && nd.pad0 == NK_STR))
                    static_cast<int32_t*>(buf_ptr(c, nd.slot_a))[0] = 0;
            }
        } else {
            W::zero_offsets(c, tid & 31);
        }
    }
#if !defined(RV_ABL_NOWALK)
    W::template walk<WM_EMIT>(c, p.n_nodes, q);
#endif
}
template <class W>
__device__ __noinline__ void emit_walk_global(const DecodeParams p, const Tile t, const SmemMap m, const TileWindow w, typename W::Cur q, const bool stage_on) {
    emit_walk<W, false>(p, t, m, w, q, stage_on);
}
template <class W>
__device__ __noinline__ void emit_walk_global_perm(const DecodeParams p, const Tile t, const SmemMap m, const TileWindow w, typename W::Cur q, const bool stage_on,
                                                   const uint32_t bad) {
    emit_walk<W, false>(p, t, m, w, q, stage_on, bad);
}

template <class W, bool PERM>
__device__ __forceinline__ void emit_precise(const DecodeParams& p, const Tile& t, const SmemMap& m, const TileWindow& w, typename W::Cur& q, const bool stage_on,
                                             const uint32_t bad) {
    if constexpr (PERM) emit_walk_global_perm<W>(p, t, m, w, q, stage_on, bad);
    else { (void)bad; emit_walk_global<W>(p, t, m, w, q, stage_on); }
}

// Coalesced write-out of the staged Utf8 bytes, one warp per stream at a time.
__device__ __forceinline__ void stage_write_out(const DecodeParams& p, const SmemMap& m) {
    const uint32_t* tbase = reinterpret_cast<const uint32_t*>(rv_smem + m.tbase);
    const uint32_t* ttot = reinterpret_cast<const uint32_t*>(rv_smem + m.ttot);
    const uint32_t* adj = reinterpret_cast<const uint32_t*>(rv_smem + m.adj);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // staged bytes -> visible to the copy engine
    __syncthreads();
    for (int s = warp; s < p.n_streams; s += kWarps) {
        const int slot = p.stream_slot[s];
        const uint32_t n = ttot[s];
        if (slot < 0 || n == 0) continue;
        const uint32_t tb = tbase[s];
        uint8_t* g = *reinterpret_cast<uint8_t* const*>(rv_smem + m.ptrs + uint32_t(slot) * 8u) + tb;
        const uint32_t so = m.stage + adj[s] + tb;  // rv_smem offset of the region's first byte
        const uint32_t head = min(n, (16u - uint32_t(reinterpret_cast<uintptr_t>(g) & 15u)) & 15u);
        for (uint32_t i = lane; i < head; i += 32) g[i] = rv_smem[so + i];
        const uint32_t nvec = (n - head) >> 4;
        // the 16-byte aligned body leaves through the copy engine (shared -> global bulk store): one
        // instruction per column instead of a store loop, and the warp does not wait for the data to drain
        if (lane == 0 && nvec > 0)
            asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
                         ::"l"(g + head), "r"(smem_addr(rv_smem + so + head)), "r"(nvec << 4) : "memory");
        const uint32_t done = head + (nvec << 4);
        for (uint32_t i = done + lane; i < n; i += 32) g[i] = rv_smem[so + i];
    }
    if (lane == 0) {  // shared memory must outlive the engine's reads
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    }
}

// ---- the fused pass ---------------------------------------------------------------------------
// PERM (permissive decodes, rv_schema_permissive): a record with a record error (record_error) does not fail the call.
// Its lane counts nothing, appends (record << 8 | code) to the bad-record list (bad_list_word) and emits its row absent
// on the precise path; only the other codes (E_OVERFLOW, E_SCHEMA) are reported to CW_ERR and end the CTA's work.
template <class W, bool PERM = false>
__device__ __forceinline__ void fused_body(const DecodeParams& p, const int tile_id) {
    const Tile t = tile_of(p, tile_id);
    const SmemMap m = smem_map(p.n_nodes, p.n_streams, p.n_slots, p.smem_data_cap, p.smem_stage_cap, W::kRegCursors, W::kItemBytes);
    typename W::Cur q;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const TileWindow w = stage_in<W>(p, t, tile_id, m);
    __syncthreads();
    wait_window(w, m);

    // ---- COUNT: validation + what this record adds to every stream.  Records that are not plain (non-canonical
    // encodings, or malformed) are repeated by their lane with the precise walker, which settles what they are; their
    // warp then also emits with the precise walker.
    uint32_t my_err;
    bool warp_precise = false;
    if (w.staged) {
        my_err = count_walk<W, true>(p, t, m, w, q);
        const bool not_plain = my_err != 0u;
        if (not_plain) {
            const CountOut<W> o = count_precise<W, PERM>(p, t, m, w);
            q = o.q;
            my_err = o.err;
        }
        warp_precise = __any_sync(0xFFFFFFFFu, not_plain);
    } else {
        const CountOut<W> o = count_precise<W, PERM>(p, t, m, w);
        q = o.q;
        my_err = o.err;
    }
    // A bad record (always settled by the precise walk above, so its warp emits with the precise walker too) counts
    // nothing and is listed.  Every pass lists afresh: the host clears CW_BAD with the rest of the control block.
    uint32_t bad = 0u;
    if constexpr (PERM) {
        if (my_err != 0u && record_error(my_err)) {
            bad = my_err;
            my_err = 0u;
            if constexpr (W::kRegCursors) {
#pragma unroll
                for (int s = 0; s < W::kStreams; ++s) q.v[s] = 0;
            } else {
                uint32_t* cz = reinterpret_cast<uint32_t*>(rv_smem + m.cur);
                for (int s = 0; s < p.n_streams; ++s) cz[s * kBlock + tid] = 0;
            }
            const unsigned long long* lw = p.ctrl + bad_list_word(p.k, p.n_streams);
            const unsigned long long i = atomicAdd(p.ctrl + CW_BAD, 1ull);
            if (i < lw[1]) reinterpret_cast<unsigned long long*>(lw[0])[i] = (static_cast<unsigned long long>(t.r0 + tid) << 8) | bad;
        }
    }

    // ---- CTA-wide exclusive scan of every stream's lane counts.  One WARP scans one stream: each lane takes kBlock / 32
    // consecutive records (8 or 12: two or three 128-bit loads), sums them serially, and a single 5-step shuffle scan
    // joins the 32 lane totals.  (384-row tiles give a plan of up to twelve streams one stream per warp.)
    constexpr int kPerLane = kBlock / 32;  // 4, 8, 12, ...: a multiple of 4, so every lane moves whole uint4
    uint32_t* cur = reinterpret_cast<uint32_t*>(rv_smem + m.cur);
    uint32_t* ttot = reinterpret_cast<uint32_t*>(rv_smem + m.ttot);
    uint32_t* tbase = reinterpret_cast<uint32_t*>(rv_smem + m.tbase);
    uint32_t* flags = reinterpret_cast<uint32_t*>(rv_smem + m.flags);
    if constexpr (W::kRegCursors) {  // the scan area overlays the (still unused) Utf8 staging area
#pragma unroll
        for (int s = 0; s < W::kStreams; ++s) cur[s * kBlock + tid] = q.v[s];
    }
    const bool any_err = __syncthreads_or(my_err != 0u) != 0;
    for (int s = warp; s < p.n_streams; s += kWarps) {
        uint32_t* cl = cur + s * kBlock + lane * kPerLane;
        uint32_t v[kPerLane];
        uint32_t any = 0;
        if constexpr (kPerLane % 4 == 0) {
#pragma unroll
            for (int i = 0; i < kPerLane; i += 4) {
                const uint4 x = *reinterpret_cast<const uint4*>(cl + i);
                v[i] = x.x; v[i + 1] = x.y; v[i + 2] = x.z; v[i + 3] = x.w;
                any |= x.x | x.y | x.z | x.w;
            }
        } else {
#pragma unroll
            for (int i = 0; i < kPerLane; ++i) { v[i] = cl[i]; any |= v[i]; }
        }
        uint32_t tile_total;
        // kBlock values below 2^31 / kBlock cannot overflow 31 bits; anything bigger (a tile of huge zero-width
        // lists) takes the exact 64-bit path below
        if (__any_sync(0xFFFFFFFFu, any >= (0x80000000u / uint32_t(kBlock)))) {
            unsigned long long run = 0;
            if (lane == 0) {
                uint32_t* cs = cur + s * kBlock;
                for (int i = 0; i < kBlock; ++i) {
                    const uint32_t x = cs[i];
                    cs[i] = uint32_t(run);
                    run += x;
                }
                if (run > 0x7FFFFFFFull) { report(p, t.r0, E_OVERFLOW); run = 0x7FFFFFFFull; }
            }
            __syncwarp();
            tile_total = __shfl_sync(0xFFFFFFFFu, uint32_t(run), 0);
        } else {
            uint32_t tot = 0;
#pragma unroll
            for (int i = 0; i < kPerLane; ++i) {  // lane-local exclusive prefix
                const uint32_t x = v[i];
                v[i] = tot;
                tot += x;
            }
            uint32_t incl = tot;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) {
                const uint32_t u = __shfl_up_sync(0xFFFFFFFFu, incl, d);
                if (lane >= d) incl += u;
            }
            const uint32_t base = incl - tot;
            if constexpr (kPerLane % 4 == 0) {
#pragma unroll
                for (int i = 0; i < kPerLane; i += 4)
                    *reinterpret_cast<uint4*>(cl + i) = make_uint4(base + v[i], base + v[i + 1], base + v[i + 2], base + v[i + 3]);
            } else {
#pragma unroll
                for (int i = 0; i < kPerLane; ++i) cl[i] = base + v[i];
            }
            tile_total = __shfl_sync(0xFFFFFFFFu, incl, 31);  // < 2^31 by construction
        }
        // publish right away: the successors' look-backs are waiting for it
        if (lane == 0) {
            ttot[s] = tile_total;
            st_state(p.tile_state + size_t(s) * p.n_tiles + t.lin, (t.local_tile == 0 ? kStPrefix : kStAgg) | tile_total);
        }
    }
    __syncwarp();  // lane 0's ttot[s] stores above are read by the whole warp below
    // ---- chain the tile totals: exclusive prefix within the chunk
    for (int s = warp; s < p.n_streams; s += kWarps) {
        unsigned long long base = 0;
        const uint32_t tot = ttot[s];
        if (t.local_tile != 0) {
            unsigned long long* st = p.tile_state + size_t(s) * p.n_tiles;
#if !defined(RV_ABL_NOLOOKBACK)
            base = look_back(st, t.lin, t.lin - t.local_tile);
#endif
            if (lane == 0) st_state(st + t.lin, kStPrefix | ((base + tot) & kStMask));
        }
        if (lane == 0) {
            const unsigned long long incl = base + tot;
            const bool last = int64_t(t.local_tile + 1) * kBlock >= t.chunk_len;
            if (last) {
                p.ctrl[CW_CHUNK_TOT + size_t(t.chunk) * p.n_streams + s] = incl;
                if (incl > 0x7FFFFFFFull) report(p, int64_t(t.chunk) * p.chunk_rows, E_OVERFLOW);
            }
            const unsigned long long cap = p.caps ? static_cast<unsigned long long>(p.caps[size_t(t.chunk) * p.n_streams + s]) : 0ull;
            if (incl > cap && !p.count_only) {  // this tile's range does not fit the buffer the host sized: exact totals, then a repeat
                atomicOr(flags, 1u);
                if (p.ctrl[CW_OVER] == 0ull) atomicMax(p.ctrl + CW_OVER, 1ull);
            }
            tbase[s] = uint32_t(base > 0x7FFFFFFFull ? 0x7FFFFFFFull : base);
        }
    }
    __syncthreads();
    if (warp == 0 && p.n_utf8 > 0) {  // staging need of this tile (upper bound: 31 bytes of alignment per column)
        uint32_t need = 0;
        for (int s = lane; s < p.n_streams; s += 32)
            if (p.stream_slot[s] >= 0) need += ttot[s] + 31u;
#pragma unroll
        for (int d = 16; d; d >>= 1) need += __shfl_xor_sync(0xFFFFFFFFu, need, d);
        if (lane == 0 && static_cast<unsigned long long>(need) > p.ctrl[CW_MAX_UTF8]) atomicMax(p.ctrl + CW_MAX_UTF8, static_cast<unsigned long long>(need));
    }
    if (p.count_only || any_err || (flags[0] & 1u)) return;  // uniform: the whole CTA leaves

    // ---- cursors: tile base + in-tile prefix; staging map (warp 0) while the rest zero the staging area
    if constexpr (W::kRegCursors) {
#pragma unroll
        for (int s = 0; s < W::kStreams; ++s) q.v[s] = cur[s * kBlock + tid] + tbase[s];
    } else {
        for (int s = 0; s < p.n_streams; ++s) cur[s * kBlock + tid] += tbase[s];
    }
    if constexpr (W::kRegCursors) __syncthreads();  // every lane read its prefixes: the staging area may be overwritten
    if (warp == 0) stage_map(p, t, m);
    if (w.staged && p.n_utf8 > 0) {
        uint4* z = reinterpret_cast<uint4*>(rv_smem + m.stage);
        for (uint32_t i = tid; i < (p.smem_stage_cap >> 4); i += kBlock) z[i] = make_uint4(0u, 0u, 0u, 0u);
    }
    __syncthreads();
    const bool fast = w.staged && (flags[0] & 2u);
    if (fast) {
        if (!warp_precise) emit_walk<W, true>(p, t, m, w, q, true);
        else emit_precise<W, PERM>(p, t, m, w, q, true, bad);  // (warp-uniform) stages its strings like the other warps
        prefetch_window(p, w);
        if (p.n_utf8 > 0) stage_write_out(p, m);
    } else {
        // the tile's bytes or its strings do not fit shared memory: walk the records in global memory and write
        // strings straight to their Arrow buffers (slow; window sizing keeps such tiles rare)
        if (tid == 0) atomicAdd(p.ctrl + CW_SLOW_TILES, 1ull);
        emit_precise<W, PERM>(p, t, m, w, q, false, bad);
    }
}

}  // namespace rv
