// TEST INFRASTRUCTURE ONLY — host emulation of a permissive decode (rv_schema_permissive).
//
// The pipeline of resolve.cpp for the product's permissive plan (optional_fields + resolve_schemas +
// build_resolved_plan, optionally projected), with the per-lane steps of fused_body<W, true>:
//   1. FAST count; a lane whose record is not plain repeats it PRECISE, which settles what it is;
//   2. a lane whose record has a record error (record_error) counts nothing and is listed; the scan follows;
//   3. the emit of such a lane runs on the precise path with c.err set to its code, which writes its row absent.
// Any other error fails the call as in a strict decode.  Framed input (Confluent, single-object) is checked as the
// kernel's record setup does.
#include "projection.cpp"

namespace {

struct Frame { uint32_t skip = 0; int32_t check = 0; uint32_t id = 0; unsigned long long fp = 0; };

// fused_body's init_ctx framing check, for either flavour (the context already points at the record).
template <class C>
void frame_check(C& c, const Frame& fr) {
    if (!c.in_range || !fr.skip) return;
    if (c.end - c.pos < fr.skip) { c.err = E_FRAME; return; }
    if (fr.check == kFrameSingleObject) {
        unsigned long long fp = 0;
        for (uint32_t b = 0; b < 8; ++b) fp |= static_cast<unsigned long long>(ld_u8(c, c.pos + 2 + b)) << (8 * b);
        if (ld_u8(c, c.pos) != 0xC3u || ld_u8(c, c.pos + 1) != 0x01u || fp != fr.fp) c.err = E_FRAME;
    } else if (fr.check) {
        const uint32_t id = (ld_u8(c, c.pos + 1) << 24) | (ld_u8(c, c.pos + 2) << 16) | (ld_u8(c, c.pos + 3) << 8) | ld_u8(c, c.pos + 4);
        if (ld_u8(c, c.pos) != 0u || (fr.check == 2 && id != fr.id)) c.err = E_FRAME;
    }
    c.pos += fr.skip;
}

template <class Q>
void zero_cursors(Q& q) {
    if constexpr (EmuWalker::kRegCursors) for (int s = 0; s < EmuWalker::kStreams; ++s) q.v[s] = 0;
}

// Steps 1 and 2 for one tile.  bad[lane] = the lane's record error (0: none); returns the first fatal lane or -1.
int count_tile_perm(const Plan& plan, const uint8_t* data, const int64_t* off, const Tile& t, int S, const Frame& fr, std::vector<uint32_t>& cur,
                    bool* warp_precise, uint32_t* bad, uint32_t* err_code, EmuWalker::Cur* qs) {
    std::fill(cur.begin(), cur.end(), 0u);
    const std::vector<uint8_t> window = make_window(data, off, t);
    for (int w = 0; w < kTile / 32; ++w) warp_precise[w] = false;
    for (int lane = 0; lane < kTile; ++lane) {
        bad[lane] = 0;
        FastCtx f;
        init_fast(f, plan, window, off, t, lane, cur.data(), nullptr);
        frame_check(f, fr);
        EmuWalker::Cur q{};
        EmuWalker::walk<WM_COUNT>(f, int(plan.nodes.size()), q);
        if (f.in_range && f.pos > f.end + kWindowPad) { std::fprintf(stderr, "emu: fast reader ran %u bytes past the record\n", f.pos - f.end); std::abort(); }
        if (f.in_range && f.err) {
            warp_precise[lane / 32] = true;
            for (int s = 0; s < S; ++s) cur[size_t(s) * kTile + lane] = 0;
            Ctx c;
            init_ctx(c, plan, data, off, t, lane, cur.data(), S, nullptr);
            frame_check(c, fr);
            q = EmuWalker::Cur{};
            EmuWalker::walk<WM_COUNT>(c, int(plan.nodes.size()), q);
            if (c.err && !record_error(c.err)) { *err_code = c.err; return lane; }
            if (c.err) {
                bad[lane] = c.err;
                for (int s = 0; s < S; ++s) cur[size_t(s) * kTile + lane] = 0;
                zero_cursors(q);
            }
        }
        store_cursors(q, cur.data() + lane, S);
        qs[lane] = q;
    }
    return -1;
}

int decode_permissive(const char* json, size_t len, const char* reader_json, size_t reader_len, const uint8_t* data, const int64_t* off, int64_t n,
                      int64_t num_chunks, const char* const* columns, int64_t n_columns, const Frame& fr, Decoded& out,
                      std::vector<unsigned long long>& bad_list, int64_t* err_record) {
    std::shared_ptr<const AvroNode> writer = parse_avro_schema(json, len);
    std::shared_ptr<const AvroNode> reader = reader_json ? std::shared_ptr<const AvroNode>(parse_avro_schema(reader_json, reader_len)) : writer;
    std::string why;
    if (!is_supported(*writer, &why) || !is_supported(*reader, &why)) throw std::runtime_error("unsupported: " + why);
    std::shared_ptr<const AvroNode> r2 = optional_fields(*reader);
    const Resolution res = resolve_schemas(*writer, *r2);
    const std::vector<ArrowField> all = to_arrow_fields(*r2);
    std::vector<int> selected;
    if (columns) {
        std::vector<std::string> names, requested(columns, columns + n_columns);
        for (const ArrowField& f : all) names.push_back(f.name);
        selected = select_columns(names, requested);
        for (int i : selected) out.fields.push_back(all[size_t(i)]);
    } else {
        out.fields = all;
    }
    auto plan_sp = std::make_shared<Plan>(build_resolved_plan(res, all, columns ? &selected : nullptr));
    plan_sp->permissive = true;
    out.plan = plan_sp;
    const Plan& plan = *plan_sp;
    const int S = int(plan.streams.size()), S1 = std::max(S, 1);
    const int k = int(clamp_chunks(num_chunks, n));
    out.k = k;
    auto tiles = make_tiles(n, k);
    std::vector<uint32_t> cur(size_t(S1) * kTile);
    std::vector<EmuWalker::Cur> qs(kTile);
    uint32_t bad[kTile];
    std::vector<std::vector<uint32_t>> tile_agg(tiles.size(), std::vector<uint32_t>(size_t(S1), 0));
    for (size_t ti = 0; ti < tiles.size(); ++ti) {  // count
        bool wp[kTile / 32];
        uint32_t code = 0;
        const int fatal = count_tile_perm(plan, data, off, tiles[ti], S, fr, cur, wp, bad, &code, qs.data());
        if (fatal >= 0) { *err_record = tiles[ti].r0 + fatal; return int(code); }
        for (int lane = 0; lane < tiles[ti].nrec; ++lane)
            if (bad[lane]) bad_list.push_back((static_cast<unsigned long long>(tiles[ti].r0 + lane) << 8) | bad[lane]);
        for (int s = 0; s < S; ++s) {
            uint64_t sum = 0;
            for (int lane = 0; lane < kTile; ++lane) sum += cur[size_t(s) * kTile + lane];
            if (sum > 0x7FFFFFFFull) { *err_record = tiles[ti].r0; return int(E_OVERFLOW); }
            tile_agg[ti][size_t(s)] = uint32_t(sum);
        }
    }
    std::vector<unsigned long long> chunk_tot(size_t(k) * size_t(S1), 0ull);  // per-chunk scan
    std::vector<std::vector<uint32_t>> tile_base(tiles.size(), std::vector<uint32_t>(size_t(S1), 0));
    for (size_t ti = 0; ti < tiles.size(); ++ti)
        for (int s = 0; s < S; ++s) {
            unsigned long long& tot = chunk_tot[size_t(tiles[ti].chunk) * size_t(S1) + size_t(s)];
            tile_base[ti][size_t(s)] = uint32_t(tot);
            tot += tile_agg[ti][size_t(s)];
            if (tot > 0x7FFFFFFFull) { *err_record = tiles[ti].r0; return int(E_OVERFLOW); }
        }
    Layout L = compute_layout(plan, n, k, chunk_tot.data());
    auto keep = std::make_shared<Keep>();
    keep->plan = plan_sp;
    keep->arena = static_cast<uint8_t*>(std::calloc(std::max<size_t>(L.total_bytes, 64), 1));
    const int n_slots = int(plan.slots.size());
    std::vector<void*> bufs(size_t(k) * size_t(std::max(n_slots, 1)));
    for (int j = 0; j < k; ++j)
        for (int sl = 0; sl < n_slots; ++sl) bufs[size_t(j) * size_t(n_slots) + size_t(sl)] = keep->arena + L.chunks[size_t(j)].slot_off[size_t(sl)];
    for (size_t ti = 0; ti < tiles.size(); ++ti) {  // emit
        const Tile& t = tiles[ti];
        void* const* cb = bufs.data() + size_t(t.chunk) * size_t(n_slots);
        bool wp[kTile / 32];
        uint32_t code = 0;
        (void)count_tile_perm(plan, data, off, t, S, fr, cur, wp, bad, &code, qs.data());
        for (int s = 0; s < S; ++s) {
            uint32_t run = tile_base[ti][size_t(s)];
            for (int lane = 0; lane < kTile; ++lane) { uint32_t v = cur[size_t(s) * kTile + lane]; cur[size_t(s) * kTile + lane] = run; run += v; }
        }
        if (t.local == 0)
            for (const DNode& nd : plan.nodes)
                if (!(nd.flags & NF_SKIP) && (nd.kind == NK_STR || nd.kind == NK_ENUM || nd.kind == NK_LIST || nd.kind == NK_MAP || nd.kind == NK_BYTES ||
                                              (nd.kind == NK_DEFAULT && nd.pad0 == NK_STR)))
                    static_cast<int32_t*>(cb[nd.slot_a])[0] = 0;
        const std::vector<uint8_t> window = make_window(data, off, t);
        for (int lane = 0; lane < kTile; ++lane) {
            EmuWalker::Cur q = qs[size_t(lane)];
            load_cursors(q, cur.data() + lane, S);
            if (wp[lane / 32]) {
                Ctx c;
                init_ctx(c, plan, data, off, t, lane, cur.data(), S, cb);
                frame_check(c, fr);
                if (bad[lane]) c.err = bad[lane];
                EmuWalker::walk<WM_EMIT>(c, int(plan.nodes.size()), q);
            } else {
                // the FAST emit (and with it the item-position table and the skip_end jump) never meets a bad lane
                if (bad[lane]) { std::fprintf(stderr, "emu: a bad record reached the FAST emit\n"); std::abort(); }
                FastCtx f;
                init_fast(f, plan, window, off, t, lane, cur.data(), cb);
                frame_check(f, fr);
                EmuWalker::walk<WM_EMIT>(f, int(plan.nodes.size()), q);
            }
        }
    }
    for (int j = 0; j < k; ++j)  // null counts
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

}  // namespace

// The permissive decode of data written with `json`, read as `reader_json` (NULL: the writer's schema) made permissive,
// projected to `columns` (NULL: all).  frame: {header bytes, check (0, 1, 2 or kFrameSingleObject), schema id} and the
// fingerprint.  bad_out (room for n entries) receives (record << 8 | code) of each bad record in record order, *n_bad
// their count.  Returns 0, or a fatal error's code with *err_record set, or -1 with msg set.
extern "C" int emu_decode_permissive(const char* json, size_t len, const char* reader_json, size_t reader_len, const uint8_t* data,
                                     const int64_t* off, int64_t n, int64_t num_chunks, const char* const* columns, int64_t n_columns,
                                     const int64_t* frame, unsigned long long frame_fp, ArrowArray* out_batches, ArrowSchema* out_schema,
                                     int64_t* k_out, unsigned long long* bad_out, int64_t* n_bad, int64_t* err_record, char* msg, size_t msg_cap) {
    try {
        Frame fr;
        fr.skip = uint32_t(frame[0]);
        fr.check = int32_t(frame[1]);
        fr.id = uint32_t(frame[2]);
        fr.fp = frame_fp;
        Decoded d;
        std::vector<unsigned long long> bad;
        const int rc = decode_permissive(json, len, reader_json, reader_len, data, off, n, num_chunks, columns, n_columns, fr, d, bad, err_record);
        *k_out = d.k;
        if (rc) return rc;
        std::copy(bad.begin(), bad.end(), bad_out);
        *n_bad = int64_t(bad.size());
        for (int j = 0; j < d.k; ++j) export_batch(*d.plan, d.keep->chunks[size_t(j)], d.keep->arena, d.keep, &out_batches[j]);
        if (out_schema) export_arrow_schema(d.fields, out_schema);
        return 0;
    } catch (const std::exception& e) {
        std::snprintf(msg, msg_cap, "%s", e.what());
        return -1;
    }
}
