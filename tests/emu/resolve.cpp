// TEST INFRASTRUCTURE ONLY — host emulation of a resolved decode (rv_schema_resolve).
//
// The pipeline of projection.cpp (each lane's walker state carried from its count walk to its emit walk) for a plan
// built from the product's resolve_schemas + build_resolved_plan, optionally projected to the reader's top-level fields.
#include "projection.cpp"

namespace {

int decode_resolved(const char* json, size_t len, const char* reader_json, size_t reader_len, const uint8_t* data, const int64_t* off, int64_t n,
                    int64_t num_chunks, const char* const* columns, int64_t n_columns, Decoded& out, int64_t* err_record) {
    std::shared_ptr<const AvroNode> writer = parse_avro_schema(json, len), reader = parse_avro_schema(reader_json, reader_len);
    std::string why;
    if (!is_supported(*writer, &why) || !is_supported(*reader, &why)) throw std::runtime_error("unsupported: " + why);
    const Resolution res = resolve_schemas(*writer, *reader);
    const std::vector<ArrowField> all = to_arrow_fields(*reader);
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
    out.plan = plan_sp;
    const Plan& plan = *plan_sp;
    const int S = int(plan.streams.size()), S1 = std::max(S, 1);
    const int k = int(clamp_chunks(num_chunks, n));
    out.k = k;
    auto tiles = make_tiles(n, k);
    std::vector<uint32_t> cur(size_t(S1) * kTile);
    std::vector<EmuWalker::Cur> qs(kTile);
    std::vector<std::vector<uint32_t>> tile_agg(tiles.size(), std::vector<uint32_t>(size_t(S1), 0));
    for (size_t ti = 0; ti < tiles.size(); ++ti) {  // count
        bool wp[kTile / 32];
        uint32_t code = 0;
        const int bad = count_tile_q(plan, data, off, tiles[ti], S, cur, wp, &code, qs.data());
        if (bad >= 0) { *err_record = tiles[ti].r0 + bad; return int(code); }
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
        (void)count_tile_q(plan, data, off, t, S, cur, wp, &code, qs.data());
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
                EmuWalker::walk<WM_EMIT>(c, int(plan.nodes.size()), q);
            } else {
                FastCtx f;
                init_fast(f, plan, window, off, t, lane, cur.data(), cb);
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

// emu_decode of data written with `json`, read as `reader_json`; columns may be NULL (all the reader's fields).
extern "C" int emu_decode_resolved(const char* json, size_t len, const char* reader_json, size_t reader_len, const uint8_t* data,
                                   const int64_t* off, int64_t n, int64_t num_chunks, const char* const* columns, int64_t n_columns,
                                   ArrowArray* out_batches, ArrowSchema* out_schema, int64_t* k_out, int64_t* err_record, char* msg,
                                   size_t msg_cap) {
    try {
        Decoded d;
        const int rc = decode_resolved(json, len, reader_json, reader_len, data, off, n, num_chunks, columns, n_columns, d, err_record);
        *k_out = d.k;
        if (rc) return rc == int(E_ENUM_MAP) ? int(E_ENUM) : rc;   // the status the library reports (engine.cu status_of)
        for (int j = 0; j < d.k; ++j) export_batch(*d.plan, d.keep->chunks[size_t(j)], d.keep->arena, d.keep, &out_batches[j]);
        if (out_schema) export_arrow_schema(d.fields, out_schema);
        return 0;
    } catch (const std::exception& e) {
        std::snprintf(msg, msg_cap, "%s", e.what());
        return -1;
    }
}
