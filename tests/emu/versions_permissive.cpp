// TEST INFRASTRUCTURE ONLY — host emulation of the permissive multi-version decode (rv_versions_permissive).
//
// versions.cpp's pipeline for a permissive registry: the partition's classification (take.cuh vp_header) with a message
// that fails it put in its chunk's bad group (a kNoRow row-map entry, listed as the partition lists it), one permissive
// resolved decode per (output chunk, writer) group through permissive.cpp's emulated pipeline, its bad rows mapped back
// to messages through the inverse of the row map, the layout with every chunk's bad rows (versions.cpp) and the take's
// per-row steps with the null-row path (emulate_take_level_perm).  Groups are packed without their headers, as in
// versions.cpp.
#include "permissive.cpp"

#include "../../pyruhvro_b200/csrc/take.cuh"
#include "../../pyruhvro_b200/csrc/versions.hpp"

namespace {

// The per-row steps of take_rows_body<true> / take_offsets_body<true> (versions.cu) over one level of row spaces, one
// row after the other; a kNoRow entry is a null row.
void emulate_take_level_perm(const TakePlan& tp, size_t level) {
    for (int e = tp.level_first[level]; e < tp.level_first[level + 1]; ++e) {
        const TakeSpace& sp = tp.spaces[e];
        for (int q = sp.first_job; q < sp.first_job + sp.n_jobs; ++q) {
            const TakeJob& jb = tp.jobs[q];
            const SlotRole role = SlotRole(jb.role);
            auto null_row = [&](long long r) { return sp.map[r] == kNoRow; };
            if (role == SlotRole::Validity || role == SlotRole::Bits) {
                for (long long w0 = 0; w0 < sp.rows; w0 += 32) {  // one __ballot_sync word per 32 rows
                    uint32_t word = 0;
                    for (long long r = w0; r < std::min(sp.rows, w0 + 32); ++r)
                        word |= (null_row(r) ? 0u : take_bit(jb, take_writer(sp.map[r]), take_row(sp.map[r]))) << (r - w0);
                    reinterpret_cast<uint32_t*>(jb.dst)[w0 >> 5] = word;
                }
            } else if (role == SlotRole::Offsets) {
                reinterpret_cast<int32_t*>(jb.dst)[0] = 0;
                int32_t pos = 0;
                for (long long r = 0; r < sp.rows; ++r) {
                    if (null_row(r)) { take_null_offsets_row(jb, r, pos); continue; }
                    const uint32_t w = take_writer(sp.map[r]);
                    const int64_t s = take_row(sp.map[r]);
                    const int32_t len = take_len(jb, w, s);
                    take_offsets_row(jb, w, s, r, pos, len);
                    if (jb.dst_data) take_copy(jb.dst_data + pos, jb.src_data[w] + take_start(jb, w, s), len);
                    pos += len;
                }
            } else {
                for (long long r = 0; r < sp.rows; ++r) {
                    if (null_row(r)) take_null_value(jb, r);
                    else take_value(jb, take_writer(sp.map[r]), take_row(sp.map[r]), r);
                }
            }
        }
    }
}

struct PermScratch { uint8_t* p = nullptr; ~PermScratch() { std::free(p); } };

}  // namespace

// writer_jsons[i] is the writer of ids[i] (Confluent; ascending) or of fps[i] (single-object when fps is not NULL;
// ascending).  bad_out (room for n) receives (message << 8 | status) in message order.  Returns 0, a fatal status with
// *err_record, or -1 (msg).
extern "C" int emu_decode_versions_permissive(const char* reader_json, size_t reader_len, const char* const* writer_jsons, const int64_t* ids,
                                              const unsigned long long* fps, int64_t W, const uint8_t* data, const int64_t* off, int64_t n,
                                              int64_t num_chunks, const char* const* columns, int64_t n_columns, ArrowArray* out_batches,
                                              ArrowSchema* out_schema, int64_t* k_out, unsigned long long* bad_out, int64_t* n_bad,
                                              int64_t* err_record, char* msg, size_t msg_cap) {
    try {
        // R' (rv_schema_permissive of the reader, projected) and every writer's permissive resolved plan next to it
        std::shared_ptr<const AvroNode> reader = parse_avro_schema(reader_json, reader_len);
        std::shared_ptr<const AvroNode> r2 = optional_fields(*reader);
        const std::vector<ArrowField> all = to_arrow_fields(*r2);
        std::vector<int> selected;
        std::vector<ArrowField> fields = all;
        if (columns) {
            std::vector<std::string> names, requested(columns, columns + n_columns);
            for (const ArrowField& f : all) names.push_back(f.name);
            selected = select_columns(names, requested);
            fields.clear();
            for (int i : selected) fields.push_back(all[size_t(i)]);
        }
        auto plan_sp = std::make_shared<Plan>(build_resolved_plan(resolve_schemas(*reader, *r2), all, columns ? &selected : nullptr));
        plan_sp->permissive = true;
        const Plan& rp = *plan_sp;
        std::vector<VersionPairing> pairs;
        for (int64_t w = 0; w < W; ++w) {
            std::shared_ptr<const AvroNode> wn = parse_avro_schema(writer_jsons[w], std::strlen(writer_jsons[w]));
            pairs.push_back(pair_plans(rp, build_resolved_plan(resolve_schemas(*wn, *r2), all, columns ? &selected : nullptr)));
        }
        // partition
        const int k = int(clamp_chunks(num_chunks, n));
        *k_out = k;
        const int64_t cr = n / k;
        const int64_t hdr = fps ? int64_t(kSingleObjectHeader) : 5;
        std::vector<uint32_t> ids32;
        for (int64_t w = 0; ids && w < W; ++w) ids32.push_back(uint32_t(ids[w]));
        std::vector<std::vector<uint8_t>> gdata(size_t(k) * size_t(W));
        std::vector<std::vector<int64_t>> goff(size_t(k) * size_t(W), std::vector<int64_t>{0});
        std::vector<std::vector<int64_t>> inv(size_t(k) * size_t(W));
        std::vector<unsigned long long> map0(size_t(std::max<int64_t>(n, 1)), kNoRow);
        std::vector<int64_t> null_rows(size_t(k), 0);
        std::vector<unsigned long long> bad;
        for (int64_t i = 0; i < n; ++i) {
            const int j = int(std::min<int64_t>(i / std::max<int64_t>(cr, 1), k - 1));
            int w = -1;
            const uint32_t code = fps ? vp_header(data + off[i], off[i + 1] - off[i], fps, int(W), &w)
                                      : vp_header(data + off[i], off[i + 1] - off[i], ids32.data(), int(W), &w);
            if (code) {
                bad.push_back((static_cast<unsigned long long>(i) << 8) | code);
                ++null_rows[size_t(j)];
                continue;
            }
            const size_t g = size_t(j) * size_t(W) + size_t(w);
            map0[size_t(i)] = take_pack(uint32_t(w), uint64_t(goff[g].size() - 1));
            inv[g].push_back(i);
            gdata[g].insert(gdata[g].end(), data + off[i] + hdr, data + off[i + 1]);
            goff[g].push_back(int64_t(gdata[g].size()));
        }
        // the groups' permissive resolved decodes; their bad rows are messages through inv, a fatal error fails the call
        std::vector<Decoded> subs(gdata.size());
        unsigned long long fatal = ~0ull;
        for (size_t g = 0; g < gdata.size(); ++g) {
            const int64_t cnt = int64_t(goff[g].size()) - 1;
            if (cnt == 0) continue;
            const int w = int(g % size_t(W));
            int64_t rec = -1;
            std::vector<unsigned long long> sub_bad;
            gdata[g].resize(gdata[g].size() + 64);
            const int rc = decode_permissive(writer_jsons[w], std::strlen(writer_jsons[w]), reader_json, reader_len, gdata[g].data(), goff[g].data(), cnt, 1,
                                             columns, n_columns, Frame{}, subs[g], sub_bad, &rec);
            if (rc) { fatal = std::min(fatal, (static_cast<unsigned long long>(inv[g][size_t(rec)]) << 8) | uint32_t(rc)); continue; }
            for (unsigned long long b : sub_bad) bad.push_back((static_cast<unsigned long long>(inv[g][size_t(b >> 8)]) << 8) | (b & 0xFF));
        }
        if (fatal != ~0ull) { *err_record = int64_t(fatal >> 8); return int(fatal & 0xFF); }
        // layout from the parts and the bad rows, then the take
        const int S1 = std::max(int(rp.streams.size()), 1);
        std::vector<std::vector<VersionPart>> parts(static_cast<size_t>(k), std::vector<VersionPart>(static_cast<size_t>(W)));
        std::vector<unsigned long long> chunk_tot(size_t(k) * size_t(S1), 0ull);
        for (int j = 0; j < k; ++j) {
            for (int64_t w = 0; w < W; ++w) {
                const Decoded& d = subs[size_t(j) * size_t(W) + size_t(w)];
                if (d.keep) parts[size_t(j)][size_t(w)] = VersionPart{&d.keep->chunks[0], d.keep->arena};
            }
            versions_chunk_totals(rp, pairs, parts[size_t(j)], chunk_tot.data() + size_t(j) * size_t(S1));
            for (int i = 0; i < S1; ++i)
                if (chunk_tot[size_t(j) * size_t(S1) + size_t(i)] > 0x7FFFFFFFull) { *err_record = int64_t(j) * cr; return int(E_OVERFLOW); }
        }
        Layout L = compute_layout(rp, n, k, chunk_tot.data());
        auto keep = std::make_shared<Keep>();
        keep->plan = plan_sp;
        keep->arena = static_cast<uint8_t*>(std::calloc(std::max<size_t>(L.total_bytes, 64), 1));
        std::vector<const unsigned long long*> m0(static_cast<size_t>(k));
        for (int j = 0; j < k; ++j) m0[size_t(j)] = map0.data() + int64_t(j) * cr;
        PermScratch scratch;
        scratch.p = static_cast<uint8_t*>(std::calloc(std::max<size_t>(plan_take(rp, pairs, parts, L.chunks, keep->arena, m0, nullptr).total_bytes, 64), 1));
        const TakePlan tp = plan_take(rp, pairs, parts, L.chunks, keep->arena, m0, scratch.p);
        std::memcpy(scratch.p, tp.header.data(), tp.header_bytes);
        for (size_t l = 0; l + 1 < tp.level_first.size(); ++l) emulate_take_level_perm(tp, l);
        for (int j = 0; j < k; ++j) versions_null_counts(rp, pairs, parts[size_t(j)], L.chunks[size_t(j)], null_rows[size_t(j)]);
        keep->chunks = L.chunks;
        // the report: message order, each code as the status the library reports
        std::sort(bad.begin(), bad.end());
        for (size_t i = 0; i < bad.size(); ++i) {
            const uint32_t code = uint32_t(bad[i] & 0xFF);
            const uint32_t status = code == E_ENUM_MAP ? uint32_t(E_ENUM) : code == E_FRAME_ID ? uint32_t(E_FRAME) : code;
            bad_out[i] = (bad[i] & ~0xFFull) | status;
        }
        *n_bad = int64_t(bad.size());
        for (int j = 0; j < k; ++j) export_batch(rp, keep->chunks[size_t(j)], keep->arena, keep, &out_batches[j]);
        if (out_schema) export_arrow_schema(fields, out_schema);
        return 0;
    } catch (const std::exception& e) {
        std::snprintf(msg, msg_cap, "%s", e.what());
        return -1;
    }
}
