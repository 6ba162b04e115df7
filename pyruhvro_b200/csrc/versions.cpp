#include "versions.hpp"

#include <algorithm>
#include <cstring>
#include <stdexcept>

namespace rv {
namespace {

void pair_array(const Plan& r, const Plan& w, int ra, int wa, VersionPairing& p) {
    const OutArray& a = r.arrays[size_t(ra)];
    const OutArray& b = w.arrays[size_t(wa)];
    if (a.type != b.type || a.width != b.width || a.always_validity != b.always_validity || a.children.size() != b.children.size())
        throw std::runtime_error("the writer's resolved output tree differs from the reader's");
    int& sp = p.space[size_t(a.space)];
    if (sp >= 0 && sp != b.space) throw std::runtime_error("the writer's resolved row spaces differ from the reader's");
    sp = b.space;
    const int rs[3] = {a.slot_v, a.slot_a, a.slot_b}, ws[3] = {b.slot_v, b.slot_a, b.slot_b};
    for (int i = 0; i < 3; ++i) {
        if (rs[i] < 0) {
            if (ws[i] >= 0) throw std::runtime_error("the writer's resolved plan has a buffer the reader's does not");
            continue;
        }
        if (ws[i] < 0) {
            if (i == 0) continue;  // validity the writer never needs: all valid
            throw std::runtime_error("the writer's resolved plan lacks a buffer of the reader's");
        }
        const Slot& x = r.slots[size_t(rs[i])];
        const Slot& y = w.slots[size_t(ws[i])];
        if (x.role != y.role || x.width != y.width) throw std::runtime_error("the writer's resolved buffers differ from the reader's");
        p.slot[size_t(rs[i])] = ws[i];
    }
    for (size_t c = 0; c < a.children.size(); ++c) pair_array(r, w, a.children[c], b.children[c], p);
}

int role_width(const Slot& s) {
    switch (s.role) {
        case SlotRole::Values32: return 4;
        case SlotRole::Values64: return 8;
        case SlotRole::ValuesW: return s.width;
        case SlotRole::TypeIds: return 1;
        case SlotRole::Offsets: return 4;
        default: return 0;
    }
}

size_t align16(size_t v) { return (v + 15) & ~size_t(15); }

}  // namespace

VersionPairing pair_plans(const Plan& reader, const Plan& writer) {
    VersionPairing p;
    p.slot.assign(reader.slots.size(), -1);
    p.space.assign(size_t(reader.n_spaces), -1);
    p.space[0] = 0;
    if (reader.top_arrays.size() != writer.top_arrays.size()) throw std::runtime_error("the writer's resolved columns differ from the reader's");
    for (size_t i = 0; i < reader.top_arrays.size(); ++i) pair_array(reader, writer, reader.top_arrays[i], writer.top_arrays[i], p);
    for (int s = 0; s < reader.n_spaces; ++s)
        if (p.space[size_t(s)] < 0) throw std::runtime_error("a reader row space has no writer row space");
    for (size_t s = 0; s < reader.slots.size(); ++s)
        if (p.slot[s] < 0 && reader.slots[s].role != SlotRole::Validity && reader.slots[s].role != SlotRole::Data)
            throw std::runtime_error("a reader buffer has no writer buffer");
    return p;
}

void versions_chunk_totals(const Plan& reader, const std::vector<VersionPairing>& pairs, const std::vector<VersionPart>& parts,
                           unsigned long long* tot) {
    const int S = int(reader.streams.size());
    for (int i = 0; i < std::max(S, 1); ++i) tot[i] = 0;
    for (int i = 0; i < S; ++i) {
        const Stream& st = reader.streams[size_t(i)];
        int data_slot = -1;
        if (!st.is_rows)
            for (size_t sl = 0; sl < reader.slots.size(); ++sl)
                if (reader.slots[sl].role == SlotRole::Data && reader.slots[sl].stream == i) data_slot = int(sl);
        for (size_t w = 0; w < parts.size(); ++w) {
            const ChunkOut* c = parts[w].c;
            if (!c) continue;
            if (st.is_rows) tot[i] += (unsigned long long)c->space_rows[size_t(pairs[w].space[size_t(st.space)])];
            else if (data_slot >= 0) tot[i] += (unsigned long long)c->slot_bytes[size_t(pairs[w].slot[size_t(data_slot)])];
        }
    }
}

void versions_null_counts(const Plan& reader, const std::vector<VersionPairing>& pairs, const std::vector<VersionPart>& parts, ChunkOut& out,
                          int64_t null_rows) {
    for (int sl : reader.validity_slots) {
        int64_t nulls = reader.slots[size_t(sl)].space == 0 ? null_rows : 0;
        for (size_t w = 0; w < parts.size(); ++w)
            if (parts[w].c && pairs[w].slot[size_t(sl)] >= 0) nulls += parts[w].c->null_count[size_t(pairs[w].slot[size_t(sl)])];
        out.null_count[size_t(sl)] = nulls;
    }
}

TakePlan plan_take(const Plan& reader, const std::vector<VersionPairing>& pairs, const std::vector<std::vector<VersionPart>>& parts,
                   const std::vector<ChunkOut>& chunks, uint8_t* out_base, const std::vector<const unsigned long long*>& map0, uint8_t* base) {
    const int k = int(chunks.size()), W = int(pairs.size()), n_slots = int(reader.slots.size());
    // the row space each list / map offsets slot opens
    std::vector<int> child_space(size_t(n_slots), -1);
    for (const OutArray& a : reader.arrays)
        if ((a.type == AT::List || a.type == AT::Map) && a.slot_a >= 0) child_space[size_t(a.slot_a)] = reader.arrays[size_t(a.children[0])].space;
    std::vector<int> data_of(size_t(n_slots), -1);
    for (const OutArray& a : reader.arrays)
        if ((a.type == AT::Utf8 || a.type == AT::Binary) && a.slot_a >= 0) data_of[size_t(a.slot_a)] = a.slot_b;
    const int levels = reader.max_depth + 1;
    struct Entry { int j, sp; };
    std::vector<Entry> entries;
    TakePlan tp;
    tp.level_first.push_back(0);
    for (int l = 0; l < levels; ++l) {
        for (int sp = 0; sp < reader.n_spaces; ++sp)
            if (reader.space_depth[size_t(sp)] == l)
                for (int j = 0; j < k; ++j) entries.push_back(Entry{j, sp});
        tp.level_first.push_back(int(entries.size()));
    }
    std::vector<int> job_slots;
    std::vector<int> entry_first(entries.size()), entry_n(entries.size());
    for (size_t e = 0; e < entries.size(); ++e) {
        entry_first[e] = int(job_slots.size());
        for (int sl = 0; sl < n_slots; ++sl) {
            const Slot& s = reader.slots[size_t(sl)];
            if (s.space == entries[e].sp && s.role != SlotRole::Data) job_slots.push_back(sl);
        }
        entry_n[e] = int(job_slots.size()) - entry_first[e];
    }
    const size_t n_jobs = job_slots.size();
    auto blocks_of = [](long long rows) { return std::max<long long>(1, (rows + kTakeBlock - 1) / kTakeBlock); };
    // header
    size_t off = 0;
    const size_t off_spaces = off; off = align16(off + entries.size() * sizeof(TakeSpace));
    const size_t off_jobs = off; off = align16(off + n_jobs * sizeof(TakeJob));
    size_t n_scans = 0;
    for (int sl : job_slots) n_scans += reader.slots[size_t(sl)].role == SlotRole::Offsets ? 1 : 0;
    const size_t off_scans = off; off = align16(off + n_scans * sizeof(TakeScan));
    const size_t off_ptrs = off; off = align16(off + n_jobs * 2 * size_t(std::max(W, 1)) * sizeof(void*));
    tp.header_bytes = off;
    tp.header.assign(off, 0);
    // block sums and child maps follow the header
    auto* h_spaces = reinterpret_cast<TakeSpace*>(tp.header.data() + off_spaces);
    auto* h_jobs = reinterpret_cast<TakeJob*>(tp.header.data() + off_jobs);
    auto* h_scans = reinterpret_cast<TakeScan*>(tp.header.data() + off_scans);
    auto* h_ptrs = reinterpret_cast<const uint8_t**>(tp.header.data() + off_ptrs);
    std::vector<std::vector<unsigned long long*>> maps(size_t(k), std::vector<unsigned long long*>(size_t(reader.n_spaces), nullptr));
    for (int j = 0; j < k; ++j) {
        maps[size_t(j)][0] = const_cast<unsigned long long*>(map0[size_t(j)]);
        for (int sp = 1; sp < reader.n_spaces; ++sp) {
            maps[size_t(j)][size_t(sp)] = reinterpret_cast<unsigned long long*>(base + off);
            off = align16(off + size_t(std::max<int64_t>(chunks[size_t(j)].space_rows[size_t(sp)], 1)) * 8);
        }
    }
    size_t scan_i = 0;
    tp.scan_first.push_back(0);
    int level = 0;
    for (size_t e = 0; e < entries.size(); ++e) {
        while (int(e) >= tp.level_first[size_t(level) + 1]) { tp.scan_first.push_back(int(scan_i)); ++level; }
        const int j = entries[e].j, sp = entries[e].sp;
        const ChunkOut& c = chunks[size_t(j)];
        const long long rows = c.space_rows[size_t(sp)];
        h_spaces[e] = TakeSpace{maps[size_t(j)][size_t(sp)], rows, entry_first[e], entry_n[e]};
        for (int q = entry_first[e]; q < entry_first[e] + entry_n[e]; ++q) {
            const int sl = job_slots[size_t(q)];
            const Slot& s = reader.slots[size_t(sl)];
            TakeJob& jb = h_jobs[q];
            jb.dst = out_base + c.slot_off[size_t(sl)];
            jb.role = int32_t(s.role);
            jb.width = role_width(s);
            const uint8_t** src = h_ptrs + size_t(q) * 2 * size_t(W);
            const uint8_t** src_data = src + W;
            for (int w = 0; w < W; ++w) {
                const VersionPart& part = parts[size_t(j)][size_t(w)];
                const int ws = pairs[size_t(w)].slot[size_t(sl)];
                src[w] = part.c && ws >= 0 ? part.base + part.c->slot_off[size_t(ws)] : nullptr;
                const int ds = data_of[size_t(sl)];
                src_data[w] = part.c && ds >= 0 ? part.base + part.c->slot_off[size_t(pairs[size_t(w)].slot[size_t(ds)])] : nullptr;
            }
            jb.src = reinterpret_cast<const uint8_t* const*>(base + off_ptrs + size_t(q) * 2 * size_t(W) * sizeof(void*));
            jb.src_data = jb.src + W;
            jb.dst_data = data_of[size_t(sl)] >= 0 ? out_base + c.slot_off[size_t(data_of[size_t(sl)])] : nullptr;
            jb.child_map = child_space[size_t(sl)] >= 0 ? maps[size_t(j)][size_t(child_space[size_t(sl)])] : nullptr;
            jb.block_base = nullptr;
            if (s.role == SlotRole::Offsets) {
                jb.block_base = reinterpret_cast<long long*>(base + off);
                h_scans[scan_i++] = TakeScan{jb.block_base, blocks_of(rows)};
                off = align16(off + size_t(blocks_of(rows)) * 8);
            }
        }
    }
    while (int(tp.scan_first.size()) < levels + 1) tp.scan_first.push_back(int(scan_i));
    for (int l = 0; l < levels; ++l) {
        long long mx = 1;
        for (int e = tp.level_first[size_t(l)]; e < tp.level_first[size_t(l) + 1]; ++e) mx = std::max(mx, blocks_of(h_spaces[e].rows));
        tp.level_blocks.push_back(mx);
    }
    tp.total_bytes = off;
    tp.spaces = reinterpret_cast<const TakeSpace*>(base + off_spaces);
    tp.scans = reinterpret_cast<const TakeScan*>(base + off_scans);
    tp.jobs = reinterpret_cast<const TakeJob*>(base + off_jobs);
    return tp;
}

}  // namespace rv
