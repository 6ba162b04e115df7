// Builds the flattened decode plan.  Mirrors the decisions of the reference's
// decoder-tree construction (ruhvro/src/fast_decode.rs:176-414) and records, per node,
// which Arrow buffers exist and when a validity bitmap can appear (SURVEY.md A.2).
#include "plan.hpp"

#include <algorithm>
#include <cstring>
#include <stdexcept>

namespace rv {
namespace {

struct Ctx {
    int level;        // level the new node will get
    int ulevel;       // number of union ancestors
    int variant;      // index within the parent union or 0xFF
    int space;        // row space
    int depth;        // list nesting depth of `space`
    bool can_get_null;  // an ancestor in this row space may call append_null on this node
};

struct Builder {
    Plan p;

    int add_slot(SlotRole role, int node, int space, int stream) {
        if (p.slots.size() >= 32000) throw std::runtime_error("schema too wide: too many Arrow buffers");
        Slot s;
        s.role = role; s.node = node; s.space = space; s.stream = stream; s.width = 0;
        s.zero_init = (role == SlotRole::Validity || role == SlotRole::Bits) && space > 0;
        p.slots.push_back(s);
        int id = int(p.slots.size()) - 1;
        if (role == SlotRole::Validity) p.validity_slots.push_back(id);
        return id;
    }
    int add_stream(bool is_rows, int space, int node) {
        if (int(p.streams.size()) >= kMaxStreams)
            throw std::runtime_error("schema too wide: more than " + std::to_string(kMaxStreams) + " variable-length streams (strings + lists + maps)");
        p.streams.push_back(Stream{is_rows, space, node});
        return int(p.streams.size()) - 1;
    }
    int new_node(const Ctx& c, NodeKind kind, bool nullable, bool null_first) {
        if (int(p.nodes.size()) >= kMaxNodes) throw std::runtime_error("schema too large: more than " + std::to_string(kMaxNodes) + " nodes");
        if (c.level > kMaxLevel) throw std::runtime_error("schema nested deeper than " + std::to_string(kMaxLevel) + " levels");
        DNode n{};
        n.kind = kind;
        n.flags = uint8_t((nullable ? NF_NULLABLE : 0) | (null_first ? NF_NULL_FIRST : 0));
        n.level = uint8_t(c.level);
        n.ulevel = uint8_t(c.ulevel);
        n.variant = uint8_t(c.variant);
        n.space = uint8_t(c.space);
        n.slot_v = n.slot_a = n.slot_b = n.stream = -1;
        p.nodes.push_back(n);
        return int(p.nodes.size()) - 1;
    }
    int new_array(AT type, int node, int space, bool always_validity) {
        OutArray a;
        a.type = type; a.node = node; a.space = space; a.always_validity = always_validity;
        a.slot_v = a.slot_a = a.slot_b = -1;
        p.arrays.push_back(a);
        return int(p.arrays.size()) - 1;
    }

    // True when the subtree occupies zero wire bytes and owns no buffers: only nulls and
    // non-nullable records of such (a 2-variant/N-variant union always spends a branch varint).
    static bool zero_sized(const AvroNode& s) {
        if (s.k == AK::Null) return true;
        if (s.k == AK::Record) {
            for (auto& f : s.fields)
                if (!zero_sized(*f.type)) return false;
            return true;
        }
        return false;
    }

    // make_decoder + make_union_decoder + split_null_union (fast_decode.rs:176-214,372-414).
    int build(const AvroNode& s, const ArrowField& f, const Ctx& c) {
        if (s.k == AK::Union) {
            bool two_with_null = s.sub.size() == 2 && (s.sub[0]->k == AK::Null || s.sub[1]->k == AK::Null);
            if (two_with_null) {
                bool null_first = s.sub[0]->k == AK::Null;
                const AvroNode& inner = null_first ? *s.sub[1] : *s.sub[0];
                if (inner.k == AK::Null || inner.k == AK::Union)
                    throw std::runtime_error("unsupported nullable inner type");  // :338
                return build_value(inner, f, true, null_first, c);
            }
            return build_union(s, f, c);
        }
        return build_value(s, f, false, false, c);
    }

    int build_union(const AvroNode& s, const ArrowField& f, const Ctx& c) {
        if (f.type != AT::SparseUnion || f.children.size() != s.sub.size())
            throw std::runtime_error("union variant count mismatch");  // :386-392
        if (c.ulevel >= kMaxUnionLevel) throw std::runtime_error("unions nested deeper than " + std::to_string(kMaxUnionLevel));
        int id = new_node(c, NK_UNION, false, false);
        int arr = new_array(AT::SparseUnion, id, c.space, false);
        int slot = add_slot(SlotRole::TypeIds, id, c.space, -1);
        p.nodes[id].slot_a = int16_t(slot);
        p.nodes[id].aux = int32_t(s.sub.size());
        p.arrays[arr].slot_a = slot;
        for (size_t i = 0; i < s.sub.size(); ++i) {
            Ctx cc{c.level + 1, c.ulevel + 1, int(i), c.space, c.depth, s.sub.size() > 1 || c.can_get_null};
            int child = build(*s.sub[i], f.children[i], cc);
            p.arrays[arr].children.push_back(child);
        }
        p.nodes[id].end = int32_t(p.nodes.size());
        return arr;
    }

    // The value decoders, with the Nullable* wrappers folded into `nullable`.
    int build_value(const AvroNode& s, const ArrowField& f, bool nullable, bool null_first, const Ctx& c) {
        const bool may_null = nullable || c.can_get_null;
        auto leaf = [&](NodeKind nk, SlotRole role) {
            int id = new_node(c, nk, nullable, null_first);
            int arr = new_array(f.type, id, c.space, false);
            int sa = add_slot(role, id, c.space, -1);
            p.nodes[id].slot_a = int16_t(sa);
            p.arrays[arr].slot_a = sa;
            if (may_null) {
                int sv = add_slot(SlotRole::Validity, id, c.space, -1);
                p.nodes[id].slot_v = int16_t(sv);
                p.nodes[id].flags |= NF_VALIDITY;
                p.arrays[arr].slot_v = sv;
            }
            p.nodes[id].end = id + 1;
            return std::make_pair(id, arr);
        };
        auto utf8 = [&](NodeKind nk) {
            auto [id, arr] = leaf(nk, SlotRole::Offsets);
            int st = add_stream(false, c.space, id);
            int sb = add_slot(SlotRole::Data, id, c.space, st);
            p.nodes[id].slot_b = int16_t(sb);
            p.nodes[id].stream = int16_t(st);
            p.arrays[arr].slot_b = sb;
            return std::make_pair(id, arr);
        };
        auto wide = [&](NodeKind nk, int width, int aux) {  // `width` raw bytes per row
            auto [id, arr] = leaf(nk, SlotRole::ValuesW);
            p.slots[size_t(p.nodes[id].slot_a)].width = width;
            p.nodes[id].aux = aux;
            p.arrays[arr].width = width;
            return arr;
        };
        switch (s.k) {
            case AK::Int: case AK::Date: case AK::TimeMillis: return leaf(NK_I32, SlotRole::Values32).second;
            case AK::Long: case AK::TsMillis: case AK::TsMicros: case AK::TimeMicros: return leaf(NK_I64, SlotRole::Values64).second;
            case AK::Bytes: return utf8(NK_BYTES).second;
            case AK::Fixed: return wide(NK_FIXED, s.size, s.size);
            case AK::Uuid: return wide(NK_UUID, 16, 16);
            case AK::DecimalBytes: return wide(NK_DEC_BYTES, 16, 0);
            case AK::DecimalFixed: return wide(NK_DEC_FIXED, 16, s.size);
            case AK::Float: return leaf(NK_F32, SlotRole::Values32).second;
            case AK::Double: return leaf(NK_F64, SlotRole::Values64).second;
            case AK::Bool: return leaf(NK_BOOL, SlotRole::Bits).second;
            case AK::String: return utf8(NK_STR).second;
            case AK::Enum: {
                auto [id, arr] = utf8(NK_ENUM);
                p.nodes[id].aux = int32_t(p.sym_off.size());
                p.nodes[id].aux2 = int32_t(s.symbols.size());
                for (auto& sym : s.symbols) {
                    p.sym_off.push_back(int32_t(p.sym_bytes.size()));
                    p.sym_bytes.insert(p.sym_bytes.end(), sym.begin(), sym.end());
                }
                p.sym_off.push_back(int32_t(p.sym_bytes.size()));
                return arr;
            }
            case AK::Null: {
                int id = new_node(c, NK_NULL, false, false);
                p.nodes[id].end = id + 1;
                return new_array(AT::Null, id, c.space, false);
            }
            case AK::Record: {
                if (f.type != AT::Struct || f.children.size() != s.fields.size())
                    throw std::runtime_error("avro/arrow field count mismatch");  // :348-354
                if (s.fields.empty()) throw std::runtime_error("RecordDecoder produced a record with 0 fields");  // :633-635
                int id = new_node(c, NK_REC, nullable, null_first);
                int arr = new_array(AT::Struct, id, c.space, nullable);
                if (nullable) {  // explicit BooleanBufferBuilder (:363-367)
                    int sv = add_slot(SlotRole::Validity, id, c.space, -1);
                    p.nodes[id].slot_v = int16_t(sv);
                    p.nodes[id].flags |= NF_VALIDITY;
                    p.arrays[arr].slot_v = sv;
                }
                for (size_t i = 0; i < s.fields.size(); ++i) {
                    Ctx cc{c.level + 1, c.ulevel, 0xFF, c.space, c.depth, may_null};
                    int child = build(*s.fields[i].type, f.children[i], cc);
                    p.arrays[arr].children.push_back(child);
                }
                p.nodes[id].end = int32_t(p.nodes.size());
                return arr;
            }
            case AK::Array: case AK::Map: {
                const bool is_map = s.k == AK::Map;
                if (f.type != (is_map ? AT::Map : AT::List) || f.children.size() != 1)
                    throw std::runtime_error(is_map ? "expected Map" : "expected List");
                if (c.depth + 1 > kMaxListDepth)
                    throw std::runtime_error("arrays/maps nested deeper than " + std::to_string(kMaxListDepth) + " levels are not supported");
                if (p.n_spaces >= 250) throw std::runtime_error("schema has too many arrays/maps");
                int id = new_node(c, is_map ? NK_MAP : NK_LIST, nullable, null_first);
                int arr = new_array(is_map ? AT::Map : AT::List, id, c.space, nullable);
                int so = add_slot(SlotRole::Offsets, id, c.space, -1);
                p.nodes[id].slot_a = int16_t(so);
                p.arrays[arr].slot_a = so;
                if (nullable) {  // :330,335
                    int sv = add_slot(SlotRole::Validity, id, c.space, -1);
                    p.nodes[id].slot_v = int16_t(sv);
                    p.nodes[id].flags |= NF_VALIDITY;
                    p.arrays[arr].slot_v = sv;
                }
                int child_space = p.n_spaces++;
                int st = add_stream(true, child_space, id);
                p.space_stream.push_back(st);
                p.space_depth.push_back(c.depth + 1);
                if (c.depth + 1 > p.max_depth) p.max_depth = c.depth + 1;
                p.nodes[id].stream = int16_t(st);
                Ctx cc{c.level + 1, c.ulevel, 0xFF, child_space, c.depth + 1, false};
                if (is_map) {
                    const ArrowField& entries = f.children[0];
                    if (entries.type != AT::Struct || entries.children.size() != 2)
                        throw std::runtime_error("Map entries must have exactly 2 fields (keys, values)");  // :252-254
                    int earr = new_array(AT::Struct, -1, child_space, false);
                    p.arrays[arr].children.push_back(earr);
                    // dedicated key StringBuilder (:158,260)
                    AvroNode key_schema;
                    key_schema.k = AK::String;
                    int karr = build_value(key_schema, entries.children[0], false, false, cc);
                    p.arrays[earr].children.push_back(karr);
                    int varr = build(*s.sub[0], entries.children[1], cc);
                    p.arrays[earr].children.push_back(varr);
                } else {
                    if (zero_sized(*s.sub[0])) p.nodes[id].flags |= NF_ZERO_ITEMS;
                    int iarr = build(*s.sub[0], f.children[0], cc);
                    p.arrays[arr].children.push_back(iarr);
                }
                p.nodes[id].end = int32_t(p.nodes.size());
                return arr;
            }
            default:
                throw std::runtime_error("fast_decode: unsupported schema in make_decoder: " + s.what);  // :212
        }
    }

    // A field outside the column projection: the nodes build() would make, in the same pre-order, flagged NF_SKIP and
    // owning nothing (no slots, streams, row spaces or arrays).  The same nesting limits apply: the walkers still go
    // through every byte of it.
    void build_skip(const AvroNode& s, const Ctx& c) {
        const AvroNode* v = &s;
        bool nullable = false, null_first = false;
        if (s.k == AK::Union) {
            if (s.sub.size() == 2 && (s.sub[0]->k == AK::Null || s.sub[1]->k == AK::Null)) {
                null_first = s.sub[0]->k == AK::Null;
                nullable = true;
                v = null_first ? s.sub[1].get() : s.sub[0].get();
                if (v->k == AK::Null || v->k == AK::Union) throw std::runtime_error("unsupported nullable inner type");
            } else {
                if (c.ulevel >= kMaxUnionLevel) throw std::runtime_error("unions nested deeper than " + std::to_string(kMaxUnionLevel));
                const int id = skip_node(c, NK_UNION, false, false);
                p.nodes[size_t(id)].aux = int32_t(s.sub.size());
                for (size_t i = 0; i < s.sub.size(); ++i) build_skip(*s.sub[i], Ctx{c.level + 1, c.ulevel + 1, int(i), 0, c.depth, false});
                p.nodes[size_t(id)].end = int32_t(p.nodes.size());
                return;
            }
        }
        auto leaf = [&](NodeKind nk, int aux) {
            const int id = skip_node(c, nk, nullable, null_first);
            p.nodes[size_t(id)].aux = aux;
            p.nodes[size_t(id)].end = id + 1;
        };
        switch (v->k) {
            case AK::Int: case AK::Date: case AK::TimeMillis: return leaf(NK_I32, 0);
            case AK::Long: case AK::TsMillis: case AK::TsMicros: case AK::TimeMicros: return leaf(NK_I64, 0);
            case AK::Bytes: return leaf(NK_BYTES, 0);
            case AK::Fixed: return leaf(NK_FIXED, v->size);
            case AK::Uuid: return leaf(NK_UUID, 16);
            case AK::DecimalBytes: return leaf(NK_DEC_BYTES, 0);
            case AK::DecimalFixed: return leaf(NK_DEC_FIXED, v->size);
            case AK::Float: return leaf(NK_F32, 0);
            case AK::Double: return leaf(NK_F64, 0);
            case AK::Bool: return leaf(NK_BOOL, 0);
            case AK::String: return leaf(NK_STR, 0);
            case AK::Enum: {
                leaf(NK_ENUM, 0);
                p.nodes.back().aux2 = int32_t(v->symbols.size());  // the index range the walk checks
                return;
            }
            case AK::Null: return leaf(NK_NULL, 0);
            case AK::Record: {
                if (v->fields.empty()) throw std::runtime_error("RecordDecoder produced a record with 0 fields");
                const int id = skip_node(c, NK_REC, nullable, null_first);
                for (auto& f : v->fields) build_skip(*f.type, Ctx{c.level + 1, c.ulevel, 0xFF, 0, c.depth, false});
                p.nodes[size_t(id)].end = int32_t(p.nodes.size());
                return;
            }
            case AK::Array: case AK::Map: {
                const bool is_map = v->k == AK::Map;
                if (c.depth + 1 > kMaxListDepth)
                    throw std::runtime_error("arrays/maps nested deeper than " + std::to_string(kMaxListDepth) + " levels are not supported");
                const int id = skip_node(c, is_map ? NK_MAP : NK_LIST, nullable, null_first);
                const Ctx cc{c.level + 1, c.ulevel, 0xFF, 0, c.depth + 1, false};
                if (is_map) {
                    skip_node(cc, NK_STR, false, false);
                    p.nodes.back().end = int32_t(p.nodes.size());
                } else if (zero_sized(*v->sub[0])) {
                    p.nodes[size_t(id)].flags |= NF_ZERO_ITEMS;
                }
                build_skip(*v->sub[0], cc);
                p.nodes[size_t(id)].end = int32_t(p.nodes.size());
                return;
            }
            default:
                throw std::runtime_error("fast_decode: unsupported schema in make_decoder: " + v->what);
        }
    }
    // ---- resolved plans (build_resolved_plan) -------------------------------------------------------------------
    // build() for the writer node rs.w read as the reader node rs.r; `f` is the reader's Arrow field.
    int build_res(const Resolution& rs, const ArrowField& f, const Ctx& c) {
        const AvroNode& w = *rs.w;
        const AvroNode& r = *rs.r;
        if (r.k == AK::Union) {
            const bool r_nullable = r.sub.size() == 2 && (r.sub[0]->k == AK::Null || r.sub[1]->k == AK::Null);
            if (r_nullable) {
                const bool wire = w.k == AK::Union;  // false: a writer non-union, never null, no branch index on the wire
                const bool null_first = wire && w.sub[0]->k == AK::Null;
                const AvroNode& wi = wire ? (null_first ? *w.sub[1] : *w.sub[0]) : w;
                if (wi.k == AK::Null || wi.k == AK::Union) throw std::runtime_error("unsupported nullable inner type");
                const int arr = build_value_res(rs.sub[0], wi, f, true, null_first, c);
                if (!wire) p.nodes[size_t(p.arrays[size_t(arr)].node)].flags &= uint8_t(~(NF_NULLABLE | NF_NULL_FIRST));
                return arr;
            }
            if (f.type != AT::SparseUnion || f.children.size() != r.sub.size()) throw std::runtime_error("union variant count mismatch");
            if (c.ulevel >= kMaxUnionLevel) throw std::runtime_error("unions nested deeper than " + std::to_string(kMaxUnionLevel));
            const int id = new_node(c, NK_UNION, false, false);
            const int arr = new_array(AT::SparseUnion, id, c.space, false);
            const int slot = add_slot(SlotRole::TypeIds, id, c.space, -1);
            p.nodes[size_t(id)].slot_a = int16_t(slot);
            p.nodes[size_t(id)].aux = int32_t(r.sub.size());
            p.arrays[size_t(arr)].slot_a = slot;
            for (size_t i = 0; i < r.sub.size(); ++i) {
                const Ctx cc{c.level + 1, c.ulevel + 1, int(i), c.space, c.depth, r.sub.size() > 1 || c.can_get_null};
                const int child = build_res(rs.sub[i], f.children[i], cc);
                p.arrays[size_t(arr)].children.push_back(child);
            }
            p.nodes[size_t(id)].end = int32_t(p.nodes.size());
            return arr;
        }
        return build_value_res(rs, w, f, false, false, c);
    }

    // build_value() for a resolved pair whose reader side is not a union; `w` is the writer's value node (inside its
    // null union when `nullable`).
    int build_value_res(const Resolution& rs, const AvroNode& w, const ArrowField& f, bool nullable, bool null_first, const Ctx& c) {
        const AvroNode& r = *rs.r;
        const bool may_null = nullable || c.can_get_null;
        if (w.k != r.k && r.k != AK::String && r.k != AK::Bytes) {  // a promotion (string <-> bytes: same wire, same buffers)
            const NodeKind from = w.k == AK::Int ? NK_I32 : (w.k == AK::Long ? NK_I64 : NK_F32);
            const NodeKind to = r.k == AK::Long ? NK_I64 : (r.k == AK::Float ? NK_F32 : NK_F64);
            const int id = new_node(c, NK_PROMOTE, nullable, null_first);
            const int arr = new_array(f.type, id, c.space, false);
            const int sa = add_slot(to == NK_F32 ? SlotRole::Values32 : SlotRole::Values64, id, c.space, -1);
            p.nodes[size_t(id)].slot_a = int16_t(sa);
            p.nodes[size_t(id)].aux = from;
            p.nodes[size_t(id)].aux2 = to;
            p.arrays[size_t(arr)].slot_a = sa;
            if (may_null) {
                const int sv = add_slot(SlotRole::Validity, id, c.space, -1);
                p.nodes[size_t(id)].slot_v = int16_t(sv);
                p.nodes[size_t(id)].flags |= NF_VALIDITY;
                p.arrays[size_t(arr)].slot_v = sv;
            }
            p.nodes[size_t(id)].end = id + 1;
            return arr;
        }
        switch (r.k) {
            case AK::Enum: {
                const int arr = build_value(w, f, nullable, null_first, c);  // the writer's index range and symbol table ...
                DNode& nd = p.nodes[size_t(p.arrays[size_t(arr)].node)];
                p.sym_bytes.resize(size_t(p.sym_off[size_t(nd.aux)]));       // ... rewritten with the reader's text for each writer index
                p.sym_off.resize(size_t(nd.aux));
                bool unmapped = false;
                for (size_t i = 0; i < w.symbols.size(); ++i) {
                    p.sym_off.push_back(int32_t(p.sym_bytes.size()));
                    if (rs.sym[i] < 0) { unmapped = true; continue; }
                    const std::string& t = r.symbols[size_t(rs.sym[i])];
                    p.sym_bytes.insert(p.sym_bytes.end(), t.begin(), t.end());
                }
                p.sym_off.push_back(int32_t(p.sym_bytes.size()));
                if (unmapped) {
                    nd.flags |= NF_ENUM_MAP;
                    for (size_t i = 0; i < w.symbols.size(); ++i) p.sym_off.push_back(rs.sym[i] < 0 ? 1 : 0);
                }
                return arr;
            }
            case AK::Record: {
                if (f.type != AT::Struct || f.children.size() != r.fields.size()) throw std::runtime_error("avro/arrow field count mismatch");
                if (r.fields.empty()) throw std::runtime_error("RecordDecoder produced a record with 0 fields");
                const int id = new_node(c, NK_REC, nullable, null_first);
                const int arr = new_array(AT::Struct, id, c.space, nullable);
                if (nullable) {
                    const int sv = add_slot(SlotRole::Validity, id, c.space, -1);
                    p.nodes[size_t(id)].slot_v = int16_t(sv);
                    p.nodes[size_t(id)].flags |= NF_VALIDITY;
                    p.arrays[size_t(arr)].slot_v = sv;
                }
                const Ctx cc{c.level + 1, c.ulevel, 0xFF, c.space, c.depth, may_null};
                const std::vector<int> out = fields_res(rs, w, f.children, cc, nullptr);
                for (int child : out) p.arrays[size_t(arr)].children.push_back(child);
                p.nodes[size_t(id)].end = int32_t(p.nodes.size());
                return arr;
            }
            case AK::Array: case AK::Map: {
                const bool is_map = r.k == AK::Map;
                if (f.type != (is_map ? AT::Map : AT::List) || f.children.size() != 1) throw std::runtime_error(is_map ? "expected Map" : "expected List");
                if (c.depth + 1 > kMaxListDepth)
                    throw std::runtime_error("arrays/maps nested deeper than " + std::to_string(kMaxListDepth) + " levels are not supported");
                if (p.n_spaces >= 250) throw std::runtime_error("schema has too many arrays/maps");
                const int id = new_node(c, is_map ? NK_MAP : NK_LIST, nullable, null_first);
                const int arr = new_array(is_map ? AT::Map : AT::List, id, c.space, nullable);
                const int so = add_slot(SlotRole::Offsets, id, c.space, -1);
                p.nodes[size_t(id)].slot_a = int16_t(so);
                p.arrays[size_t(arr)].slot_a = so;
                if (nullable) {
                    const int sv = add_slot(SlotRole::Validity, id, c.space, -1);
                    p.nodes[size_t(id)].slot_v = int16_t(sv);
                    p.nodes[size_t(id)].flags |= NF_VALIDITY;
                    p.arrays[size_t(arr)].slot_v = sv;
                }
                const int child_space = p.n_spaces++;
                const int st = add_stream(true, child_space, id);
                p.space_stream.push_back(st);
                p.space_depth.push_back(c.depth + 1);
                if (c.depth + 1 > p.max_depth) p.max_depth = c.depth + 1;
                p.nodes[size_t(id)].stream = int16_t(st);
                const Ctx cc{c.level + 1, c.ulevel, 0xFF, child_space, c.depth + 1, false};
                if (is_map) {
                    const ArrowField& entries = f.children[0];
                    if (entries.type != AT::Struct || entries.children.size() != 2)
                        throw std::runtime_error("Map entries must have exactly 2 fields (keys, values)");
                    const int earr = new_array(AT::Struct, -1, child_space, false);
                    p.arrays[size_t(arr)].children.push_back(earr);
                    AvroNode key_schema;
                    key_schema.k = AK::String;
                    const int karr = build_value(key_schema, entries.children[0], false, false, cc);  // (p.arrays grows: index after)
                    p.arrays[size_t(earr)].children.push_back(karr);
                    const int varr = build_res(rs.sub[0], entries.children[1], cc);
                    p.arrays[size_t(earr)].children.push_back(varr);
                } else {
                    if (zero_sized(*w.sub[0])) p.nodes[size_t(id)].flags |= NF_ZERO_ITEMS;
                    const int iarr = build_res(rs.sub[0], f.children[0], cc);
                    p.arrays[size_t(arr)].children.push_back(iarr);
                }
                p.nodes[size_t(id)].end = int32_t(p.nodes.size());
                return arr;
            }
            default:
                return build_value(w, f, nullable, null_first, c);  // the same type, or string <-> bytes
        }
    }

    // The fields of a resolved record: the writer's fields in wire order (read, or skipped when the reader does not have
    // them or `keep` leaves them out), then the reader-only fields' defaults.  Returns the reader fields' arrays in reader
    // order (-1 where `keep` leaves a field out).
    std::vector<int> fields_res(const Resolution& rs, const AvroNode& w, const std::vector<ArrowField>& rf, const Ctx& cc, const std::vector<int>* keep) {
        auto kept = [&](size_t j) { return !keep || std::find(keep->begin(), keep->end(), int(j)) != keep->end(); };
        std::vector<int> out(rs.src.size(), -1);
        for (size_t i = 0; i < w.fields.size(); ++i) {
            size_t j = 0;
            while (j < rs.src.size() && rs.src[j] != int(i)) ++j;
            if (j < rs.src.size() && kept(j)) out[j] = build_res(rs.sub[j], rf[j], cc);
            else build_skip(*w.fields[i].type, Ctx{cc.level, cc.ulevel, 0xFF, 0, cc.depth, false});
        }
        for (size_t j = 0; j < rs.src.size(); ++j)
            if (rs.src[j] < 0 && kept(j)) out[j] = build_default(rs.sub[j], rf[j], cc);
        return out;
    }

    // NK_DEFAULT: a reader field the writer does not have (the resolver has checked its default against its type).
    int build_default(const Resolution& rs, const ArrowField& f, const Ctx& c) {
        const AvroNode& t = *rs.r;
        if (t.k == AK::Null) {
            const int id = new_node(c, NK_NULL, false, false);
            p.nodes[size_t(id)].end = id + 1;
            return new_array(AT::Null, id, c.space, false);
        }
        if (rs.def.is_null) {  // a null of the reader's (union) type: its plain nodes, never present (NF_ABSENT), read nothing
            const int arr = build(t, f, c);
            DNode& root = p.nodes[size_t(p.arrays[size_t(arr)].node)];
            root.flags = uint8_t((root.flags & ~(NF_NULLABLE | NF_NULL_FIRST)) | NF_ABSENT);
            return arr;
        }
        const bool out_nullable = t.k == AK::Union;  // (non-null defaults: the resolver admits only [T, "null"] unions)
        const AvroNode& v = out_nullable ? *t.sub[0] : t;
        NodeKind out = NK_STR;
        SlotRole role = SlotRole::Offsets;
        switch (v.k) {
            case AK::Bool: out = NK_BOOL; role = SlotRole::Bits; break;
            case AK::Int: case AK::Date: case AK::TimeMillis: out = NK_I32; role = SlotRole::Values32; break;
            case AK::Long: case AK::TsMillis: case AK::TsMicros: case AK::TimeMicros: out = NK_I64; role = SlotRole::Values64; break;
            case AK::Float: out = NK_F32; role = SlotRole::Values32; break;
            case AK::Double: out = NK_F64; role = SlotRole::Values64; break;
            case AK::String: case AK::Bytes: case AK::Enum: break;
            default: throw std::runtime_error("default of this type is not supported");
        }
        const int id = new_node(c, NK_DEFAULT, false, false);
        const int arr = new_array(f.type, id, c.space, false);
        DNode& nd = p.nodes[size_t(id)];
        nd.pad0 = uint8_t(out);
        const int sa = add_slot(role, id, c.space, -1);
        p.nodes[size_t(id)].slot_a = int16_t(sa);
        p.arrays[size_t(arr)].slot_a = sa;
        if (out_nullable || c.can_get_null) {
            const int sv = add_slot(SlotRole::Validity, id, c.space, -1);
            p.nodes[size_t(id)].slot_v = int16_t(sv);
            p.nodes[size_t(id)].flags |= NF_VALIDITY;
            p.arrays[size_t(arr)].slot_v = sv;
        }
        uint64_t bits = 0;
        if (out == NK_F32) { const float x = float(rs.def.d); uint32_t u; std::memcpy(&u, &x, 4); bits = u; }
        else if (out == NK_F64) std::memcpy(&bits, &rs.def.d, 8);
        else bits = uint64_t(rs.def.i);
        p.nodes[size_t(id)].aux = int32_t(uint32_t(bits));
        p.nodes[size_t(id)].aux2 = int32_t(uint32_t(bits >> 32));
        if (out == NK_STR) {
            const int st = add_stream(false, c.space, id);
            const int sb = add_slot(SlotRole::Data, id, c.space, st);
            p.nodes[size_t(id)].slot_b = int16_t(sb);
            p.nodes[size_t(id)].stream = int16_t(st);
            p.arrays[size_t(arr)].slot_b = sb;
            p.nodes[size_t(id)].aux = int32_t(p.sym_off.size());
            p.nodes[size_t(id)].aux2 = 0;
            p.sym_off.push_back(int32_t(p.sym_bytes.size()));
            p.sym_bytes.insert(p.sym_bytes.end(), rs.def.bytes.begin(), rs.def.bytes.end());
            p.sym_off.push_back(int32_t(p.sym_bytes.size()));
        }
        p.nodes[size_t(id)].end = id + 1;
        return arr;
    }

    int skip_node(const Ctx& c, NodeKind kind, bool nullable, bool null_first) {
        const int id = new_node(c, kind, nullable, null_first);
        p.nodes[size_t(id)].flags |= NF_SKIP;
        return id;
    }
};

}  // namespace

Plan build_plan(const AvroNode& top, const std::vector<ArrowField>& fields, const std::vector<int>* keep) {
    if (top.k != AK::Record) throw std::runtime_error("fast_decode::decode called on non-record schema");  // :820-823
    if (top.fields.size() != fields.size()) throw std::runtime_error("avro/arrow field count mismatch");
    // RecordBatch::try_new(schema, vec![]) at fast_decode.rs:834 (arrow-rs: a batch needs a column or a row count)
    if (top.fields.empty()) throw std::runtime_error("must either specify a row count or at least one column");
    Builder b;
    b.p.space_stream.push_back(-1);
    b.p.space_depth.push_back(0);
    std::vector<int> arr_of(top.fields.size(), -1);  // field -> its top-level array (-1: skipped)
    for (size_t i = 0; i < top.fields.size(); ++i) {
        Ctx c{1, 0, 0xFF, 0, 0, false};
        const bool kept = !keep || std::find(keep->begin(), keep->end(), int(i)) != keep->end();
        if (kept) arr_of[i] = b.build(*top.fields[i].type, fields[i], c);
        else b.build_skip(*top.fields[i].type, c);
    }
    if (!keep) b.p.top_arrays = arr_of;
    else for (int f : *keep) b.p.top_arrays.push_back(arr_of.at(size_t(f)));
    return std::move(b.p);
}

Plan build_resolved_plan(const Resolution& res, const std::vector<ArrowField>& fields, const std::vector<int>* keep) {
    const AvroNode& w = *res.w;
    if (w.k != AK::Record || res.r->k != AK::Record) throw std::runtime_error("fast_decode::decode called on non-record schema");
    if (res.r->fields.size() != fields.size()) throw std::runtime_error("avro/arrow field count mismatch");
    if (res.r->fields.empty() || w.fields.empty()) throw std::runtime_error("must either specify a row count or at least one column");
    Builder b;
    b.p.space_stream.push_back(-1);
    b.p.space_depth.push_back(0);
    const std::vector<int> arr_of = b.fields_res(res, w, fields, Ctx{1, 0, 0xFF, 0, 0, false}, keep);
    if (!keep) b.p.top_arrays = arr_of;
    else for (int f : *keep) b.p.top_arrays.push_back(arr_of.at(size_t(f)));
    return std::move(b.p);
}

}  // namespace rv
