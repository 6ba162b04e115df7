// See schema.hpp for the reference lines each function mirrors.
#include "schema.hpp"

#include <algorithm>
#include <array>
#include <cerrno>
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <map>
#include <set>
#include <stdexcept>

#include "json.hpp"

namespace rv {
namespace {

[[noreturn]] void bad(const std::string& what) { throw std::runtime_error("invalid Avro schema: " + what); }

std::unique_ptr<AvroNode> mk(AK k) {
    auto n = std::make_unique<AvroNode>();
    n->k = k;
    return n;
}
std::unique_ptr<AvroNode> unsupported(const std::string& what) {
    auto n = mk(AK::Unsupported);
    n->what = what;
    return n;
}

std::unique_ptr<AvroNode> clone_node(const AvroNode& n) {
    auto c = std::make_unique<AvroNode>();
    c->k = n.k; c->fullname = n.fullname; c->has_doc = n.has_doc; c->doc = n.doc; c->has_aliases = n.has_aliases;
    c->aliases = n.aliases; c->symbols = n.symbols; c->what = n.what; c->size = n.size; c->precision = n.precision; c->scale = n.scale;
    c->has_enum_default = n.has_enum_default; c->enum_default = n.enum_default;
    for (auto& f : n.fields) {
        AvroField cf;
        cf.name = f.name; cf.has_doc = f.has_doc; cf.doc = f.doc; cf.dflt = f.dflt; cf.aliases = f.aliases;
        cf.type = clone_node(*f.type);
        c->fields.push_back(std::move(cf));
    }
    for (auto& s : n.sub) c->sub.push_back(clone_node(*s));
    return c;
}

// Named types seen so far (record / enum / fixed), for references by name (apache_avro Schema::Ref): a reference
// decodes exactly like the definition it names, so it is replaced by a copy of it.  A name that is still being
// defined (a recursive type) has no finite Arrow type and stays unsupported.
struct Names {
    std::map<std::string, const AvroNode*> done;
    std::set<std::string> open;
};

// [A-Za-z_][A-Za-z0-9_]* — what apache-avro's validators ask of a type's short name, a record field's name and an enum
// symbol (validate_schema_name / validate_record_field_name / validate_enum_symbol_name: the specification's names).
bool is_identifier(const std::string& s) {
    if (s.empty()) return false;
    for (size_t i = 0; i < s.size(); ++i) {
        const unsigned char c = static_cast<unsigned char>(s[i]);
        const bool alpha = (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || c == '_';
        if (!(alpha || (i > 0 && c >= '0' && c <= '9'))) return false;
    }
    return true;
}

// Name resolution as apache-avro does it: a dotted name carries its own namespace,
// otherwise the "namespace" attribute, otherwise the enclosing namespace.
void resolve_name(const Json& j, const std::string& enclosing_ns, std::string* fullname, std::string* ns) {
    const Json* nm = j.find("name");
    if (!nm || !nm->is_string() || nm->str.empty()) bad("named type without a \"name\"");
    const std::string& name = nm->str;
    size_t dot = name.rfind('.');
    // Name::new -> validate_schema_name: the part behind the last dot is an identifier; the namespace part in front of it
    // is made of identifier characters and dots and does not start with a digit.  (Only what every published form of
    // that pattern rejects is rejected here.)
    if (!is_identifier(dot == std::string::npos ? name : name.substr(dot + 1))) bad("invalid name \"" + name + "\" (must match [A-Za-z_][A-Za-z0-9_]*, optionally behind a dotted namespace)");
    if (dot != std::string::npos)
        for (size_t i = 0; i < dot; ++i) {
            const unsigned char c = static_cast<unsigned char>(name[i]);
            const bool ok = (c >= 'A' && c <= 'Z') || (c >= 'a' && c <= 'z') || c == '_' || c == '.' || (i > 0 && c >= '0' && c <= '9');
            if (!ok) bad("invalid namespace in the name \"" + name + "\"");
        }
    std::string shortname;
    if (dot != std::string::npos) {
        *ns = name.substr(0, dot);
        shortname = name.substr(dot + 1);
    } else {
        const Json* nsj = j.find("namespace");
        *ns = (nsj && nsj->is_string()) ? nsj->str : enclosing_ns;
        shortname = name;
    }
    *fullname = ns->empty() ? shortname : *ns + "." + shortname;
}

void read_doc_aliases(const Json& j, const std::string& ns, AvroNode* n) {
    if (const Json* d = j.find("doc"); d && d->is_string()) { n->has_doc = true; n->doc = d->str; }
    if (const Json* a = j.find("aliases"); a && a->kind == Json::Array) {
        // (an "aliases" array with anything but strings in it is no aliases at all: apache-avro collects them into an
        // Option and drops the lot, it does not fail)
        bool all_strings = true;
        for (auto& al : a->arr) all_strings = all_strings && al.is_string();
        if (all_strings) {
            n->has_aliases = true;
            for (auto& al : a->arr) {
                if (al.str.find('.') == std::string::npos && !ns.empty()) n->aliases.push_back(ns + "." + al.str);
                else n->aliases.push_back(al.str);
            }
        }
    }
}

// "precision" / "scale" of a decimal as apache-avro reads them (parse_json_integer_for_decimal): a JSON number that is a
// non-negative integer ("4", not "4.0", "-4" or "4e0").  -1: anything else.
long long decimal_meta(const Json* j) {
    if (!j || j->kind != Json::Number || j->str.empty() || j->str.size() > 9) return -1;
    for (char c : j->str)
        if (c < '0' || c > '9') return -1;
    return std::strtoll(j->str.c_str(), nullptr, 10);
}

// nullptr: the decimal annotation is invalid.  apache-avro then IGNORES the logical type ("Ignoring invalid decimal logical
// type", a warning) and the schema is the underlying bytes / fixed — it does not fail, and it never guesses a scale.
std::unique_ptr<AvroNode> decimal_of(AK k, const Json* obj, int size) {
    const Json* pj = obj ? obj->find("precision") : nullptr;
    const Json* sj = obj ? obj->find("scale") : nullptr;
    const long long p = decimal_meta(pj);
    const long long sc = sj ? decimal_meta(sj) : 0;   // (only "scale" may be absent: 0)
    if (p < 1 || sc < 0 || sc > p) return nullptr;
    const int precision = int(p), scale = int(sc);
    if (precision > 38) return unsupported("decimal with precision above 38 (Decimal128)");
    if (k == AK::DecimalFixed && size > 16) return unsupported("decimal on a fixed wider than 16 bytes");
    auto n = mk(k);
    n->precision = precision; n->scale = scale; n->size = size;
    return n;
}

std::unique_ptr<AvroNode> primitive(const std::string& t, const Json* obj, const std::string& ns, Names& names) {
    std::string lt;
    if (obj)
        if (const Json* l = obj->find("logicalType"); l && l->is_string()) lt = l->str;
    if (t == "null") return mk(AK::Null);
    if (t == "boolean") return mk(AK::Bool);
    if (t == "float") return mk(AK::Float);
    if (t == "double") return mk(AK::Double);
    if (t == "int") {
        if (lt == "date") return mk(AK::Date);
        if (lt == "time-millis") return mk(AK::TimeMillis);
        return mk(AK::Int);  // unknown logical types degrade to the base type
    }
    if (t == "long") {
        if (lt == "timestamp-millis") return mk(AK::TsMillis);
        if (lt == "timestamp-micros") return mk(AK::TsMicros);
        if (lt == "time-micros") return mk(AK::TimeMicros);
        if (lt == "timestamp-nanos" || lt == "local-timestamp-millis" || lt == "local-timestamp-micros" || lt == "local-timestamp-nanos")
            return unsupported(lt);
        return mk(AK::Long);
    }
    if (t == "string") {
        if (lt == "uuid") return mk(AK::Uuid);
        return mk(AK::String);
    }
    if (t == "bytes") {
        if (lt == "decimal")
            if (auto d = decimal_of(AK::DecimalBytes, obj, 0)) return d;
        return mk(AK::Bytes);
    }
    // a reference to a named type defined earlier in the document (Schema::Ref)
    for (const std::string& cand : {t.find('.') == std::string::npos && !ns.empty() ? ns + "." + t : t, t}) {
        if (names.open.count(cand)) return unsupported("recursive reference to named type \"" + cand + "\"");
        auto it = names.done.find(cand);
        if (it != names.done.end()) return clone_node(*it->second);
    }
    return unsupported("reference to unknown named type \"" + t + "\"");
}

// Key used for the "unions may not contain duplicate types" rule.
std::string union_key(const AvroNode& n) {
    switch (n.k) {
        // (UnionSchema::new checks kinds that are not named: record / enum / fixed / a reference may repeat, even under one
        // name.  A decimal on a fixed is let through like the fixed it sits on — whether the library counts it as a kind of
        // its own is not settled by anything in the reference tree, and turning away a document it takes would be worse)
        case AK::Record: case AK::Enum: case AK::Fixed: case AK::DecimalFixed: return std::string();
        case AK::Unsupported: return "unsupported:" + n.what;
        default: return "kind:" + std::to_string(int(n.k));
    }
}

bool is_named_ref(const std::string& t, const std::string& ns, const Names& names) {
    static const std::set<std::string> builtin = {"null", "boolean", "int", "long", "float", "double", "bytes", "string", "array", "map", "enum", "record", "error", "fixed"};
    if (builtin.count(t)) return false;
    const std::string q = t.find('.') == std::string::npos && !ns.empty() ? ns + "." + t : t;
    return names.done.count(q) || names.open.count(q) || names.done.count(t) || names.open.count(t);
}

std::unique_ptr<AvroNode> parse_node(const Json& j, const std::string& ns, int depth, Names& names) {
    if (depth > 64) bad("schema nesting too deep");
    if (j.kind == Json::String) return primitive(j.str, nullptr, ns, names);
    if (j.kind == Json::Array) {
        auto u = mk(AK::Union);
        std::set<std::string> seen;
        for (auto& v : j.arr) {
            auto c = parse_node(v, ns, depth + 1, names);
            if (c->k == AK::Union) bad("unions may not immediately contain other unions");
            const std::string key = union_key(*c);
            if (!key.empty() && !seen.insert(key).second) bad("unions cannot contain duplicate types");
            u->sub.push_back(std::move(c));
        }
        if (u->sub.empty()) bad("empty union");
        return u;
    }
    if (j.kind != Json::Object) bad("a schema must be a string, array or object");
    const Json* t = j.find("type");
    if (!t) bad("object schema without \"type\"");
    if (!t->is_string()) return parse_node(*t, ns, depth + 1, names);
    const std::string& ts = t->str;
    if (ts == "record" || ts == "error") {
        auto r = mk(AK::Record);
        std::string rns;
        resolve_name(j, ns, &r->fullname, &rns);
        read_doc_aliases(j, rns, r.get());
        names.open.insert(r->fullname);
        const Json* fs = j.find("fields");
        if (!fs || fs->kind != Json::Array) bad("record without a \"fields\" array");
        for (auto& fj : fs->arr) {
            if (fj.kind != Json::Object) bad("record field must be an object");
            AvroField f;
            const Json* fn = fj.find("name");
            const Json* ft = fj.find("type");
            if (!fn || !fn->is_string() || !ft) bad("record field needs \"name\" and \"type\"");
            f.name = fn->str;
            if (!is_identifier(f.name)) bad("invalid record field name \"" + f.name + "\" (must match [A-Za-z_][A-Za-z0-9_]*)");   // validate_record_field_name
            for (const AvroField& earlier : r->fields)
                if (earlier.name == f.name) bad("duplicate record field name \"" + f.name + "\"");   // Error::FieldNameDuplicate
            // apache-avro 0.21 parses a record field by handing the FIELD object to its complex-type parser
            // (RecordField::parse -> Parser::parse_complex(field, ..)), so when "type" is a bare string the
            // attributes of that type are read from the field object itself: {"name":"xs","type":"array","items":..}
            // is an array (the reference relies on it: ruhvro/src/serialize.rs:185-186), an "enum" takes the field's
            // name and "symbols", and a field-level "logicalType" annotates a primitive.  A bare "record" there is a
            // look-up of an already defined type by the field's name: a named reference, which the gate rejects.
            if (ft->is_string() && ft->str != "record" && ft->str != "error" && ft->str != "fixed" && !is_named_ref(ft->str, rns, names))
                f.type = parse_node(fj, rns, depth + 1, names);
            else if (ft->is_string() && ft->str == "fixed") f.type = parse_node(fj, rns, depth + 1, names);  // {"name":..,"type":"fixed","size":..}: the field object is the fixed
            else f.type = parse_node(*ft, rns, depth + 1, names);
            if (const Json* d = fj.find("doc"); d && d->is_string()) { f.has_doc = true; f.doc = d->str; }
            if (const Json* d = fj.find("default")) f.dflt = std::make_shared<const Json>(*d);   // (checked when a resolution uses it)
            if (const Json* a = fj.find("aliases"); a && a->kind == Json::Array)
                for (auto& al : a->arr)
                    if (al.is_string()) f.aliases.push_back(al.str);
            r->fields.push_back(std::move(f));
        }
        names.open.erase(r->fullname);
        names.done[r->fullname] = r.get();
        return r;
    }
    if (ts == "enum") {
        auto e = mk(AK::Enum);
        std::string ens;
        resolve_name(j, ns, &e->fullname, &ens);
        read_doc_aliases(j, ens, e.get());
        const Json* sy = j.find("symbols");
        if (!sy || sy->kind != Json::Array) bad("enum without a \"symbols\" array");
        for (auto& s : sy->arr) {
            if (!s.is_string()) bad("enum symbols must be strings");
            if (!is_identifier(s.str)) bad("invalid enum symbol \"" + s.str + "\" (must match [A-Za-z_][A-Za-z0-9_]*)");   // validate_enum_symbol_name
            for (const std::string& earlier : e->symbols)
                if (earlier == s.str) bad("duplicate enum symbol \"" + s.str + "\"");   // Error::EnumSymbolDuplicate
            e->symbols.push_back(s.str);
        }
        if (const Json* d = j.find("default")) {   // Error::EnumDefaultWrongType / Error::GetEnumDefault
            if (!d->is_string()) bad("enum default must be a string");
            if (std::find(e->symbols.begin(), e->symbols.end(), d->str) == e->symbols.end()) bad("enum default \"" + d->str + "\" is not one of the symbols");
            e->has_enum_default = true;
            e->enum_default = d->str;
        }
        names.done[e->fullname] = e.get();
        return e;
    }
    if (ts == "fixed") {
        std::string fullname, fns;
        resolve_name(j, ns, &fullname, &fns);
        const long long size_ll = decimal_meta(j.find("size"));   // a JSON number that is a non-negative integer (as_u64)
        if (size_ll < 0) bad("fixed without a non-negative \"size\"");
        const int size = int(size_ll);
        std::string lt;
        if (const Json* l = j.find("logicalType"); l && l->is_string()) lt = l->str;
        std::unique_ptr<AvroNode> f;
        if (lt == "decimal") f = decimal_of(AK::DecimalFixed, &j, size);
        else if (lt == "duration") f = unsupported("duration");
        if (!f) { f = mk(AK::Fixed); f->size = size; }
        f->fullname = fullname;
        read_doc_aliases(j, fns, f.get());
        if (f->k != AK::Unsupported) names.done[fullname] = f.get();
        return f;
    }
    if (ts == "array" || ts == "map") {
        auto a = mk(ts == "array" ? AK::Array : AK::Map);
        const Json* it = j.find(ts == "array" ? "items" : "values");
        if (!it) bad(ts == "array" ? "array without \"items\"" : "map without \"values\"");
        a->sub.push_back(parse_node(*it, ns, depth + 1, names));
        return a;
    }
    return primitive(ts, &j, ns, names);
}

bool supported_inner(const AvroNode& n, std::string* why) {
    switch (n.k) {
        case AK::Int: case AK::Long: case AK::Float: case AK::Double: case AK::Bool: case AK::String: case AK::Null:
        case AK::Date: case AK::TsMillis: case AK::TsMicros: case AK::Enum:
        case AK::Bytes: case AK::DecimalBytes: case AK::Uuid: case AK::TimeMillis: case AK::TimeMicros:
            return true;
        case AK::Fixed: case AK::DecimalFixed:
            // a fixed of size 0 spends no wire bytes: an 8-byte list header could then announce 2^31 items, each of them
            // walked — unbounded work for bounded input.  (The reference's fast path takes no fixed at all.)
            if (n.size == 0) { if (why) *why = "fixed of size 0"; return false; }
            return true;
        case AK::Record:
            for (auto& f : n.fields)
                if (!supported_inner(*f.type, why)) return false;
            return true;
        case AK::Union: case AK::Array: case AK::Map:
            for (auto& s : n.sub)
                if (!supported_inner(*s, why)) return false;
            return true;
        default:
            if (why) *why = n.what;
            return false;
    }
}

// ---- schema_translate.rs ----------------------------------------------------

const char* default_field_name(AT t) {  // :155-220
    switch (t) {
        case AT::Null: return "null";
        case AT::Bool: return "bit";
        case AT::Int32: return "int";
        case AT::Int64: return "bigint";
        case AT::Float32: return "float4";
        case AT::Float64: return "float8";
        case AT::Date32: return "dateday";
        case AT::TsMs: return "timestampmilli";
        case AT::TsUs: return "timestampmicro";
        case AT::Utf8: return "varchar";
        case AT::Binary: return "varbinary";
        case AT::FixedSizeBinary: return "fixedsizebinary";
        case AT::Decimal128: return "decimal";
        case AT::Time32Ms: return "timemilli";
        case AT::Time64Us: return "timemicro";
        case AT::List: return "list";
        case AT::Struct: return "struct";
        case AT::SparseUnion: return "union";
        case AT::Map: throw std::runtime_error("a map cannot be an unnamed union variant (reference: default_field_name is unimplemented for Map, schema_translate.rs:212)");
    }
    return "";
}

using Props = std::vector<std::pair<std::string, std::string>>;

// schema_to_field_with_props, :43-153.  `name == nullptr` means None.
ArrowField to_field(const AvroNode& s, const std::string* name, bool nullable, const Props* props) {
    ArrowField f;
    switch (s.k) {
        case AK::Null: f.type = AT::Null; break;
        case AK::Bool: f.type = AT::Bool; break;
        case AK::Int: f.type = AT::Int32; break;
        case AK::Long: f.type = AT::Int64; break;
        case AK::Float: f.type = AT::Float32; break;
        case AK::Double: f.type = AT::Float64; break;
        case AK::String: f.type = AT::Utf8; break;
        case AK::Date: f.type = AT::Date32; break;
        case AK::TsMillis: f.type = AT::TsMs; break;
        case AK::TsMicros: f.type = AT::TsUs; break;
        case AK::Bytes: f.type = AT::Binary; break;                                        // :58
        case AK::Fixed: f.type = AT::FixedSizeBinary; f.width = s.size; break;             // :133
        case AK::Uuid: f.type = AT::FixedSizeBinary; f.width = 16; break;                  // :137
        case AK::DecimalBytes: case AK::DecimalFixed:                                      // :134-136
            f.type = AT::Decimal128; f.precision = s.precision; f.scale = s.scale; break;
        case AK::TimeMillis: f.type = AT::Time32Ms; break;                                 // :139
        case AK::TimeMicros: f.type = AT::Time64Us; break;                                 // :140
        case AK::Array: {  // :60-65
            f.type = AT::List;
            std::string item = "item";
            f.children.push_back(to_field(*s.sub[0], &item, true, nullptr));
            break;
        }
        case AK::Map: {  // :66-75
            f.type = AT::Map;
            std::string vname = "values";
            ArrowField value = to_field(*s.sub[0], &vname, false, nullptr);
            ArrowField key;
            key.name = "keys"; key.type = AT::Utf8; key.nullable = false;
            ArrowField entries;
            entries.name = "entries"; entries.type = AT::Struct; entries.nullable = nullable;  // sic: the map's own nullability
            entries.children.push_back(std::move(key));
            entries.children.push_back(std::move(value));
            f.children.push_back(std::move(entries));
            break;
        }
        case AK::Union: {  // :76-105
            bool has_null = false;
            for (auto& v : s.sub) has_null |= v->k == AK::Null;
            if (has_null && s.sub.size() == 2) {
                nullable = true;
                const AvroNode* inner = nullptr;
                for (auto& v : s.sub)
                    if (v->k != AK::Null) { inner = v.get(); break; }
                if (!inner) throw std::runtime_error("Avro union contains duplicate null variants");
                ArrowField in = to_field(*inner, nullptr, true, nullptr);
                f.type = in.type;
                f.children = std::move(in.children);
                f.width = in.width; f.precision = in.precision; f.scale = in.scale;
            } else {
                if (has_null) nullable = true;
                if (s.sub.size() > 127) throw std::runtime_error("union with more than 127 variants (Arrow type ids are i8)");
                f.type = AT::SparseUnion;
                for (auto& v : s.sub) f.children.push_back(to_field(*v, nullptr, true, nullptr));
            }
            break;
        }
        case AK::Record: {  // :106-123
            f.type = AT::Struct;
            for (auto& fld : s.fields) {
                Props p;
                if (fld.has_doc) p.emplace_back("avro::doc", fld.doc);
                f.children.push_back(to_field(*fld.type, &fld.name, nullable, &p));
            }
            break;
        }
        case AK::Enum: {  // :124-132 — early return: metadata is never attached
            f.type = AT::Utf8;
            f.name = (name && !name->empty()) ? *name : s.fullname;
            f.nullable = nullable;
            return f;
        }
        case AK::Unsupported:
            throw std::runtime_error("schema construct outside the direct-decode subset: " + s.what);
    }
    f.name = name ? *name : std::string(default_field_name(f.type));
    f.nullable = nullable;
    if (props) f.metadata = *props;
    return f;
}

Props external_props(const AvroNode& s) {  // :222-266
    Props p;
    if (s.k == AK::Record || s.k == AK::Enum || s.k == AK::Fixed || s.k == AK::DecimalFixed) {
        if (s.has_doc) p.emplace_back("avro::doc", s.doc);
        if (s.has_aliases) {
            std::string joined = "[";
            for (size_t i = 0; i < s.aliases.size(); ++i) {
                if (i) joined += ",";
                joined += s.aliases[i];
            }
            joined += "]";
            p.emplace_back("avro::aliases", joined);
        }
    }
    return p;
}

// ---- Arrow C schema export ----------------------------------------------------

struct SchemaPrivate {
    std::string format, name, metadata;
    std::vector<ArrowSchema> child_storage;
    std::vector<ArrowSchema*> child_ptrs;
};

void release_schema(ArrowSchema* s) {
    if (!s || !s->release) return;
    for (int64_t i = 0; i < s->n_children; ++i)
        if (s->children[i] && s->children[i]->release) s->children[i]->release(s->children[i]);
    delete static_cast<SchemaPrivate*>(s->private_data);
    s->release = nullptr;
}

std::string format_of(const ArrowField& f) {
    switch (f.type) {
        case AT::Null: return "n";
        case AT::Bool: return "b";
        case AT::Int32: return "i";
        case AT::Int64: return "l";
        case AT::Float32: return "f";
        case AT::Float64: return "g";
        case AT::Utf8: return "u";
        case AT::Binary: return "z";
        case AT::FixedSizeBinary: return "w:" + std::to_string(f.width);
        case AT::Decimal128: return "d:" + std::to_string(f.precision) + "," + std::to_string(f.scale);
        case AT::Time32Ms: return "ttm";
        case AT::Time64Us: return "ttu";
        case AT::Date32: return "tdD";
        case AT::TsMs: return "tsm:";
        case AT::TsUs: return "tsu:";
        case AT::Struct: return "+s";
        case AT::List: return "+l";
        case AT::Map: return "+m";
        case AT::SparseUnion: {
            std::string s = "+us:";
            for (size_t i = 0; i < f.children.size(); ++i) {
                if (i) s += ",";
                s += std::to_string(i);
            }
            return s;
        }
    }
    return "n";
}

void put_i32(std::string& o, int32_t v) { o.append(reinterpret_cast<const char*>(&v), 4); }

void fill_schema(const ArrowField& f, ArrowSchema* out) {
    auto* p = new SchemaPrivate();
    p->format = format_of(f);
    p->name = f.name;
    if (!f.metadata.empty()) {
        put_i32(p->metadata, int32_t(f.metadata.size()));
        for (auto& kv : f.metadata) {
            put_i32(p->metadata, int32_t(kv.first.size())); p->metadata += kv.first;
            put_i32(p->metadata, int32_t(kv.second.size())); p->metadata += kv.second;
        }
    }
    p->child_storage.resize(f.children.size());
    p->child_ptrs.resize(f.children.size());
    for (size_t i = 0; i < f.children.size(); ++i) {
        fill_schema(f.children[i], &p->child_storage[i]);
        p->child_ptrs[i] = &p->child_storage[i];
    }
    out->format = p->format.c_str();
    out->name = p->name.c_str();
    out->metadata = p->metadata.empty() ? nullptr : p->metadata.data();
    out->flags = f.nullable ? ARROW_FLAG_NULLABLE : 0;
    out->n_children = int64_t(f.children.size());
    out->children = p->child_ptrs.empty() ? nullptr : p->child_ptrs.data();
    out->dictionary = nullptr;
    out->release = release_schema;
    out->private_data = p;
}

}  // namespace

std::unique_ptr<AvroNode> parse_avro_schema(const char* json, size_t len) {
    JsonReader rd(json, len);
    Json doc = rd.parse_document();
    Names names;
    return parse_node(doc, std::string(), 0, names);
}

bool is_supported(const AvroNode& top, std::string* why) {
    if (top.k != AK::Record) {
        if (why) *why = "top-level schema is not a record";
        return false;
    }
    return supported_inner(top, why);
}

std::vector<ArrowField> to_arrow_fields(const AvroNode& top) {
    std::vector<ArrowField> out;
    if (top.k != AK::Record) throw std::runtime_error("top-level schema must be a record");
    for (auto& f : top.fields) {
        Props p = external_props(*f.type);
        out.push_back(to_field(*f.type, &f.name, false, &p));
    }
    return out;
}

void export_arrow_schema(const std::vector<ArrowField>& fields, ArrowSchema* out) {
    ArrowField top;
    top.name = "";
    top.type = AT::Struct;
    top.nullable = false;
    top.children = fields;
    fill_schema(top, out);
}

std::vector<int> select_columns(const std::vector<std::string>& available, const std::vector<std::string>& requested) {
    if (requested.empty()) throw std::invalid_argument("column projection: the column list is empty");
    std::vector<int> out;
    std::set<std::string> seen;
    for (const std::string& name : requested) {
        if (!seen.insert(name).second) throw std::invalid_argument("column projection: column '" + name + "' is requested twice");
        const auto it = std::find(available.begin(), available.end(), name);
        if (it == available.end()) {
            std::string avail = "[";
            for (size_t i = 0; i < available.size(); ++i) { if (i) avail += ", "; avail += "\"" + available[i] + "\""; }
            throw std::invalid_argument("column projection: no top-level field '" + name + "'. Available fields: " + avail + "]");
        }
        out.push_back(int(it - available.begin()));
    }
    return out;
}

// ---- schema resolution ----------------------------------------------------------------------------------------------
namespace {

[[noreturn]] void unresolvable(const std::string& path, const std::string& what) {
    throw std::runtime_error("schema resolution: " + (path.empty() ? std::string("top-level record") : "field '" + path + "'") + ": " + what);
}

const char* kind_text(const AvroNode& n) {
    switch (n.k) {
        case AK::Null: return "null";
        case AK::Bool: return "boolean";
        case AK::Int: return "int";
        case AK::Long: return "long";
        case AK::Float: return "float";
        case AK::Double: return "double";
        case AK::String: return "string";
        case AK::Bytes: return "bytes";
        case AK::Date: return "date";
        case AK::TsMillis: return "timestamp-millis";
        case AK::TsMicros: return "timestamp-micros";
        case AK::TimeMillis: return "time-millis";
        case AK::TimeMicros: return "time-micros";
        case AK::Uuid: return "uuid";
        case AK::DecimalBytes: case AK::DecimalFixed: return "decimal";
        case AK::Fixed: return "fixed";
        case AK::Enum: return "enum";
        case AK::Record: return "record";
        case AK::Array: return "array";
        case AK::Map: return "map";
        case AK::Union: return "union";
        default: return "unsupported type";
    }
}

bool is_logical(AK k) {
    return k == AK::Date || k == AK::TsMillis || k == AK::TsMicros || k == AK::TimeMillis || k == AK::TimeMicros || k == AK::Uuid ||
           k == AK::DecimalBytes || k == AK::DecimalFixed;
}

// ["null", T] or [T, "null"]: T; otherwise nullptr
const AvroNode* nullable_inner(const AvroNode& n) {
    if (n.k != AK::Union || n.sub.size() != 2) return nullptr;
    if (n.sub[0]->k == AK::Null) return n.sub[1].get();
    if (n.sub[1]->k == AK::Null) return n.sub[0].get();
    return nullptr;
}

std::string short_name(const std::string& full) {
    const size_t dot = full.rfind('.');
    return dot == std::string::npos ? full : full.substr(dot + 1);
}

// Named types match when the unqualified names are equal or the reader lists the writer's name among its aliases.
bool names_match(const AvroNode& w, const AvroNode& r) {
    if (short_name(w.fullname) == short_name(r.fullname)) return true;
    for (const std::string& a : r.aliases)
        if (a == w.fullname || short_name(a) == short_name(w.fullname)) return true;
    return false;
}

// Zero wire bytes and no buffers (plan.cpp's zero_sized): a list of such items is never iterated.
bool takes_no_bytes(const AvroNode& s) {
    if (s.k == AK::Null) return true;
    if (s.k == AK::Record) {
        for (auto& f : s.fields)
            if (!takes_no_bytes(*f.type)) return false;
        return true;
    }
    return false;
}

bool json_integer(const Json& j, int64_t lo, int64_t hi, int64_t* out) {
    if (j.kind != Json::Number || j.str.empty() || j.str.find_first_of(".eE") != std::string::npos) return false;
    errno = 0;
    char* end = nullptr;
    const long long v = std::strtoll(j.str.c_str(), &end, 10);
    if (errno || !end || *end || v < lo || v > hi) return false;
    *out = v;
    return true;
}

DefaultValue default_of(const AvroNode& t, const Json* j, const std::string& path) {
    if (!j) unresolvable(path, "the writer's schema has no such field and the reader's has no \"default\" for it");
    DefaultValue d;
    const AvroNode* v = &t;
    // A union's default belongs to its first branch.  A null one is a null of the reader's type, whatever the other
    // branches are (a null record, list, map, fixed, ...: plan.cpp builds it as a subtree that is never present).
    if (t.k == AK::Null || (t.k == AK::Union && t.sub[0]->k == AK::Null)) {
        if (j->kind != Json::Null) unresolvable(path, std::string("the default does not match the field's type (") + (t.k == AK::Null ? "null" : "union whose first branch is null") + ")");
        d.is_null = true;
        return d;
    }
    if (t.k == AK::Union) {
        const AvroNode* in = nullable_inner(t);
        if (!in) unresolvable(path, "default of union is not supported (a non-null default needs [T, \"null\"])");
        v = in;
    }
    switch (v->k) {  // the value of the default: leaves only
        case AK::Record: case AK::Array: case AK::Map: case AK::Fixed: case AK::DecimalBytes: case AK::DecimalFixed: case AK::Uuid:
            unresolvable(path, std::string("default of ") + kind_text(*v) + " is not supported");
        default: break;
    }
    auto mismatch = [&]() { unresolvable(path, std::string("the default does not match the field's type (") + kind_text(*v) + ")"); };
    switch (v->k) {
        case AK::Bool:
            if (j->kind != Json::Bool) mismatch();
            d.i = j->b ? 1 : 0;
            break;
        case AK::Int: case AK::Date: case AK::TimeMillis:
            if (!json_integer(*j, INT32_MIN, INT32_MAX, &d.i)) mismatch();
            break;
        case AK::Long: case AK::TsMillis: case AK::TsMicros: case AK::TimeMicros:
            if (!json_integer(*j, INT64_MIN, INT64_MAX, &d.i)) mismatch();
            break;
        case AK::Float: case AK::Double: {
            if (j->kind != Json::Number) mismatch();
            char* end = nullptr;
            errno = 0;
            d.d = std::strtod(j->str.c_str(), &end);
            if (!end || *end) mismatch();
            // A number beyond the double range (1e400) is not a JSON number other Avro libraries read: serde_json refuses
            // it.  Underflow (1e-400 -> 0, 5e-325 -> a subnormal) is accepted, as there.
            if (errno == ERANGE && std::isinf(d.d)) mismatch();
            break;
        }
        case AK::String:
            if (!j->is_string()) mismatch();
            d.bytes = j->str;
            break;
        case AK::Bytes: {  // a JSON string of code points 0-255, one byte each
            if (!j->is_string()) mismatch();
            const std::string& u = j->str;
            for (size_t i = 0; i < u.size();) {
                const unsigned char c0 = static_cast<unsigned char>(u[i]);
                if (c0 < 0x80) { d.bytes.push_back(char(c0)); i += 1; continue; }
                if ((c0 & 0xE0) != 0xC0 || i + 1 >= u.size()) mismatch();   // 2-byte UTF-8 sequences reach U+07FF
                const unsigned cp = ((c0 & 0x1Fu) << 6) | (static_cast<unsigned char>(u[i + 1]) & 0x3Fu);
                if (cp > 0xFF) mismatch();
                d.bytes.push_back(char(cp));
                i += 2;
            }
            break;
        }
        case AK::Enum:
            if (!j->is_string() || std::find(v->symbols.begin(), v->symbols.end(), j->str) == v->symbols.end()) mismatch();
            d.bytes = j->str;
            break;
        default:
            mismatch();
    }
    return d;
}

Resolution resolve_node(const AvroNode& w, const AvroNode& r, const std::string& path) {
    Resolution res;
    res.w = &w;
    res.r = &r;
    auto unsupported_pair = [&]() {
        unresolvable(path, std::string("a writer ") + kind_text(w) + " cannot be read as a reader " + kind_text(r));
    };
    if (r.k == AK::Union) {
        if (const AvroNode* ri = nullable_inner(r)) {
            if (w.k == AK::Union) {
                const AvroNode* wi = nullable_inner(w);
                if (!wi) unresolvable(path, "union branches added, removed or reordered are not supported");
                res.sub.push_back(resolve_node(*wi, *ri, path));
            } else {
                if (w.k == AK::Null) unresolvable(path, "a writer null read as a reader union is not supported");
                res.sub.push_back(resolve_node(w, *ri, path));
            }
            return res;
        }
        if (w.k != AK::Union || w.sub.size() != r.sub.size() || nullable_inner(w))
            unresolvable(path, "union branches added, removed or reordered are not supported");
        for (size_t i = 0; i < r.sub.size(); ++i) res.sub.push_back(resolve_node(*w.sub[i], *r.sub[i], path));
        return res;
    }
    if (w.k == AK::Union) unresolvable(path, "a writer union read as a reader non-union is not supported");
    if (w.k != r.k) {
        if (is_logical(w.k) || is_logical(r.k)) unresolvable(path, std::string("promotions between logical types are not supported (writer ") + kind_text(w) + ", reader " + kind_text(r) + ")");
        const bool ok = (w.k == AK::Int && (r.k == AK::Long || r.k == AK::Float || r.k == AK::Double)) ||
                        (w.k == AK::Long && (r.k == AK::Float || r.k == AK::Double)) || (w.k == AK::Float && r.k == AK::Double) ||
                        (w.k == AK::String && r.k == AK::Bytes) || (w.k == AK::Bytes && r.k == AK::String);
        if (!ok) unsupported_pair();
        return res;
    }
    switch (r.k) {
        case AK::Fixed: case AK::DecimalFixed:
            if (!names_match(w, r)) unresolvable(path, "fixed \"" + w.fullname + "\" does not match \"" + r.fullname + "\"");
            if (w.size != r.size) unresolvable(path, "fixed sizes differ");
            if (w.precision != r.precision || w.scale != r.scale) unresolvable(path, "decimal precision or scale differ");
            return res;
        case AK::DecimalBytes:
            if (w.precision != r.precision || w.scale != r.scale) unresolvable(path, "decimal precision or scale differ");
            return res;
        case AK::Enum: {
            if (!names_match(w, r)) unresolvable(path, "enum \"" + w.fullname + "\" does not match \"" + r.fullname + "\"");
            int dflt = -1;
            if (r.has_enum_default) dflt = int(std::find(r.symbols.begin(), r.symbols.end(), r.enum_default) - r.symbols.begin());
            for (const std::string& sym : w.symbols) {
                const auto it = std::find(r.symbols.begin(), r.symbols.end(), sym);
                res.sym.push_back(it != r.symbols.end() ? int(it - r.symbols.begin()) : dflt);
            }
            return res;
        }
        case AK::Record: {
            if (!names_match(w, r)) unresolvable(path, "record \"" + w.fullname + "\" does not match \"" + r.fullname + "\"");
            for (const AvroField& rf : r.fields) {
                const std::string fp = path.empty() ? rf.name : path + "." + rf.name;
                int src = -1;  // the writer field of the same name, else the one the first matching reader alias names
                for (size_t i = 0; i < w.fields.size() && src < 0; ++i)
                    if (w.fields[i].name == rf.name) src = int(i);
                for (const std::string& a : rf.aliases)
                    for (size_t i = 0; i < w.fields.size() && src < 0; ++i)
                        if (w.fields[i].name == a) src = int(i);
                for (int earlier : res.src)
                    if (src >= 0 && earlier == src) unresolvable(fp, "writer field '" + w.fields[size_t(src)].name + "' is read by two reader fields");
                res.src.push_back(src);
                if (src >= 0) {
                    res.sub.push_back(resolve_node(*w.fields[size_t(src)].type, *rf.type, fp));
                } else {
                    Resolution d;
                    d.r = rf.type.get();
                    d.def = default_of(*rf.type, rf.dflt.get(), fp);
                    res.sub.push_back(std::move(d));
                }
            }
            return res;
        }
        case AK::Array: case AK::Map:
            if (r.k == AK::Array && takes_no_bytes(*w.sub[0]) && !takes_no_bytes(*r.sub[0]))
                unresolvable(path, "list items that take no wire bytes cannot be read as items that own buffers (DESIGN.md §10)");
            res.sub.push_back(resolve_node(*w.sub[0], *r.sub[0], path));
            return res;
        case AK::Unsupported:
            unresolvable(path, "unsupported type: " + r.what);
        default:
            return res;  // the same primitive / logical type
    }
}

}  // namespace

Resolution resolve_schemas(const AvroNode& writer, const AvroNode& reader) {
    if (writer.k != AK::Record || reader.k != AK::Record) throw std::runtime_error("schema resolution: both schemas must be records");
    return resolve_node(writer, reader, std::string());
}

std::unique_ptr<AvroNode> optional_fields(const AvroNode& top) {
    if (top.k != AK::Record) throw std::runtime_error("a permissive decode needs a record schema");
    auto r = clone_node(top);
    for (AvroField& f : r->fields) {
        // (a map stays as it is: ["null", map] has no Arrow form here, as in the reference's schema_translate)
        if (f.type->k == AK::Union || f.type->k == AK::Null || f.type->k == AK::Map) continue;
        auto u = mk(AK::Union);
        const bool value_default = f.dflt && f.dflt->kind != Json::Null;
        if (value_default) u->sub.push_back(std::move(f.type));
        u->sub.push_back(mk(AK::Null));
        if (!value_default) u->sub.push_back(std::move(f.type));
        f.type = std::move(u);
    }
    return r;
}

// ---- Parsing Canonical Form and CRC-64-AVRO (the specification's "Schema Fingerprints") -------------------------------
namespace {

// The parser replaces a reference by a copy of the definition it names, so a named type met again is written as its
// fullname here, as the reference was.
void canonical_node(const AvroNode& n, std::set<std::string>& named, std::string& o) {
    auto named_head = [&](const char* type) -> bool {  // false: already written, the fullname alone
        if (!named.insert(n.fullname).second) { o += "\"" + n.fullname + "\""; return false; }
        o += "{\"name\":\"" + n.fullname + "\",\"type\":\"" + type + "\"";
        return true;
    };
    switch (n.k) {
        case AK::Null: o += "\"null\""; return;
        case AK::Bool: o += "\"boolean\""; return;
        case AK::Int: case AK::Date: case AK::TimeMillis: o += "\"int\""; return;
        case AK::Long: case AK::TsMillis: case AK::TsMicros: case AK::TimeMicros: o += "\"long\""; return;
        case AK::Float: o += "\"float\""; return;
        case AK::Double: o += "\"double\""; return;
        case AK::String: case AK::Uuid: o += "\"string\""; return;
        case AK::Bytes: case AK::DecimalBytes: o += "\"bytes\""; return;
        case AK::Fixed: case AK::DecimalFixed:
            if (named_head("fixed")) o += ",\"size\":" + std::to_string(n.size) + "}";
            return;
        case AK::Enum:
            if (!named_head("enum")) return;
            o += ",\"symbols\":[";
            for (size_t i = 0; i < n.symbols.size(); ++i) o += (i ? ",\"" : "\"") + n.symbols[i] + "\"";
            o += "]}";
            return;
        case AK::Record:
            if (!named_head("record")) return;
            o += ",\"fields\":[";
            for (size_t i = 0; i < n.fields.size(); ++i) {
                o += (i ? ",{\"name\":\"" : "{\"name\":\"") + n.fields[i].name + "\",\"type\":";
                canonical_node(*n.fields[i].type, named, o);
                o += "}";
            }
            o += "]}";
            return;
        case AK::Union:
            o += "[";
            for (size_t i = 0; i < n.sub.size(); ++i) {
                if (i) o += ",";
                canonical_node(*n.sub[i], named, o);
            }
            o += "]";
            return;
        case AK::Array: case AK::Map:
            o += n.k == AK::Array ? "{\"type\":\"array\",\"items\":" : "{\"type\":\"map\",\"values\":";
            canonical_node(*n.sub[0], named, o);
            o += "}";
            return;
        case AK::Unsupported:
            throw std::runtime_error("Parsing Canonical Form: unsupported type: " + n.what);
    }
}

}  // namespace

std::string canonical_form(const AvroNode& top) {
    std::set<std::string> named;
    std::string o;
    canonical_node(top, named, o);
    return o;
}

uint64_t crc64_avro(const std::string& bytes) {
    static const auto table = [] {
        std::array<uint64_t, 256> t{};
        for (uint64_t i = 0; i < 256; ++i) {
            uint64_t fp = i;
            for (int j = 0; j < 8; ++j) fp = (fp >> 1) ^ (kCrc64AvroEmpty & (0 - (fp & 1)));
            t[size_t(i)] = fp;
        }
        return t;
    }();
    uint64_t fp = kCrc64AvroEmpty;
    for (unsigned char b : bytes) fp = (fp >> 8) ^ table[size_t((fp ^ b) & 0xFF)];
    return fp;
}

}  // namespace rv
