// Avro schema model, the fast-path gate, and the Avro -> Arrow schema translation.
//
// Mirrors (behaviour, not code) of the reference:
//   - apache_avro::Schema::parse_str as used at ruhvro/src/deserialize.rs:18-20
//   - fast_decode::is_supported            ruhvro/src/fast_decode.rs:38-61
//   - schema_translate::to_arrow_schema    ruhvro/src/schema_translate.rs:19-280
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "arrow_c.h"

namespace rv {

enum class AK : uint8_t {
    Null, Bool, Int, Long, Float, Double, String, Date, TsMillis, TsMicros, Enum, Record, Union, Array, Map,
    // the wider subset (SURVEY.md 8(f) rank 3): schemas the reference's fast path rejects (fast_decode.rs:16-17,59) and
    // its Value-tree fallback cannot build either (complex.rs:414-431 `unimplemented!`); Arrow types per
    // schema_translate.rs:58,133-143, values per the Avro specification
    Bytes, Fixed, DecimalBytes, DecimalFixed, Uuid, TimeMillis, TimeMicros,
    Unsupported  // duration, local-timestamp-*, timestamp-nanos, decimals beyond 128 bits, recursive named references
};

struct AvroNode;
struct Json;
struct AvroField {
    std::string name;
    std::unique_ptr<AvroNode> type;
    bool has_doc = false;
    std::string doc;
    std::shared_ptr<const Json> dflt;  // the field's "default" as written (nullptr: none); checked only when a resolution uses it
    std::vector<std::string> aliases;  // the field's "aliases" (strings only)
};
struct AvroNode {
    AK k = AK::Null;
    std::string fullname;  // record / enum
    bool has_doc = false;
    std::string doc;
    bool has_aliases = false;
    std::vector<std::string> aliases;  // namespace-qualified
    std::vector<AvroField> fields;     // record
    std::vector<std::string> symbols;  // enum
    bool has_enum_default = false;     // enum: "default" (one of the symbols)
    std::string enum_default;
    std::vector<std::unique_ptr<AvroNode>> sub;  // union variants; array: [items]; map: [values]
    std::string what;                  // Unsupported: which construct
    int32_t size = 0;                  // fixed / decimal on fixed: bytes
    int32_t precision = 0, scale = 0;  // decimal
};

// Throws std::runtime_error on malformed documents.
std::unique_ptr<AvroNode> parse_avro_schema(const char* json, size_t len);

// fast_decode.rs:38-61.  `why` receives the first offending construct.
bool is_supported(const AvroNode& top, std::string* why);

enum class AT : uint8_t { Null, Bool, Int32, Int64, Float32, Float64, Utf8, Date32, TsMs, TsUs, Struct, List, Map, SparseUnion,
                          Binary, FixedSizeBinary, Decimal128, Time32Ms, Time64Us };

struct ArrowField {
    std::string name;
    AT type = AT::Null;
    bool nullable = false;
    std::vector<std::pair<std::string, std::string>> metadata;
    std::vector<ArrowField> children;  // struct fields / union variants / list: [item] / map: [entries{keys,values}]
    int32_t width = 0;                 // FixedSizeBinary
    int32_t precision = 0, scale = 0;  // Decimal128
};

// schema_translate.rs:19-37: one ArrowField per top-level record field.
std::vector<ArrowField> to_arrow_fields(const AvroNode& top);

// Arrow C Data Interface export of a whole schema ("+s" with the fields as children).
void export_arrow_schema(const std::vector<ArrowField>& fields, ArrowSchema* out);

// Column projection: the indices into `available` (top-level field names) of `requested`, in the requested order.
// Throws std::invalid_argument for an empty list, a repeated name, or a name that is not a field (the message lists the
// available ones).
std::vector<int> select_columns(const std::vector<std::string>& available, const std::vector<std::string>& requested);

// ---- schema resolution (rv_schema_resolve): data written with one schema, read as another --------------------------
// The constant that fills a reader field the writer does not have.
struct DefaultValue {
    bool is_null = false;
    int64_t i = 0;      // boolean, int, long and their logical types
    double d = 0;       // float, double
    std::string bytes;  // string, bytes (code points 0-255), enum symbol
};

// How the writer's node `w` is read as the reader's node `r` (the Avro specification's "Schema Resolution", restricted
// as DESIGN.md §7 lists).  w == nullptr: a reader record field the writer does not have, filled with `def`.
struct Resolution {
    const AvroNode* w = nullptr;
    const AvroNode* r = nullptr;
    std::vector<int> src;         // record: for each reader field, the writer field it reads (-1: its default)
    std::vector<Resolution> sub;  // record: one per reader field; union: one per variant; nullable: [inner]; array / map: [items]
    std::vector<int> sym;         // enum: for each writer symbol, the reader symbol it becomes (-1: none, the record fails)
    DefaultValue def;
};

// The resolution of two top-level records.  Throws std::runtime_error ("schema resolution: field 'a.b': ...") for the
// first pair outside the rules, naming the reader field's path.  The single place the rules live: the product's plan
// and the host emulation both build from it.
Resolution resolve_schemas(const AvroNode& writer, const AvroNode& reader);

// The reader schema of a permissive decode (rv_schema_permissive): the record `top` with every top-level field whose type
// is not a union, null or a map made optional, T -> ["null", T].  A field with a non-null default becomes [T, "null"]
// instead, where the default stays valid (a union's default belongs to its first branch); both are the same Arrow column.
// A map stays as it is: a nullable map has no Arrow form here (to_arrow_fields refuses ["null", map], as the reference does).
std::unique_ptr<AvroNode> optional_fields(const AvroNode& top);

// ---- schema fingerprints (the specification's "Parsing Canonical Form" and "Schema Fingerprints") --------------------
// The canonical form of a parsed schema: primitives as bare names, named types by fullname (written in full at their
// first occurrence, by fullname after that), only name / type / fields / symbols / items / values / size in that order,
// logical types, docs, aliases and defaults dropped, no whitespace.  Throws std::runtime_error for a schema the parser
// keeps as AK::Unsupported (its underlying type is not kept).
std::string canonical_form(const AvroNode& top);

// CRC-64-AVRO of `bytes`: the 64-bit Rabin fingerprint the single-object encoding names its writer schema by.
constexpr uint64_t kCrc64AvroEmpty = 0xc15d213aa4d7a795ull;
uint64_t crc64_avro(const std::string& bytes);

}  // namespace rv
