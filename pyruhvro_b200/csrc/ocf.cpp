// See ocf.hpp.
#include "ocf.hpp"

#include <cstring>
#include <stdexcept>

namespace rv {
namespace {

struct Rd {
    const uint8_t* p;
    int64_t len, pos = 0;
    [[noreturn]] void bad(const char* what) const { throw std::runtime_error(std::string("object container file: ") + what); }
    int64_t varint() {
        uint64_t r = 0;
        for (int shift = 0; shift < 70; shift += 7) {
            if (pos >= len) bad("truncated varint");
            const uint8_t b = p[pos++];
            r |= uint64_t(b & 0x7F) << shift;
            if (!(b & 0x80)) return int64_t(r >> 1) ^ -int64_t(r & 1);
        }
        bad("varint too long");
    }
    std::string bytes() {
        const int64_t n = varint();
        if (n < 0 || n > len - pos) bad("truncated string");
        std::string s(reinterpret_cast<const char*>(p + pos), size_t(n));
        pos += n;
        return s;
    }
};

}  // namespace

OcfIndex ocf_index(const uint8_t* file, int64_t len) {
    Rd r{file, len};
    if (len < 4 || std::memcmp(file, "Obj\x01", 4) != 0) r.bad("missing magic \"Obj\\x01\"");
    r.pos = 4;
    OcfIndex ix;
    ix.codec = "null";
    for (;;) {  // file metadata: map<bytes>
        int64_t n = r.varint();
        if (n == 0) break;
        if (n < 0) { (void)r.varint(); n = -n; }
        for (int64_t i = 0; i < n; ++i) {
            const std::string key = r.bytes(), val = r.bytes();
            if (key == "avro.schema") ix.schema_json = val;
            else if (key == "avro.codec") ix.codec = val;
        }
    }
    if (ix.schema_json.empty()) r.bad("no avro.schema in the header");
    if (ix.codec != "null" && !ix.codec.empty()) throw std::runtime_error("object container file: codec \"" + ix.codec + "\" is not supported (blocks must be uncompressed)");
    if (len - r.pos < 16) r.bad("truncated sync marker");
    uint8_t sync[16];
    std::memcpy(sync, file + r.pos, 16);
    r.pos += 16;
    ix.end_off = r.pos;
    for (int64_t i = 0; r.pos < len; ++i) {
        const int64_t count = r.varint(), size = r.varint();
        if (count < 0 || size < 0 || size > len - r.pos - 16) r.bad("truncated block");
        // Every datum takes at least one byte unless the schema's datums are always empty, so a block cannot hold more
        // records than bytes.  (It also bounds the work: one lane walks `count` records and writes 8 bytes of offsets
        // for each, so a forged count must not get that far; with it n_records <= len, and the sum cannot overflow.)
        if (count > size)
            r.bad(("block " + std::to_string(i) + " holds " + std::to_string(count) + " records in " + std::to_string(size) + " bytes").c_str());
        OcfBlock b{r.pos, size, count, ix.n_records};
        r.pos += size;
        if (std::memcmp(file + r.pos, sync, 16) != 0) r.bad("sync marker mismatch");
        r.pos += 16;
        if (count > 0) {
            ix.blocks.push_back(b);
            ix.n_records += count;
            ix.end_off = b.data_off + b.size;
        }
    }
    return ix;
}

}  // namespace rv
