"""Avro single-object encoding, restated from the specification for the tests: the Parsing Canonical Form of a schema,
its CRC-64-AVRO fingerprint and the 10-byte message header.  Works on the raw JSON document (json.loads) and never on
the product's parser, so a test that compares the two checks the product against the specification's rules:

- [PRIMITIVES] a primitive, also written as {"type": "int", ...}, is its bare name;
- [FULLNAMES] names are fullnames (a dotted name carries its namespace, else "namespace", else the enclosing one), and
  "namespace" itself is dropped;
- [STRIP] only name, type, fields, symbols, items, values and size are kept (so logical types, doc, aliases and every
  default go), field objects keep name and type;
- [ORDER] in that order;
- [WHITESPACE] no whitespace; [INTEGERS] size as a bare integer;
- a named type is written in full where it first occurs and as its fullname after that (how Avro's own normalisation
  writes a reference); an "error" is written as a "record" (Avro has one Schema type for both).

One reading is apache-avro's rather than the specification's: a record field whose "type" is the bare string "array",
"map", "enum" or "fixed" is itself that type's object ({"name": "xs", "type": "array", "items": "int"} is a field xs of
an array of ints).  The reference's schemas are written that way, and the library parses them so.
"""
import json
import struct

PRIMITIVES = ("null", "boolean", "int", "long", "float", "double", "bytes", "string")
EMPTY = 0xC15D213AA4D7A795


def _crc_table():
    t = []
    for i in range(256):
        fp = i
        for _ in range(8):
            fp = (fp >> 1) ^ (EMPTY & -(fp & 1))
        t.append(fp)
    return t


_TABLE = _crc_table()


def crc64_avro(data: bytes) -> int:
    """The specification's table-driven 64-bit Rabin fingerprint."""
    fp = EMPTY
    for b in data:
        fp = (fp >> 8) ^ _TABLE[(fp ^ b) & 0xFF]
    return fp


def _q(s: str) -> str:
    return json.dumps(s, ensure_ascii=False)


def _fullname(name: str, ns: str) -> str:
    return name if "." in name or not ns else ns + "." + name


def _pcf(s, ns: str, seen: set) -> str:
    if isinstance(s, str):
        return _q(s) if s in PRIMITIVES else _q(_fullname(s, ns))   # a primitive, or a reference to a named type
    if isinstance(s, list):
        return "[" + ",".join(_pcf(x, ns, seen) for x in s) + "]"
    t = s["type"]
    if not isinstance(t, str):
        return _pcf(t, ns, seen)
    if t in PRIMITIVES:
        return _q(t)
    if t in ("record", "error", "enum", "fixed"):
        name = s["name"]
        if "." in name:
            full, inner = name, name.rsplit(".", 1)[0]
        else:
            inner = s.get("namespace", ns) or ""
            full = _fullname(name, inner)
        if full in seen:
            return _q(full)
        seen.add(full)
        out = '{"name":' + _q(full) + ',"type":' + _q("record" if t == "error" else t)
        if t in ("record", "error"):
            out += ',"fields":[' + ",".join('{"name":' + _q(f["name"]) + ',"type":' + _pcf(_field_type(f), inner, seen) + "}"
                                            for f in s["fields"]) + "]"
        elif t == "enum":
            out += ',"symbols":[' + ",".join(_q(x) for x in s["symbols"]) + "]"
        else:
            out += ',"size":' + str(int(s["size"]))
        return out + "}"
    if t == "array":
        return '{"type":"array","items":' + _pcf(s["items"], ns, seen) + "}"
    if t == "map":
        return '{"type":"map","values":' + _pcf(s["values"], ns, seen) + "}"
    return _q(_fullname(t, ns))   # {"type": "some.Named"}


def _field_type(f: dict):
    t = f["type"]
    return f if isinstance(t, str) and t in ("array", "map", "enum", "fixed") else t


def canonical_form(schema_json: str) -> str:
    return _pcf(json.loads(schema_json), "", set())


def fingerprint(schema_json: str) -> int:
    return crc64_avro(canonical_form(schema_json).encode("utf-8"))


def header(fp: int) -> bytes:
    """C3 01, then the fingerprint little-endian."""
    return b"\xc3\x01" + struct.pack("<Q", fp)


def frame(fp: int, datum: bytes) -> bytes:
    return header(fp) + datum
