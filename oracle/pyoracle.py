"""pyoracle — TEST INFRASTRUCTURE (not product code).

Three things live here, all used only by tests/, ``__graft_entry__.smoke()`` and
``bench.py``'s CPU-baseline legs:

1. ``AvroSchema`` / ``parse_schema`` / ``to_arrow_schema`` — an independent
   pure-Python restatement of the output-schema rules in
   ``/root/reference/ruhvro/src/schema_translate.rs:19-280`` (names, nullability
   propagation, sparse-union child names, map/list shapes, metadata).
2. ``py_decode`` — a pure-Python, row-at-a-time restatement of
   ``/root/reference/ruhvro/src/fast_decode.rs:420-922`` with arrow-rs builder
   semantics.  Slow; for small cases only.  It cross-checks the C oracle
   (``oracle/avro_oracle.c``), which is the fast parity anchor.
3. ``COracle`` — ctypes binding of ``oracle/liboracle.so``.

Every decoder returns the same *canonical form*: a list (one per top-level
column) of nested dicts holding the exact Arrow buffers as ``bytes``:

    {"kind": "int32"|"int64"|"float32"|"float64"|"bool"|"utf8"|"null"|
             "struct"|"union"|"list"|"map",
     "length": n, "null_count": k,
     "validity": None | bytes (ceil(n/8), LSB-first, zero padded),
     "buffers": [bytes, ...]      # values | [offsets, data] | [type_ids] | [offsets]
     "children": [canon, ...]}

``canon_from_arrow`` extracts the same form from a pyarrow array, so the product's
output can be compared buffer-for-buffer (the L2 "buffer-exact" level of
SURVEY.md A.2).  ``encode_datum`` / ``random_value`` make Avro test inputs
following the grammar the reference's encoder emits
(``ruhvro/src/fast_encode.rs:397-599``).

Parity status: pinned against the reference's literal golden datums
(``deserialize.rs:244,303``, ``lib.rs:165-167``) in tests/test_oracle_golden.py.
The reference (Rust) cannot be built in this image, so no ``oracle/_ref`` exists.
"""
from __future__ import annotations

import copy
import ctypes
import json
import os
import struct
import subprocess
from typing import Any, List, Optional

import pyarrow as pa

HERE = os.path.dirname(os.path.abspath(__file__))

# --------------------------------------------------------------------------- #
# Avro schema model (what apache_avro::Schema::parse_str yields, for the subset
# the path matches on; deserialize.rs:18-20)
# --------------------------------------------------------------------------- #
PRIMS = {"null", "boolean", "int", "long", "float", "double", "bytes", "string"}


class AvroSchema:
    __slots__ = ("kind", "fullname", "doc", "aliases", "fields", "symbols", "items", "values", "variants", "size", "precision", "scale")

    def __init__(self, kind: str, **kw: Any):
        self.kind = kind
        self.fullname: Optional[str] = kw.get("fullname")
        self.doc: Optional[str] = kw.get("doc")
        self.aliases: Optional[List[str]] = kw.get("aliases")
        self.fields: List[tuple] = kw.get("fields", [])  # (name, AvroSchema, doc)
        self.symbols: List[str] = kw.get("symbols", [])
        self.items: Optional["AvroSchema"] = kw.get("items")
        self.values: Optional["AvroSchema"] = kw.get("values")
        self.variants: List["AvroSchema"] = kw.get("variants", [])
        self.size: int = kw.get("size", 0)            # fixed / decimal on fixed / uuid (16)
        self.precision: int = kw.get("precision", 0)  # decimal
        self.scale: int = kw.get("scale", 0)

    def __repr__(self) -> str:  # pragma: no cover
        return f"AvroSchema({self.kind})"


def _name(j: dict, enclosing_ns: Optional[str]):
    name = j["name"]
    if "." in name:
        ns, _, short = name.rpartition(".")
    else:
        ns, short = j.get("namespace"), name
        if not isinstance(ns, str):     # (only a string is a namespace; anything else is as good as absent)
            ns = enclosing_ns
    ns = ns or None
    return (f"{ns}.{short}" if ns else short), ns


def _fix_aliases(aliases, ns):
    if not isinstance(aliases, list) or not all(isinstance(a, str) for a in aliases):
        return None   # (apache-avro collects the aliases into an Option: anything but an array of strings is no aliases)
    return [a if ("." in a or not ns) else f"{ns}.{a}" for a in aliases]


# The WIDER SUBSET (SURVEY.md 8(f) rank 3).  The reference's fast path rejects bytes / fixed / uuid / decimal / time-* /
# named references (fast_decode.rs:16-17,59) and its Value-tree fallback cannot build those columns either
# (complex.rs:414-431 `unimplemented!`), so with wide=False this module restates the reference (they are
# "unsupported"), and with wide=True it restates what the product adds: Arrow types per schema_translate.rs:58,133-143,
# values per the Avro specification.
class _Names:
    def __init__(self):
        self.done, self.open = {}, set()


def _parse(j: Any, ns: Optional[str], wide: bool = False, names: Optional[_Names] = None) -> AvroSchema:
    names = names if names is not None else _Names()
    if isinstance(j, str):
        return _prim(j, None, wide, ns, names)
    if isinstance(j, list):
        vs = [_parse(v, ns, wide, names) for v in j]
        if any(v.kind == "union" for v in vs):
            raise ValueError("unions may not immediately contain other unions")
        return AvroSchema("union", variants=vs)
    if not isinstance(j, dict) or "type" not in j:
        raise ValueError("invalid schema")
    t = j["type"]
    if not isinstance(t, str):
        return _parse(t, ns, wide, names)
    if t in ("record", "error"):
        full, rns = _name(j, ns)
        names.open.add(full)
        # apache-avro 0.21 RecordField::parse hands the FIELD object to Parser::parse_complex: with a bare-string
        # "type", items / values / symbols / logicalType are read from the field object (ruhvro/src/serialize.rs:185
        # relies on {"name":..,"type":"array","items":..}); a bare "record" is a named look-up -> unsupported Ref
        fields = []
        for f in j["fields"]:
            ft = f["type"]
            is_ref = isinstance(ft, str) and wide and _is_named_ref(ft, rns, names)
            if isinstance(ft, str) and ft not in ("record", "error") and not is_ref:
                fs = _parse(f, rns, wide, names)
            else:
                fs = _parse(ft, rns, wide, names)
            fields.append((f["name"], fs, f.get("doc")))
        r = AvroSchema("record", fullname=full, doc=j.get("doc"), aliases=_fix_aliases(j.get("aliases"), rns), fields=fields)
        names.open.discard(full)
        names.done[full] = r
        return r
    if t == "enum":
        full, ens = _name(j, ns)
        e = AvroSchema("enum", fullname=full, doc=j.get("doc"), aliases=_fix_aliases(j.get("aliases"), ens), symbols=list(j["symbols"]))
        names.done[full] = e
        return e
    if t == "array":
        return AvroSchema("array", items=_parse(j["items"], ns, wide, names))
    if t == "map":
        return AvroSchema("map", values=_parse(j["values"], ns, wide, names))
    if t == "fixed" and wide:
        full, fns = _name(j, ns)
        size = int(j["size"])
        lt = j.get("logicalType")
        f = None
        if lt == "decimal":
            f = _decimal("decimal-fixed", j, size)
        elif lt == "duration":
            f = AvroSchema("unsupported")
        if f is None:
            f = AvroSchema("fixed", size=size)
        f.fullname, f.doc, f.aliases = full, j.get("doc"), _fix_aliases(j.get("aliases"), fns)
        if f.kind != "unsupported":
            names.done[full] = f
        return f
    return _prim(t, j, wide, ns, names)


_BUILTIN = {"null", "boolean", "int", "long", "float", "double", "bytes", "string", "array", "map", "enum", "record", "error", "fixed"}


def _is_named_ref(t: str, ns: Optional[str], names: _Names) -> bool:
    if t in _BUILTIN:
        return False
    q = f"{ns}.{t}" if "." not in t and ns else t
    return q in names.done or q in names.open or t in names.done or t in names.open


def _decimal(kind: str, obj: dict, size: int) -> Optional[AvroSchema]:
    """None: invalid precision / scale.  apache-avro 0.21 then ignores the logical type with a warning ("Ignoring invalid
    decimal logical type") and the schema is the underlying bytes / fixed; precision and scale must be JSON numbers that are
    non-negative integers (parse_json_integer_for_decimal), only "scale" may be absent (0)."""
    def meta(key, absent):
        v = obj.get(key, absent) if obj else absent
        return v if isinstance(v, int) and not isinstance(v, bool) and 0 <= v < 10**9 else -1
    precision, scale = meta("precision", -1), meta("scale", 0)
    if precision < 1 or scale < 0 or scale > precision:
        return None
    if precision > 38 or (kind == "decimal-fixed" and size > 16):
        return AvroSchema("unsupported")
    return AvroSchema(kind, size=size, precision=precision, scale=scale)


def _prim(t: str, obj: Optional[dict], wide: bool = False, ns: Optional[str] = None, names: Optional[_Names] = None) -> AvroSchema:
    lt = obj.get("logicalType") if obj else None
    if t == "int":
        if lt == "date":
            return AvroSchema("date")
        if lt == "time-millis":
            return AvroSchema("time-millis" if wide else "unsupported")
        return AvroSchema("int")
    if t == "long":
        if lt == "timestamp-millis":
            return AvroSchema("timestamp-millis")
        if lt == "timestamp-micros":
            return AvroSchema("timestamp-micros")
        if lt == "time-micros":
            return AvroSchema("time-micros" if wide else "unsupported")
        if lt in ("timestamp-nanos", "local-timestamp-millis", "local-timestamp-micros", "local-timestamp-nanos"):
            return AvroSchema("unsupported")
        return AvroSchema("long")
    if t == "string":
        if lt == "uuid":
            return AvroSchema("uuid", size=16) if wide else AvroSchema("unsupported")
        return AvroSchema("string")
    if t in ("null", "boolean", "float", "double"):
        return AvroSchema(t)
    if not wide:
        return AvroSchema("unsupported")  # bytes, fixed, named Ref (fast_decode.rs:59)
    if t == "bytes":
        return (_decimal("decimal-bytes", obj, 0) if lt == "decimal" else None) or AvroSchema("bytes")
    if names is not None:
        for cand in ((f"{ns}.{t}" if "." not in t and ns else t), t):
            if cand in names.open:
                return AvroSchema("unsupported")  # recursive type
            if cand in names.done:
                return copy.deepcopy(names.done[cand])
    return AvroSchema("unsupported")


def parse_schema(schema_json: str, wide: bool = False) -> AvroSchema:
    return _parse(json.loads(schema_json), None, wide, _Names())


WIDE_LEAVES = {"bytes", "fixed", "uuid", "decimal-bytes", "decimal-fixed", "time-millis", "time-micros"}
LEAVES = {"int", "long", "float", "double", "boolean", "string", "null", "date", "timestamp-millis", "timestamp-micros", "enum"}


def is_supported(s: AvroSchema) -> bool:
    """fast_decode.rs:38-61"""
    def inner(x: AvroSchema) -> bool:
        if x.kind in ("fixed", "decimal-fixed") and x.size == 0:   # zero wire bytes per value: outside the subset (csrc/schema.cpp)
            return False
        if x.kind in LEAVES or x.kind in WIDE_LEAVES:  # (wide kinds only exist when parsed with wide=True)
            return True
        if x.kind == "record":
            return all(inner(f[1]) for f in x.fields)
        if x.kind == "union":
            return all(inner(v) for v in x.variants)
        if x.kind == "array":
            return inner(x.items)
        if x.kind == "map":
            return inner(x.values)
        return False
    return s.kind == "record" and inner(s)


# --------------------------------------------------------------------------- #
# schema_translate.rs restated
# --------------------------------------------------------------------------- #
def _default_field_name(t: pa.DataType) -> str:
    """schema_translate.rs:155-220 (only the types this path can produce)"""
    if pa.types.is_null(t):
        return "null"
    if pa.types.is_boolean(t):
        return "bit"
    if pa.types.is_int32(t):
        return "int"
    if pa.types.is_int64(t):
        return "bigint"
    if pa.types.is_float32(t):
        return "float4"
    if pa.types.is_float64(t):
        return "float8"
    if pa.types.is_date32(t):
        return "dateday"
    if pa.types.is_timestamp(t):
        return {"ms": "timestampmilli", "us": "timestampmicro"}[t.unit]
    if pa.types.is_string(t):
        return "varchar"
    if pa.types.is_binary(t):
        return "varbinary"
    if pa.types.is_fixed_size_binary(t):
        return "fixedsizebinary"
    if pa.types.is_decimal(t):
        return "decimal"
    if pa.types.is_time32(t) or pa.types.is_time64(t):
        return {"ms": "timemilli", "us": "timemicro"}[t.unit]
    if pa.types.is_map(t):
        raise NotImplementedError("Map support not implemented")  # :212 unimplemented!()
    if pa.types.is_list(t):
        return "list"
    if pa.types.is_struct(t):
        return "struct"
    if pa.types.is_union(t):
        return "union"
    raise NotImplementedError(str(t))


def _field(s: AvroSchema, name: Optional[str], nullable: bool, props: Optional[dict]) -> pa.Field:
    """schema_to_field_with_props, schema_translate.rs:43-153"""
    k = s.kind
    if k == "null":
        t = pa.null()
    elif k == "boolean":
        t = pa.bool_()
    elif k == "int":
        t = pa.int32()
    elif k == "long":
        t = pa.int64()
    elif k == "float":
        t = pa.float32()
    elif k == "double":
        t = pa.float64()
    elif k == "string":
        t = pa.string()
    elif k == "date":
        t = pa.date32()
    elif k == "timestamp-millis":
        t = pa.timestamp("ms")
    elif k == "timestamp-micros":
        t = pa.timestamp("us")
    elif k == "bytes":
        t = pa.binary()                               # schema_translate.rs:58
    elif k in ("fixed", "uuid"):
        t = pa.binary(s.size)                         # :133,137 FixedSizeBinary
    elif k in ("decimal-bytes", "decimal-fixed"):
        t = pa.decimal128(s.precision, s.scale)       # :134-136
    elif k == "time-millis":
        t = pa.time32("ms")                           # :139
    elif k == "time-micros":
        t = pa.time64("us")                           # :140
    elif k == "array":
        t = pa.list_(_field(s.items, "item", True, None))
    elif k == "map":
        value_field = _field(s.values, "values", False, None)
        key_field = pa.field("keys", pa.string(), nullable=False)
        # NOTE: the reference gives the "entries" field the incoming `nullable` (:69-73); pyarrow's
        # MapType cannot express a nullable entries field, so `entries_nullable` is tracked by tests
        # that care via expected_entries_nullable().
        t = pa.map_(key_field, value_field)
    elif k == "union":
        has_null = any(v.kind == "null" for v in s.variants)
        if has_null and len(s.variants) == 2:
            nullable = True
            inner = next((v for v in s.variants if v.kind != "null"), None)
            if inner is None:
                raise ValueError("Avro union contains duplicate null variants")
            t = _field(inner, None, True, None).type
        else:
            if has_null:
                nullable = True
            fields = [_field(v, None, True, None) for v in s.variants]
            t = pa.union(fields, mode="sparse", type_codes=list(range(len(fields))))
    elif k == "record":
        fields = []
        for fname, fs, fdoc in s.fields:
            p = {"avro::doc": fdoc} if fdoc is not None else {}
            fields.append(_field(fs, fname, nullable, p))
        t = pa.struct(fields)
    elif k == "enum":
        fname = name if name else s.fullname
        return pa.field(fname, pa.string(), nullable=nullable)  # early return: no metadata (:131)
    else:
        raise NotImplementedError(k)
    fname = name if name is not None else _default_field_name(t)
    f = pa.field(fname, t, nullable=nullable)
    if props:
        f = f.with_metadata(props)
    return f


def _external_props(s: AvroSchema) -> dict:
    """schema_translate.rs:222-266"""
    props = {}
    if s.kind in ("record", "enum", "fixed", "decimal-fixed"):
        if s.doc is not None:
            props["avro::doc"] = s.doc
        if s.aliases is not None:
            props["avro::aliases"] = "[" + ",".join(s.aliases) + "]"
    return props


def to_arrow_schema(s: AvroSchema) -> pa.Schema:
    """schema_translate.rs:19-37"""
    if s.kind != "record":
        return pa.schema([_field(s, "", False, None)])
    return pa.schema([_field(fs, fname, False, _external_props(fs)) for fname, fs, _ in s.fields])


# --------------------------------------------------------------------------- #
# pure-Python decode with arrow-rs builder semantics -> canonical form
# --------------------------------------------------------------------------- #
class DecodeError(ValueError):
    def __init__(self, code: str, record: int = -1):
        super().__init__(f"{code} (record {record})")
        self.code = code
        self.record = record


class _Bits:
    def __init__(self):
        self.b = bytearray()
        self.n = 0

    def append(self, v: bool):
        if self.n % 8 == 0:
            self.b.append(0)
        if v:
            self.b[self.n >> 3] |= 1 << (self.n & 7)
        self.n += 1


class _LazyNulls:
    """arrow-rs NullBufferBuilder: materialised on the first null."""
    def __init__(self):
        self.bits: Optional[_Bits] = None
        self.len = 0
        self.nulls = 0

    def append(self, valid: bool):
        if not valid and self.bits is None:
            self.bits = _Bits()
            for _ in range(self.len):
                self.bits.append(True)
        if self.bits is not None:
            self.bits.append(valid)
        self.len += 1
        self.nulls += 0 if valid else 1


_FIXED = {"int": ("int32", "<i", 4), "date": ("int32", "<i", 4), "long": ("int64", "<q", 8),
          "timestamp-millis": ("int64", "<q", 8), "timestamp-micros": ("int64", "<q", 8),
          "float": ("float32", None, 4), "double": ("float64", None, 8),
          "time-millis": ("int32", "<i", 4), "time-micros": ("int64", "<q", 8)}
_RAW = ("fixed", "uuid", "decimal-bytes", "decimal-fixed")  # `width` raw bytes per row


def _raw_width(s: AvroSchema) -> int:
    return 16 if s.kind in ("uuid", "decimal-bytes", "decimal-fixed") else s.size


def uuid_bytes(text: bytes) -> bytes:
    """The 16 bytes (RFC 4122 order) of a UUID text: hyphenated 8-4-4-4-12 or 32 plain hex digits."""
    try:
        t = text.decode("ascii")
    except UnicodeDecodeError:
        raise DecodeError("value") from None
    if len(t) == 36:
        if any(t[i] != "-" for i in (8, 13, 18, 23)):
            raise DecodeError("value")
        t = t[:8] + t[9:13] + t[14:18] + t[19:23] + t[24:]
    if len(t) != 32 or any(ch not in "0123456789abcdefABCDEF" for ch in t):
        raise DecodeError("value")
    return bytes.fromhex(t)


def decimal128_le(be: bytes) -> bytes:
    """Unscaled big-endian two's complement of any length <= 16 -> 16 bytes little-endian."""
    if len(be) > 16:
        raise DecodeError("value")
    return int.from_bytes(be, "big", signed=True).to_bytes(16, "little", signed=True) if be else bytes(16)


class _Dec:
    """One FieldDecoder (fast_decode.rs:73-120); Nullable* folded into nullable/null_first."""
    def __init__(self, s: AvroSchema, nullable=False, null_first=False):
        self.s, self.k, self.nullable, self.null_first = s, s.kind, nullable, null_first
        self.values = bytearray()
        self.bools = _Bits()
        self.offsets = bytearray(struct.pack("<i", 0)) if s.kind in ("string", "enum", "array", "map", "bytes") else bytearray()
        self.nulls = _LazyNulls()
        self.explicit = _Bits()
        self.len = 0
        self.cur = 0
        self.type_ids = bytearray()
        self.children: List[_Dec] = []
        if self.k == "record":
            self.children = [_make(f[1]) for f in s.fields]
        elif self.k == "union":
            self.children = [_make(v) for v in s.variants]
        elif self.k == "array":
            self.children = [_make(s.items)]
        elif self.k == "map":
            self.children = [_Dec(AvroSchema("string")), _make(s.values)]


def _make(s: AvroSchema) -> _Dec:
    """make_decoder / make_union_decoder / split_null_union (fast_decode.rs:176-214,372-414)"""
    if s.kind == "union" and len(s.variants) == 2 and any(v.kind == "null" for v in s.variants):
        null_first = s.variants[0].kind == "null"
        inner = s.variants[1] if null_first else s.variants[0]
        if inner.kind in ("null", "union"):
            raise DecodeError("schema")
        return _Dec(inner, True, null_first)
    return _Dec(s)


class _Cur:
    def __init__(self, b: bytes):
        self.b, self.p = b, 0

    def byte(self) -> int:
        if self.p >= len(self.b):
            raise DecodeError("eof")
        v = self.b[self.p]
        self.p += 1
        return v

    def zigzag(self) -> int:
        """fast_decode.rs:854-869"""
        result, shift = 0, 0
        while True:
            byte = self.byte()
            result |= ((byte & 0x7F) << shift) & 0xFFFFFFFFFFFFFFFF
            if byte & 0x80 == 0:
                v = (result >> 1) ^ -(result & 1)
                return v  # already in i64 range
            shift += 7
            if shift >= 64:
                raise DecodeError("varint")

    def take(self, n: int) -> bytes:
        if len(self.b) - self.p < n:
            raise DecodeError("eof")
        v = self.b[self.p:self.p + n]
        self.p += n
        return v

    def string(self) -> bytes:
        """fast_decode.rs:902-922"""
        n = self.zigzag()
        if n < 0:
            raise DecodeError("neg_len")
        return self.take(n)


def _append_null(d: _Dec):
    """fast_decode.rs:503-534 + :608-616, :660-668, :721-727, :764-770"""
    k = d.k
    if k in _FIXED:
        d.values += bytes(_FIXED[k][2])
        d.nulls.append(False)
    elif k == "boolean":
        d.bools.append(False)
        d.nulls.append(False)
    elif k in ("string", "enum", "bytes"):
        d.offsets += struct.pack("<i", len(d.values))
        d.nulls.append(False)
    elif k in _RAW:
        d.values += bytes(_raw_width(d.s))
        d.nulls.append(False)
    elif k == "null":
        d.len += 1
    elif k == "record":
        if d.nullable:
            d.explicit.append(False)
        d.len += 1
        for c in d.children:
            _append_null(c)
    elif k == "union":
        for c in d.children:
            _append_null(c)
        d.type_ids.append(0)
    else:  # array / map: children untouched
        d.offsets += struct.pack("<i", d.cur)
        if d.nullable:
            d.explicit.append(False)


def _decode(d: _Dec, c: _Cur):
    """fast_decode.rs:420-499"""
    if d.nullable:
        idx = c.zigzag()  # union_branch :585-593
        if idx not in (0, 1):
            raise DecodeError("branch")
        is_null = (idx == 0) == d.null_first
        if is_null:
            _append_null(d)
            return
    k = d.k
    if k in ("int", "date", "time-millis"):
        v = c.zigzag() & 0xFFFFFFFF  # `as i32` wrapping truncation
        d.values += struct.pack("<I", v)
        d.nulls.append(True)
    elif k in ("long", "timestamp-millis", "timestamp-micros", "time-micros"):
        d.values += struct.pack("<q", c.zigzag())
        d.nulls.append(True)
    elif k == "bytes":
        d.values += c.string()
        d.offsets += struct.pack("<i", len(d.values))
        d.nulls.append(True)
    elif k == "fixed":
        d.values += c.take(d.s.size)
        d.nulls.append(True)
    elif k == "uuid":
        d.values += uuid_bytes(c.string())
        d.nulls.append(True)
    elif k == "decimal-bytes":
        d.values += decimal128_le(c.string())
        d.nulls.append(True)
    elif k == "decimal-fixed":
        d.values += decimal128_le(c.take(d.s.size))
        d.nulls.append(True)
    elif k == "float":
        d.values += c.take(4)
        d.nulls.append(True)
    elif k == "double":
        d.values += c.take(8)
        d.nulls.append(True)
    elif k == "boolean":
        b = c.byte()
        if b > 1:
            raise DecodeError("bool")
        d.bools.append(bool(b))
        d.nulls.append(True)
    elif k == "string":
        d.values += c.string()
        d.offsets += struct.pack("<i", len(d.values))
        d.nulls.append(True)
    elif k == "enum":
        idx = c.zigzag()
        if idx < 0 or idx >= len(d.s.symbols):
            raise DecodeError("enum")
        d.values += d.s.symbols[idx].encode("utf-8")
        d.offsets += struct.pack("<i", len(d.values))
        d.nulls.append(True)
    elif k == "null":
        d.len += 1
    elif k == "record":
        if d.nullable:
            d.explicit.append(True)
        d.len += 1
        for ch in d.children:
            _decode(ch, c)
    elif k == "union":
        idx = c.zigzag()
        if idx < 0 or idx >= len(d.children):
            raise DecodeError("branch")
        for i, ch in enumerate(d.children):
            if i == idx:
                _decode(ch, c)
            else:
                _append_null(ch)
        d.type_ids.append(idx)
    else:  # array / map
        while True:
            n = c.zigzag()  # read_block_count :689-700
            if n < 0:
                c.zigzag()
                n = -n
                if n >= 1 << 63:   # `-n` wraps in the release build: i64::MIN stays negative and `0..n` is an empty range
                    n -= 1 << 64
            if n == 0:
                break
            for _ in range(max(n, 0)):
                if k == "map":
                    key = d.children[0]
                    key.values += c.string()
                    key.offsets += struct.pack("<i", len(key.values))
                    key.nulls.append(True)
                    _decode(d.children[1], c)
                else:
                    _decode(d.children[0], c)
                d.cur += 1
        d.offsets += struct.pack("<i", d.cur)
        if d.nullable:
            d.explicit.append(True)


def _canon(kind, length, null_count=0, validity=None, buffers=(), children=()):
    return {"kind": kind, "length": length, "null_count": null_count, "validity": validity,
            "buffers": [bytes(b) for b in buffers], "children": list(children)}


def _lazy(d: _Dec):
    if d.nulls.bits is None:
        return 0, None
    return d.nulls.nulls, bytes(d.nulls.bits.b)


def _explicit(d: _Dec):
    if not d.nullable:
        return 0, None
    b = d.explicit
    zeros = sum(1 for i in range(b.n) if not (b.b[i >> 3] >> (i & 7)) & 1)
    return zeros, bytes(b.b)


def _finish(d: _Dec) -> dict:
    """fast_decode.rs:536-567 and the Record/Union/List/Map finish impls"""
    k = d.k
    if k in _FIXED:
        name, _, w = _FIXED[k]
        nc, v = _lazy(d)
        return _canon(name, len(d.values) // w, nc, v, [d.values])
    if k == "boolean":
        nc, v = _lazy(d)
        return _canon("bool", d.bools.n, nc, v, [d.bools.b])
    if k in ("string", "enum", "bytes"):
        nc, v = _lazy(d)
        return _canon("utf8", len(d.offsets) // 4 - 1, nc, v, [d.offsets, d.values])
    if k in _RAW:
        nc, v = _lazy(d)
        w = _raw_width(d.s)
        return _canon("raw%d" % w, d.nulls.len, nc, v, [d.values])
    if k == "null":
        return _canon("null", d.len, d.len)
    if k == "record":
        if not d.children:
            raise DecodeError("schema")
        nc, v = _explicit(d)
        return _canon("struct", d.len, nc, v, [], [_finish(c) for c in d.children])
    if k == "union":
        return _canon("union", len(d.type_ids), 0, None, [d.type_ids], [_finish(c) for c in d.children])
    nc, v = _explicit(d)
    n = len(d.offsets) // 4 - 1
    if k == "array":
        return _canon("list", n, nc, v, [d.offsets], [_finish(d.children[0])])
    keys = _finish(d.children[0])
    entries = _canon("struct", keys["length"], 0, None, [], [keys, _finish(d.children[1])])
    return _canon("map", n, nc, v, [d.offsets], [entries])


def _has_empty_record(s: AvroSchema) -> bool:
    """A record with no fields always fails at finish: nested -> "RecordDecoder produced a record with 0 fields"
    (fast_decode.rs:633-635); top level -> RecordBatch::try_new with no columns (:834)."""
    if s.kind == "record":
        return not s.fields or any(_has_empty_record(f[1]) for f in s.fields)
    if s.kind == "union":
        return any(_has_empty_record(v) for v in s.variants)
    if s.kind == "array":
        return _has_empty_record(s.items)
    if s.kind == "map":
        return _has_empty_record(s.values)
    return False


def py_decode(schema: AvroSchema, records: List[bytes]) -> List[dict]:
    """decode_with_arrow_schema (fast_decode.rs:815-835): canonical columns of one batch."""
    if not is_supported(schema) or _has_empty_record(schema):
        raise DecodeError("schema")
    top = [_make(f[1]) for f in schema.fields]
    for r, rec in enumerate(records):
        c = _Cur(rec)
        try:
            for d in top:
                _decode(d, c)
        except DecodeError as e:
            raise DecodeError(e.code, r) from None
        # trailing bytes are ignored (:825-828)
    return [_finish(d) for d in top]


def clamp_chunks(num_chunks: int, n: int) -> int:
    """deserialize.rs:53-55"""
    return min(max(num_chunks, 1), max(n, 1))


def chunk_bounds(n: int, k: int):
    """build_slices, deserialize.rs:57-68"""
    cs = n // k
    return [(i * cs, n if i == k - 1 else (i + 1) * cs) for i in range(k)]


# --------------------------------------------------------------------------- #
# canonical form <-> pyarrow
# --------------------------------------------------------------------------- #
_W = {"int32": 4, "int64": 8, "float32": 4, "float64": 8}


def _kind_of(t: pa.DataType) -> str:
    if pa.types.is_int32(t) or pa.types.is_date32(t) or pa.types.is_time32(t):
        return "int32"
    if pa.types.is_int64(t) or pa.types.is_timestamp(t) or pa.types.is_time64(t):
        return "int64"
    if pa.types.is_fixed_size_binary(t):
        return "raw%d" % t.byte_width
    if pa.types.is_decimal(t):
        return "raw16"
    if pa.types.is_binary(t):
        return "utf8"
    if pa.types.is_float32(t):
        return "float32"
    if pa.types.is_float64(t):
        return "float64"
    if pa.types.is_boolean(t):
        return "bool"
    if pa.types.is_string(t):
        return "utf8"
    if pa.types.is_null(t):
        return "null"
    if pa.types.is_map(t):
        return "map"
    if pa.types.is_list(t):
        return "list"
    if pa.types.is_struct(t):
        return "struct"
    if pa.types.is_union(t):
        return "union"
    raise NotImplementedError(str(t))


def _buf(b: Optional[pa.Buffer], nbytes: int) -> bytes:
    if nbytes == 0:
        return b""
    assert b is not None and b.size >= nbytes, (None if b is None else b.size, nbytes)
    return b.to_pybytes()[:nbytes] if b.size != nbytes else b.to_pybytes()


def canon_from_arrow(arr: pa.Array) -> dict:
    """Exact buffers of a pyarrow array (offset must be 0: the product never exports slices)."""
    assert arr.offset == 0, "sliced arrays are not expected"
    t, n = arr.type, len(arr)
    kind = _kind_of(t)
    bufs = arr.buffers()
    validity = None
    if kind not in ("null", "union") and bufs[0] is not None:
        validity = _buf(bufs[0], (n + 7) // 8)
    out = _canon(kind, n, arr.null_count, validity)
    if kind in _W:
        out["buffers"] = [_buf(bufs[1], n * _W[kind])]
    elif kind.startswith("raw"):
        out["buffers"] = [_buf(bufs[1], n * int(kind[3:]))]
    elif kind == "bool":
        out["buffers"] = [_buf(bufs[1], (n + 7) // 8)]
    elif kind == "utf8":
        offs = _buf(bufs[1], 4 * (n + 1))
        last = struct.unpack_from("<i", offs, 4 * n)[0]
        out["buffers"] = [offs, _buf(bufs[2], last)]
    elif kind == "union":
        out["buffers"] = [_buf(bufs[1], n)]  # pyarrow keeps a null placeholder in slot 0
        out["children"] = [canon_from_arrow(arr.field(i)) for i in range(t.num_fields)]
    elif kind == "struct":
        out["children"] = [canon_from_arrow(arr.field(i)) for i in range(t.num_fields)]
    elif kind == "list":
        out["buffers"] = [_buf(bufs[1], 4 * (n + 1))]
        out["children"] = [canon_from_arrow(arr.values)]
    elif kind == "map":
        out["buffers"] = [_buf(bufs[1], 4 * (n + 1))]
        keys, items = canon_from_arrow(arr.keys), canon_from_arrow(arr.items)
        out["children"] = [_canon("struct", keys["length"], 0, None, [], [keys, items])]
    if kind == "null":
        out["null_count"] = n
    return out


def canon_from_batch(batch: pa.RecordBatch) -> List[dict]:
    return [canon_from_arrow(batch.column(i)) for i in range(batch.num_columns)]


def canon_to_arrow(c: dict, t: pa.DataType) -> pa.Array:
    """Build a pyarrow array of type `t` from canonical buffers (zero-copy of the bytes objects)."""
    n, kind = c["length"], c["kind"]
    v = pa.py_buffer(c["validity"]) if c["validity"] is not None else None
    nc = c["null_count"]
    if kind in _W or kind == "bool" or kind.startswith("raw"):
        return pa.Array.from_buffers(t, n, [v, pa.py_buffer(c["buffers"][0])], null_count=nc)
    if kind == "utf8":
        return pa.Array.from_buffers(t, n, [v, pa.py_buffer(c["buffers"][0]), pa.py_buffer(c["buffers"][1])], null_count=nc)
    if kind == "null":
        return pa.nulls(n)
    if kind == "struct":
        kids = [canon_to_arrow(ch, t.field(i).type) for i, ch in enumerate(c["children"])]
        return pa.Array.from_buffers(t, n, [v], null_count=nc, children=kids)
    if kind == "union":
        kids = [canon_to_arrow(ch, t.field(i).type) for i, ch in enumerate(c["children"])]
        return pa.Array.from_buffers(t, n, [None, pa.py_buffer(c["buffers"][0])], children=kids)
    if kind == "list":
        kid = canon_to_arrow(c["children"][0], t.value_type)
        return pa.Array.from_buffers(t, n, [v, pa.py_buffer(c["buffers"][0])], null_count=nc, children=[kid])
    if kind == "map":
        en = c["children"][0]
        et = pa.struct([t.key_field, t.item_field])
        kid = canon_to_arrow(en, et)
        return pa.Array.from_buffers(t, n, [v, pa.py_buffer(c["buffers"][0])], null_count=nc, children=[kid])
    raise NotImplementedError(kind)


def canon_to_batch(cols: List[dict], schema: pa.Schema) -> pa.RecordBatch:
    arrays = [canon_to_arrow(c, schema.field(i).type) for i, c in enumerate(cols)]
    return pa.RecordBatch.from_arrays(arrays, schema=schema)


def canon_diff(a: Any, b: Any, path: str = "") -> Optional[str]:
    """First difference between two canonical forms (None if identical)."""
    if isinstance(a, list) and isinstance(b, list):
        if len(a) != len(b):
            return f"{path}: list length {len(a)} != {len(b)}"
        for i, (x, y) in enumerate(zip(a, b)):
            d = canon_diff(x, y, f"{path}[{i}]")
            if d:
                return d
        return None
    if isinstance(a, dict) and isinstance(b, dict):
        for key in ("kind", "length", "null_count"):
            if a[key] != b[key]:
                return f"{path}.{key}: {a[key]!r} != {b[key]!r}"
        if a["length"] == 0:
            pass  # a zero-byte bitmap is indistinguishable from an absent one across the C Data Interface
        elif (a["validity"] is None) != (b["validity"] is None):
            return f"{path}.validity presence: {a['validity'] is not None} != {b['validity'] is not None}"
        elif a["validity"] != b["validity"]:
            return f"{path}.validity bytes differ"
        if len(a["buffers"]) != len(b["buffers"]):
            return f"{path}.buffers count {len(a['buffers'])} != {len(b['buffers'])}"
        for i, (x, y) in enumerate(zip(a["buffers"], b["buffers"])):
            if x != y:
                j = next((q for q in range(min(len(x), len(y))) if x[q] != y[q]), min(len(x), len(y)))
                return f"{path}.buffers[{i}] differ (len {len(x)} vs {len(y)}, first diff at byte {j})"
        return canon_diff(a["children"], b["children"], path + ".children")
    return None if a == b else f"{path}: {a!r} != {b!r}"


def canon_nbytes(c: Any) -> int:
    """Exact Arrow output bytes (SURVEY.md 8(d): B_out)."""
    if isinstance(c, list):
        return sum(canon_nbytes(x) for x in c)
    n = len(c["validity"]) if c["validity"] is not None else 0
    return n + sum(len(b) for b in c["buffers"]) + canon_nbytes(c["children"])


# --------------------------------------------------------------------------- #
# C oracle binding
# --------------------------------------------------------------------------- #
class _OrcArray(ctypes.Structure):
    _fields_ = [("kind", ctypes.c_int32), ("n_children", ctypes.c_int32), ("length", ctypes.c_int64),
                ("null_count", ctypes.c_int64), ("has_validity", ctypes.c_int32), ("n_buffers", ctypes.c_int32),
                ("validity", ctypes.c_void_p), ("validity_bytes", ctypes.c_int64),
                ("buf0", ctypes.c_void_p), ("buf0_bytes", ctypes.c_int64),
                ("buf1", ctypes.c_void_p), ("buf1_bytes", ctypes.c_int64)]


_DKIND = ["int32", "int64", "float32", "float64", "bool", "utf8", "int32", "int64", "int64", "utf8",
          "null", "struct", "union", "list", "map"]
ERR_NAMES = {0: "ok", 1: "eof", 2: "varint", 3: "bool", 4: "neg_len", 5: "branch", 6: "enum", 7: "schema", 8: "overflow", 11: "value", 12: "frame"}


def build_oracle(force: bool = False) -> str:
    so = os.path.join(HERE, "liboracle.so")
    src = os.path.join(HERE, "avro_oracle.c")
    if force or not os.path.exists(so) or (os.path.exists(src) and os.path.getmtime(src) > os.path.getmtime(so)):
        subprocess.check_call(["make", "-C", HERE, "-B", "liboracle.so"], stdout=subprocess.DEVNULL)
    return so


class COracle:
    def __init__(self):
        self.lib = L = ctypes.CDLL(build_oracle())
        L.orc_schema_parse.restype = ctypes.c_void_p
        L.orc_schema_parse.argtypes = [ctypes.c_char_p, ctypes.c_int64]
        L.orc_schema_free.argtypes = [ctypes.c_void_p]
        L.orc_schema_ok.argtypes = [ctypes.c_void_p]
        L.orc_schema_is_supported.argtypes = [ctypes.c_void_p]
        L.orc_decode.restype = ctypes.c_void_p
        L.orc_decode.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64]
        L.orc_decode_threaded.restype = ctypes.c_int64
        L.orc_decode_threaded.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64,
                                          ctypes.c_int64, ctypes.c_int, ctypes.c_void_p]
        L.orc_set_pin.argtypes = [ctypes.c_int]
        L.orc_set_pin.restype = None
        L.orc_clamp_chunks.restype = ctypes.c_int64
        L.orc_clamp_chunks.argtypes = [ctypes.c_int64, ctypes.c_int64]
        L.orc_batch_free.argtypes = [ctypes.c_void_p]
        L.orc_batch_error.argtypes = [ctypes.c_void_p]
        L.orc_batch_error_record.restype = ctypes.c_int64
        L.orc_batch_error_record.argtypes = [ctypes.c_void_p]
        L.orc_batch_n_arrays.argtypes = [ctypes.c_void_p]
        L.orc_batch_array.restype = ctypes.POINTER(_OrcArray)
        L.orc_batch_array.argtypes = [ctypes.c_void_p, ctypes.c_int]

    # -- schema -------------------------------------------------------------
    def schema(self, schema_json: str):
        b = schema_json.encode("utf-8")
        h = self.lib.orc_schema_parse(b, len(b))
        return h

    def schema_free(self, h):
        self.lib.orc_schema_free(h)

    def is_supported(self, schema_json: str) -> bool:
        h = self.schema(schema_json)
        try:
            return bool(self.lib.orc_schema_is_supported(h))
        finally:
            self.schema_free(h)

    # -- decode -------------------------------------------------------------
    def _canon_batch(self, b) -> List[dict]:
        L = self.lib
        err = L.orc_batch_error(b)
        if err:
            raise DecodeError(ERR_NAMES.get(err, str(err)), L.orc_batch_error_record(b))
        n = L.orc_batch_n_arrays(b)
        pos = 0

        def grab(p, nb):
            return ctypes.string_at(p, nb) if nb else b""

        def rec():
            nonlocal pos
            a = L.orc_batch_array(b, pos).contents
            pos += 1
            kind = _DKIND[a.kind]
            validity = grab(a.validity, a.validity_bytes) if a.has_validity else None
            bufs = []
            if a.n_buffers >= 1:
                bufs.append(grab(a.buf0, a.buf0_bytes))
            if a.n_buffers >= 2:
                bufs.append(grab(a.buf1, a.buf1_bytes))
            kids = [rec() for _ in range(a.n_children)]
            return _canon(kind, a.length, a.null_count, validity, bufs, kids)

        cols = []
        while pos < n:
            cols.append(rec())
        return cols

    def decode_packed(self, schema_json: str, data, offsets, n: int) -> List[dict]:
        """data: bytes-like/numpy uint8, offsets: numpy int64[n+1]."""
        import numpy as np
        data = np.ascontiguousarray(np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else data)
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        h = self.schema(schema_json)
        try:
            if not self.lib.orc_schema_ok(h):
                raise DecodeError("schema")
            b = self.lib.orc_decode(h, data.ctypes.data, offsets.ctypes.data, n)
            try:
                return self._canon_batch(b)
            finally:
                self.lib.orc_batch_free(b)
        finally:
            self.schema_free(h)

    def decode(self, schema_json: str, records: List[bytes]) -> List[dict]:
        data, offsets = pack_records(records)
        return self.decode_packed(schema_json, data, offsets, len(records))

    def decode_threaded_packed(self, schema_json: str, data, offsets, n: int, num_chunks: int, threads: int,
                               materialize: bool = True):
        """per_datum_deserialize_threaded analogue.  Returns list of canonical batches (or the
        chunk count when materialize=False, which is what the timed CPU baseline uses)."""
        import numpy as np
        h = self.schema(schema_json)
        try:
            if not self.lib.orc_schema_ok(h):
                raise DecodeError("schema")
            k = self.lib.orc_clamp_chunks(num_chunks, n)
            out = (ctypes.c_void_p * k)()
            self.lib.orc_decode_threaded(h, data.ctypes.data, offsets.ctypes.data, n, num_chunks, threads, out)
            try:
                if not materialize:
                    for i in range(k):
                        e = self.lib.orc_batch_error(out[i])
                        if e:
                            raise DecodeError(ERR_NAMES.get(e, str(e)), self.lib.orc_batch_error_record(out[i]))
                    return k
                return [self._canon_batch(out[i]) for i in range(k)]
            finally:
                for i in range(k):
                    self.lib.orc_batch_free(out[i])
        finally:
            self.schema_free(h)


def pack_records(records: List[bytes]):
    """BinaryArray::from_vec analogue (deserialize.rs:90): contiguous values + int64 offsets."""
    import numpy as np
    lens = np.fromiter((len(r) for r in records), dtype=np.int64, count=len(records))
    offsets = np.zeros(len(records) + 1, dtype=np.int64)
    np.cumsum(lens, out=offsets[1:])
    data = np.frombuffer(b"".join(records), dtype=np.uint8)
    if data.size == 0:
        data = np.zeros(1, dtype=np.uint8)[:0]
    return data, offsets


# --------------------------------------------------------------------------- #
# Avro encoder + random values (test inputs; grammar of fast_encode.rs:397-599)
# --------------------------------------------------------------------------- #
def zigzag_bytes(v: int) -> bytes:
    """write_zigzag_long, fast_encode.rs:586-593"""
    u = ((v << 1) ^ (v >> 63)) & 0xFFFFFFFFFFFFFFFF
    out = bytearray()
    while u >= 0x80:
        out.append((u & 0x7F) | 0x80)
        u >>= 7
    out.append(u)
    return bytes(out)


def encode_value(s: AvroSchema, v: Any, out: bytearray, neg_blocks: bool = False):
    """Value model: None=null; union -> (branch, value); record -> dict; array -> list;
    map -> list of (key, value); enum -> symbol index; string -> str or bytes."""
    k = s.kind
    if k == "null":
        return
    if k == "boolean":
        out.append(1 if v else 0)
    elif k in ("int", "long", "date", "timestamp-millis", "timestamp-micros", "enum", "time-millis", "time-micros"):
        out += zigzag_bytes(int(v))
    elif k in ("bytes", "uuid", "decimal-bytes"):   # uuid: its text; decimal: the unscaled value's big-endian bytes
        b = v.encode("ascii") if isinstance(v, str) else bytes(v)
        out += zigzag_bytes(len(b))
        out += b
    elif k in ("fixed", "decimal-fixed"):
        assert len(v) == s.size
        out += bytes(v)
    elif k == "float":
        out += struct.pack("<f", v)
    elif k == "double":
        out += struct.pack("<d", v)
    elif k == "string":
        b = v.encode("utf-8") if isinstance(v, str) else bytes(v)
        out += zigzag_bytes(len(b))
        out += b
    elif k == "record":
        for fname, fs, _ in s.fields:
            encode_value(fs, v[fname], out, neg_blocks)
    elif k == "union":
        idx, inner = v
        out += zigzag_bytes(idx)
        encode_value(s.variants[idx], inner, out, neg_blocks)
    elif k in ("array", "map"):
        items = list(v)
        if items:
            body = bytearray()
            for it in items:
                if k == "map":
                    kb = it[0].encode("utf-8") if isinstance(it[0], str) else bytes(it[0])
                    body += zigzag_bytes(len(kb))
                    body += kb
                    encode_value(s.values, it[1], body, neg_blocks)
                else:
                    encode_value(s.items, it, body, neg_blocks)
            if neg_blocks:
                out += zigzag_bytes(-len(items))
                out += zigzag_bytes(len(body))
            else:
                out += zigzag_bytes(len(items))
            out += body
        out += zigzag_bytes(0)
    else:
        raise NotImplementedError(k)


def encode_datum(s: AvroSchema, v: Any, neg_blocks: bool = False) -> bytes:
    out = bytearray()
    encode_value(s, v, out, neg_blocks)
    return bytes(out)


def random_value(s: AvroSchema, rng, depth: int = 0) -> Any:
    k = s.kind
    if k == "null":
        return None
    if k == "boolean":
        return rng.random() < 0.5
    if k in ("int", "date"):
        return rng.choice([0, 1, -1, 63, 64, -64, -65, 2**31 - 1, -2**31, rng.randint(-10**6, 10**6)])
    if k in ("long", "timestamp-millis", "timestamp-micros"):
        return rng.choice([0, -1, 2**63 - 1, -2**63, rng.randint(-2**40, 2**40), rng.randint(0, 200)])
    if k == "time-millis":
        return rng.randrange(86_400_000)
    if k == "time-micros":
        return rng.randrange(86_400_000_000)
    if k == "bytes":
        return bytes(rng.randrange(256) for _ in range(rng.choice([0, 0, 1, 5, 16, 33, rng.randint(0, 120)])))
    if k == "fixed":
        return bytes(rng.randrange(256) for _ in range(s.size))
    if k == "uuid":
        h = "%032x" % rng.getrandbits(128)
        if rng.random() < 0.5:
            h = h.upper()
        return h if rng.random() < 0.2 else f"{h[:8]}-{h[8:12]}-{h[12:16]}-{h[16:20]}-{h[20:]}"
    if k in ("decimal-bytes", "decimal-fixed"):
        lim = 10 ** s.precision - 1
        v = rng.choice([0, 1, -1, lim, -lim, rng.randint(-lim, lim), max(-lim, min(lim, rng.randint(-1000, 1000)))])
        if k == "decimal-fixed":
            return v.to_bytes(s.size, "big", signed=True) if s.size and -(1 << (8 * s.size - 1)) <= v < (1 << (8 * s.size - 1)) else bytes(s.size)
        n = max(1, (v.bit_length() + 8) // 8)
        n = min(16, n + rng.choice([0, 0, 1, 3]))  # writers may pad with sign bytes
        return v.to_bytes(n, "big", signed=True) if rng.random() < 0.95 else b""
    if k == "float":
        return struct.unpack("<f", struct.pack("<f", rng.uniform(-1e6, 1e6)))[0]
    if k == "double":
        return rng.uniform(-1e12, 1e12)
    if k == "string":
        n = rng.choice([0, 0, 1, 3, 7, 15, 16, 17, 31, 40, rng.randint(0, 200)])
        return "".join(rng.choice("abcdefghijklmnopqrstuvwxyzé✓") for _ in range(n))
    if k == "enum":
        return rng.randrange(len(s.symbols))
    if k == "record":
        return {f[0]: random_value(f[1], rng, depth + 1) for f in s.fields}
    if k == "union":
        i = rng.randrange(len(s.variants))
        return (i, random_value(s.variants[i], rng, depth + 1))
    if k == "array":
        return [random_value(s.items, rng, depth + 1) for _ in range(rng.choice([0, 0, 1, 2, 3, 5]))]
    if k == "map":
        return [("k%d" % rng.randint(0, 99999), random_value(s.values, rng, depth + 1)) for _ in range(rng.choice([0, 0, 1, 2, 4]))]
    raise NotImplementedError(k)


def random_schema_json(rng, max_depth: int = 3, wide: bool = False) -> str:
    """A random schema inside the supported subset (no nullable maps: SURVEY.md 8(a) hazard).  wide=True mixes in the
    wider subset's leaves (bytes, fixed, uuid, decimal, time-*) and references to named types defined earlier."""
    counter = [0]
    defined = []  # names of fixed / enum types a later field may reference by name

    def nm(prefix):
        counter[0] += 1
        return f"{prefix}{counter[0]}"

    def wide_leaf():
        r = rng.randrange(9)
        if r == 0:
            return "bytes"
        if r == 1:
            name = nm("Fx")
            defined.append(name)
            return {"type": "fixed", "name": name, "size": rng.choice([1, 1, 3, 4, 7, 16, 20])}
        if r == 2:
            return {"type": "string", "logicalType": "uuid"}
        if r == 3:
            p = rng.randint(1, 38)
            return {"type": "bytes", "logicalType": "decimal", "precision": p, "scale": rng.randint(0, p)}
        if r == 4:
            size = rng.randint(1, 16)
            p = rng.randint(1, min(38, max(1, int((8 * size - 1) * 0.30103))))
            return {"type": "fixed", "name": nm("Dx"), "size": size, "logicalType": "decimal", "precision": p, "scale": rng.randint(0, p)}
        if r == 5:
            return {"type": "int", "logicalType": "time-millis"}
        if r == 6:
            return {"type": "long", "logicalType": "time-micros"}
        if r == 7 and defined:
            return rng.choice(defined)  # a reference by name
        return "bytes"

    def leaf():
        if wide and rng.random() < 0.5:
            return wide_leaf()
        return rng.choice(["int", "long", "float", "double", "boolean", "string",
                           {"type": "int", "logicalType": "date"},
                           {"type": "long", "logicalType": "timestamp-millis"},
                           {"type": "long", "logicalType": "timestamp-micros"}])

    def enum():
        name = nm("E")
        if wide:
            defined.append(name)
        return {"type": "enum", "name": name, "symbols": [f"S{i}" * rng.randint(1, 3) for i in range(rng.randint(1, 5))]}

    def record(d, in_nullable):
        return {"type": "record", "name": nm("R"), "fields": [{"name": nm("f"), "type": typ(d + 1, in_nullable)} for _ in range(rng.randint(1, 4))]}

    def typ(d, in_nullable=False, allow_union=True):
        r = rng.random()
        if d >= max_depth or r < 0.35:
            return enum() if rng.random() < 0.15 else leaf()
        if r < 0.5 and allow_union:
            inner = typ(d + 1, True, False)
            if isinstance(inner, dict) and inner.get("type") == "map":
                inner = leaf()
            return ["null", inner] if rng.random() < 0.7 else [inner, "null"]
        if r < 0.62 and allow_union:
            # N-variant union: distinct kinds; maps cannot be variants (default_field_name is unimplemented for Map)
            pool = ["null", "string", "int", "long", "float", "double", "boolean"]
            rng.shuffle(pool)
            vs = pool[:rng.randint(2, 5)]
            if len(vs) == 2 and "null" in vs:
                vs.append("string" if "string" not in vs else "long")
            if rng.random() < 0.4:
                vs.append(record(d + 1, True))
            if rng.random() < 0.3:
                vs.append(enum())
            if rng.random() < 0.3:
                vs.append({"type": "array", "items": typ(d + 1, True, False)})
            return vs
        if r < 0.75:
            return record(d, in_nullable)
        if r < 0.9:
            return {"type": "array", "items": typ(d + 1, True)}  # item fields are nullable=true: no maps below
        if in_nullable:
            return leaf()
        return {"type": "map", "values": typ(d + 1, False)}

    top = {"type": "record", "name": "Top", "fields": [{"name": nm("c"), "type": typ(0)} for _ in range(rng.randint(1, 6))]}
    return json.dumps(top)


# --------------------------------------------------------------------------- #
# Arrow -> Avro: pure-Python restatement of ruhvro/src/fast_encode.rs (test oracle for the
# serialize direction).  Walks pyarrow arrays through their raw buffers so that null slots of
# NON-nullable Avro fields encode whatever value the slot holds, exactly like `array.value(row)`
# in the reference (fast_encode.rs:401-409).
# --------------------------------------------------------------------------- #
class EncodeError(ValueError):
    pass


def _bit(buf: Optional[pa.Buffer], i: int) -> bool:
    if buf is None:
        return True
    return bool((buf.to_pybytes()[i >> 3] >> (i & 7)) & 1) if False else bool((memoryview(buf)[i >> 3] >> (i & 7)) & 1)


class _Enc:
    def __init__(self, s: AvroSchema, arr: pa.Array, nullable=False, null_first=False):
        self.s, self.k, self.nullable, self.null_first = s, s.kind, nullable, null_first
        self.arr = arr
        self.off = arr.offset if arr is not None else 0
        bufs = arr.buffers() if arr is not None else []
        self.validity = bufs[0] if bufs else None
        self.children: List[_Enc] = []
        t = arr.type if arr is not None else None
        k = self.k
        # exact downcasts, like `downcast::<Int32Array>` etc. in the reference (fast_encode.rs:196-204, 292-324)
        if k == "int":
            self._need(pa.types.is_int32(t), "Int32")
        elif k == "date":
            self._need(pa.types.is_date32(t), "Date32")
        elif k == "long":
            self._need(pa.types.is_int64(t), "Int64")
        elif k == "timestamp-millis":
            self._need(pa.types.is_timestamp(t) and t.unit == "ms", "Timestamp(ms)")
        elif k == "timestamp-micros":
            self._need(pa.types.is_timestamp(t) and t.unit == "us", "Timestamp(us)")
        elif k == "float":
            self._need(pa.types.is_float32(t), "Float32")
        elif k == "double":
            self._need(pa.types.is_float64(t), "Float64")
        elif k == "boolean":
            self._need(pa.types.is_boolean(t), "Boolean")
        elif k in ("string", "enum"):
            self._need(pa.types.is_string(t), "Utf8")
        elif k == "record":
            self._need(pa.types.is_struct(t), "Struct")
            names = [t.field(i).name for i in range(t.num_fields)]
            for fname, fs, _ in s.fields:  # match by NAME (fast_encode.rs:157-181)
                if fname not in names:
                    raise EncodeError(f"Arrow struct missing column '{fname}' required by Avro schema. Available columns: {names}")
                self.children.append(_make_enc(fs, arr.field(names.index(fname))))
        elif k == "union":
            self._need(pa.types.is_union(t) and t.mode == "sparse", "sparse Union")
            if t.num_fields != len(s.variants):
                raise EncodeError("fast_encode: union variant count mismatch")
            # Avro variant i is the Arrow child whose type code is i (`ua.child(i as i8)`, fast_encode.rs:276)
            codes = list(t.type_codes)
            if sorted(codes) != list(range(len(codes))):
                raise EncodeError(f"fast_encode: union type codes {codes} are not a permutation of 0..{len(codes) - 1}")
            for i, v in enumerate(s.variants):
                self.children.append(_make_enc(v, arr.field(codes.index(i))))
        elif k == "array":
            self._need(pa.types.is_list(t) and not pa.types.is_map(t), "List")
            self.children.append(_make_enc(s.items, arr.values))
        elif k == "map":
            self._need(pa.types.is_map(t), "Map")
            entries = arr.values  # the raw entries struct: field() applies its own offset, which arr.keys / arr.items ignore
            self.children.append(_Enc(AvroSchema("string"), entries.field(0)))
            self.children.append(_make_enc(s.values, entries.field(1)))

    def _need(self, ok, what):
        if not ok:
            raise EncodeError(f"fast_encode: arrow array downcast failed (expected {what}, got {self.arr.type})")


def _make_enc(s: AvroSchema, arr: pa.Array) -> _Enc:
    if s.kind == "union" and len(s.variants) == 2 and any(v.kind == "null" for v in s.variants):
        null_first = s.variants[0].kind == "null"
        inner = s.variants[1] if null_first else s.variants[0]
        if inner.kind in ("null", "union"):
            raise EncodeError("fast_encode: unsupported nullable inner type")
        return _Enc(inner, arr, True, null_first)
    if s.kind == "null":
        e = _Enc.__new__(_Enc)
        e.s, e.k, e.nullable, e.null_first, e.arr, e.off, e.validity, e.children = s, "null", False, False, arr, 0, None, []
        return e
    return _Enc(s, arr)


def _np_view(buf: pa.Buffer, dtype):
    import numpy as np
    return np.frombuffer(buf, dtype=dtype)


def _write(e: _Enc, row: int, out: bytearray):
    """FieldEncoder::write (fast_encode.rs:397-502); `row` is the logical row of e.arr.  Struct fields and sparse
    union children come from `field()`, which has applied the parent's offset, so they get the same logical row; list
    and map offsets index the raw child (`arr.values`, the entries' fields) logically."""
    k = e.k
    if k == "null":
        return
    i = row + e.off
    if e.nullable:
        is_null = e.validity is not None and not _bit(e.validity, i)
        out += zigzag_bytes((0 if e.null_first else 1) if is_null else (1 if e.null_first else 0))
        if is_null:
            return
    bufs = e.arr.buffers()
    if k in ("int", "date"):
        out += zigzag_bytes(int(_np_view(bufs[1], "<i4")[i]))
    elif k in ("long", "timestamp-millis", "timestamp-micros"):
        out += zigzag_bytes(int(_np_view(bufs[1], "<i8")[i]))
    elif k == "float":
        out += bytes(memoryview(bufs[1])[4 * i:4 * i + 4])
    elif k == "double":
        out += bytes(memoryview(bufs[1])[8 * i:8 * i + 8])
    elif k == "boolean":
        out.append(1 if _bit(bufs[1], i) else 0)
    elif k in ("string", "enum"):
        offs = _np_view(bufs[1], "<i4")
        s0, s1 = int(offs[i]), int(offs[i + 1])
        raw = bytes(memoryview(bufs[2])[s0:s1]) if bufs[2] is not None else b""
        if k == "string":
            out += zigzag_bytes(len(raw))
            out += raw
        else:
            sym = raw.decode("utf-8", "replace")
            if sym not in e.s.symbols:
                raise EncodeError(f"fast_encode: enum symbol '{sym}' not in schema")
            out += zigzag_bytes(e.s.symbols.index(sym))
    elif k == "record":
        for ch in e.children:  # field() already applied the struct's offset: children take the LOGICAL row
            _write(ch, row, out)
    elif k == "union":
        tid = int(_np_view(bufs[0] if len(bufs) == 1 else bufs[1], "i1")[i])
        if tid < 0 or tid >= len(e.children):
            raise EncodeError(f"fast_encode: union type_id {tid} out of range")
        out += zigzag_bytes(tid)
        _write(e.children[tid], row, out)  # sparse: field() already applied the union's offset
    else:  # array / map (ListEncoder / MapEncoder :518-554)
        offs = _np_view(bufs[1], "<i4")
        s0, s1 = int(offs[i]), int(offs[i + 1])
        if s1 > s0:
            out += zigzag_bytes(s1 - s0)
            for j in range(s0, s1):
                if k == "map":
                    _write(e.children[0], j, out)
                    _write(e.children[1], j, out)
                else:
                    _write(e.children[0], j, out)
        out += zigzag_bytes(0)


def py_encode(schema: AvroSchema, batch: pa.RecordBatch, num_chunks: int = 1) -> List[List[bytes]]:
    """serialize_record_batch (serialize.rs:38-67) + serialize_chunk (fast_encode.rs:27-53): one list of
    datums per chunk."""
    if not is_supported(schema):
        raise EncodeError("schema not supported by the direct encoder")
    sa = batch.to_struct_array()
    top = _Enc(schema, sa)
    n = batch.num_rows
    k = clamp_chunks(num_chunks, n)
    out = []
    for r0, r1 in chunk_bounds(n, k):
        rows = []
        for r in range(r0, r1):
            b = bytearray()
            for ch in top.children:
                _write(ch, r, b)
            rows.append(bytes(b))
        out.append(rows)
    return out
