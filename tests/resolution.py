"""Schema resolution, restated for the tests (rv_schema_resolve / Schema.read_as / `reader_schema=`).

resolve_value(writer, reader, v) converts a value of the oracle's value model (oracle/pyoracle.py encode_value) written
with `writer` into the reader's, following the rules in DESIGN.md §7; the expected batches of a resolved decode are then
the oracle's decode of the re-encoded values with the reader's schema.  random_evolution(rng, writer_json) makes a reader
schema from a writer schema the way schemas evolve in practice.  Test infrastructure only."""
import copy
import json

import numpy as np

from oracle import pyoracle as po


class Unmapped(ValueError):
    """A writer enum symbol the reader has neither a symbol nor a default for."""


def _short(name):
    return name.rpartition(".")[2] if name else name


class ReaderMeta:
    """What oracle/pyoracle.py's schema model leaves out of a reader schema: field defaults and aliases, enum defaults
    (keyed by the unqualified type name; the generated schemas have unique names)."""

    def __init__(self, reader_json: str):
        self.fields, self.enum_default = {}, {}
        self._walk(json.loads(reader_json))

    def _walk(self, j):
        if isinstance(j, list):
            for v in j:
                self._walk(v)
        elif isinstance(j, dict):
            t = j.get("type")
            if t in ("record", "error"):
                self.fields[_short(j["name"])] = {f["name"]: f for f in j["fields"]}
                for f in j["fields"]:
                    self._walk(f if isinstance(f["type"], str) and f["type"] in ("array", "map", "enum") else f["type"])
            elif t == "enum":
                if "default" in j:
                    self.enum_default[_short(j["name"])] = j["default"]
            elif t == "array":
                self._walk(j["items"])
            elif t == "map":
                self._walk(j["values"])
            elif isinstance(t, (dict, list)):
                self._walk(t)


def _nullable(s):
    """(null branch index, inner) of ["null", T] / [T, "null"], else None."""
    if s.kind == "union" and len(s.variants) == 2:
        for i, v in enumerate(s.variants):
            if v.kind == "null":
                return i, s.variants[1 - i]
    return None


def _to_float(v, dtype):
    return float(np.array([v], dtype=np.int64).astype(dtype)[0])   # one rounding step, to nearest even


def default_value(s, d, meta):
    """The value of a reader-only field's default `d` (JSON) for its schema `s`."""
    if s.kind == "union" and s.variants[0].kind == "null":   # a union's default belongs to its first branch
        assert d is None
        return (0, None)
    nb = _nullable(s)
    if nb is not None:
        return (0, default_value(nb[1], d, meta))
    k = s.kind
    if k == "null":
        return None
    if k == "float":
        return float(np.float32(d))
    if k == "double":
        return float(d)
    if k == "bytes":
        return bytes(ord(c) for c in d)
    if k == "enum":
        return s.symbols.index(d)
    return d


def resolve_value(w, r, v, meta: ReaderMeta):
    nb = _nullable(r)
    if nb is not None:
        null_idx, ri = nb
        wn = _nullable(w)
        if wn is not None:
            i, x = v
            if w.variants[i].kind == "null":
                return (null_idx, None)
            return (1 - null_idx, resolve_value(wn[1], ri, x, meta))
        return (1 - null_idx, resolve_value(w, ri, v, meta))
    if r.kind == "union":
        i, x = v
        return (i, resolve_value(w.variants[i], r.variants[i], x, meta))
    wk, rk = w.kind, r.kind
    if wk in ("int", "long") and rk == "float":
        return _to_float(v, np.float32)
    if wk in ("int", "long") and rk == "double":
        return _to_float(v, np.float64)
    if wk == "string" and rk == "bytes":
        return v.encode("utf-8") if isinstance(v, str) else bytes(v)
    if rk == "enum":
        sym = w.symbols[v]
        if sym in r.symbols:
            return r.symbols.index(sym)
        d = meta.enum_default.get(_short(r.fullname))
        if d is None:
            raise Unmapped(sym)
        return r.symbols.index(d)
    if rk == "record":
        fm = meta.fields[_short(r.fullname)]
        wnames = {f[0]: f[1] for f in w.fields}
        out = {}
        for name, rs, _ in r.fields:
            src = name if name in wnames else next((a for a in fm[name].get("aliases", []) if a in wnames), None)
            out[name] = resolve_value(wnames[src], rs, v[src], meta) if src is not None else default_value(rs, fm[name]["default"], meta)
        return out
    if rk == "array":
        return [resolve_value(w.items, r.items, x, meta) for x in v]
    if rk == "map":
        return [(key, resolve_value(w.values, r.values, x, meta)) for key, x in v]
    return v


def expected_batches(coracle, writer_json, reader_json, values, k, wide=False):
    """The oracle's batches of a resolved decode of `values` (written with `writer_json`), or ("error", record) when a
    record has an enum symbol the reader cannot map."""
    ws, rs = po.parse_schema(writer_json, wide=wide), po.parse_schema(reader_json, wide=wide)
    meta = ReaderMeta(reader_json)
    rvals = []
    for i, v in enumerate(values):
        try:
            rvals.append(resolve_value(ws, rs, v, meta))
        except Unmapped:
            return ("error", i)
    recs = [po.encode_datum(rs, v) for v in rvals]
    n = len(recs)
    if wide:
        return [po.py_decode(rs, recs[a:b]) for a, b in po.chunk_bounds(n, po.clamp_chunks(k, n))]
    data, off = po.pack_records(recs)
    return coracle.decode_threaded_packed(reader_json, data, off, n, k, threads=4)


# ---- random evolutions ----------------------------------------------------------------------------------------------
_PROMOTE = {"int": ["long", "float", "double"], "long": ["float", "double"], "float": ["double"]}


def random_evolution(rng, writer_json: str, wide: bool = False, unmapped_ok: bool = False) -> str:
    """A reader schema for `writer_json`: at every depth it drops, adds (with defaults), reorders and renames (with an
    alias) record fields, promotes leaves, adds and removes enum symbols (with a default, and without one when
    `unmapped_ok`) and makes fields optional.  Named types keep their names.  (A reordering that moves a named type's
    definition behind a reference to it is drawn again.)"""
    import pyruhvro_b200 as pr
    for _ in range(50):
        rj = _evolve_once(rng, writer_json, wide, unmapped_ok)
        if po.is_supported(po.parse_schema(rj, wide=wide)) and pr.Schema(rj).is_supported:   # (nesting limits, too)
            return rj
    return writer_json


def _evolve_once(rng, writer_json, wide, unmapped_ok):
    j = copy.deepcopy(json.loads(writer_json))
    counter = [0]
    seen_enums = {}

    def fresh(prefix):
        counter[0] += 1
        return f"{prefix}{counter[0]}"

    def null_default_type():
        # optional fields of every kind whose default is null: a null of the reader's type, whatever it holds
        kinds = ["record", "array", "union", "array_of_records"] + (["fixed", "decimal", "decimal_fixed", "uuid"] if wide else [])
        k = rng.choice(kinds)
        if k == "record":
            t = {"type": "record", "name": fresh("NR"), "fields": [{"name": "x", "type": "int"}, {"name": "y", "type": ["null", "string"]},
                                                                    {"name": "z", "type": {"type": "array", "items": "long"}}]}
        elif k == "array":
            t = {"type": "array", "items": "string"}
        elif k == "array_of_records":
            t = {"type": "array", "items": {"type": "record", "name": fresh("NI"), "fields": [{"name": "s", "type": "string"},
                                                                                              {"name": "e", "type": {"type": "enum", "name": fresh("NIE"), "symbols": ["U", "V"]}}]}}
        elif k == "union":
            return ["null", "string", "int", {"type": "record", "name": fresh("NU"), "fields": [{"name": "b", "type": "boolean"}]}]
        elif k == "fixed":
            t = {"type": "fixed", "name": fresh("NF"), "size": 5}
        elif k == "decimal":
            t = {"type": "bytes", "logicalType": "decimal", "precision": 10, "scale": 2}
        elif k == "decimal_fixed":
            t = {"type": "fixed", "name": fresh("ND"), "size": 8, "logicalType": "decimal", "precision": 12, "scale": 3}
        else:
            t = {"type": "string", "logicalType": "uuid"}
        return ["null", t]

    def new_field():
        r = rng.randrange(12 if wide else 11)
        name = fresh("new_")
        if r == 10:
            return {"name": name, "type": null_default_type(), "default": None}
        if r == 0:
            return {"name": name, "type": ["null", "string"], "default": None}
        if r == 1:
            return {"name": name, "type": "int", "default": rng.choice([0, 7, -2**31, 2**31 - 1])}
        if r == 2:
            return {"name": name, "type": "long", "default": rng.choice([-3, 2**63 - 1, -2**63])}
        if r == 3:
            return {"name": name, "type": "double", "default": rng.choice([1.5, -0.0, 1e300])}
        if r == 4:
            return {"name": name, "type": "float", "default": rng.choice([0.25, 0.1, 3])}
        if r == 5:
            return {"name": name, "type": "boolean", "default": rng.random() < 0.5}
        if r == 6:
            return {"name": name, "type": "string", "default": rng.choice(["", "dflt", "é✓ text", "x" * 40])}
        if r == 7:
            syms = ["P", "Q", "R"]
            return {"name": name, "type": {"type": "enum", "name": fresh("NE"), "symbols": syms}, "default": rng.choice(syms)}
        if r == 8:
            return {"name": name, "type": ["string", "null"], "default": "s"}
        if r == 9:
            return {"name": name, "type": ["null", {"type": "long", "logicalType": "timestamp-millis"}], "default": None}
        return {"name": name, "type": "bytes", "default": "ÿ\u0000ab"}

    def evolve(t, promote_ok=True):
        if isinstance(t, str):
            if promote_ok and t in _PROMOTE and rng.random() < 0.3:
                return rng.choice(_PROMOTE[t])
            if promote_ok and wide and t in ("string", "bytes") and rng.random() < 0.3:
                return "bytes" if t == "string" else "string"
            return t
        if isinstance(t, list):
            two_with_null = len(t) == 2 and "null" in t
            return [evolve(v, two_with_null) for v in t]   # (N-variant unions: a promoted branch could repeat a kind)
        kind = t.get("type")
        if kind in ("record", "error"):
            return record(t)
        if kind == "enum":
            if t["name"] in seen_enums:
                return seen_enums[t["name"]]
            syms = list(t["symbols"])
            e = dict(t)
            r = rng.random()
            if r < 0.3:
                syms.insert(rng.randint(0, len(syms)), fresh("Z"))
            elif r < 0.6 and len(syms) > 1:
                syms.pop(rng.randrange(len(syms)))
                if not unmapped_ok or rng.random() < 0.5:
                    e["default"] = rng.choice(syms)
            elif r < 0.7:
                rng.shuffle(syms)
            e["symbols"] = syms
            seen_enums[t["name"]] = e
            return e
        if kind == "array":
            return dict(t, items=evolve(t["items"]))
        if kind == "map":
            return dict(t, values=evolve(t["values"]))
        if promote_ok and isinstance(kind, str) and kind in _PROMOTE and "logicalType" not in t and rng.random() < 0.3:
            return rng.choice(_PROMOTE[kind])
        return t

    def optional(t):
        if isinstance(t, list) or (isinstance(t, dict) and t.get("type") == "map"):
            return t
        return ["null", t] if rng.random() < 0.6 else [t, "null"]

    def record(rec):
        fields = []
        for f in rec["fields"]:
            if len(rec["fields"]) > 1 and rng.random() < 0.15:
                continue   # dropped
            if isinstance(f["type"], str) and f["type"] in ("array", "map", "enum"):
                nf = evolve_field_object(f)
            else:
                nf = dict(f, type=evolve(f["type"]))
            if rng.random() < 0.1:
                nf["aliases"] = [f["name"]]
                nf["name"] = fresh("renamed_")
            if rng.random() < 0.12:
                nf["type"] = optional(nf["type"])
            fields.append(nf)
        if not fields:
            fields.append(dict(rec["fields"][0]))
        for _ in range(rng.choice([0, 0, 1, 2])):
            fields.insert(rng.randint(0, len(fields)), new_field())
        if rng.random() < 0.5:
            rng.shuffle(fields)
        return dict(rec, fields=fields)

    def evolve_field_object(f):
        # {"name":..,"type":"array","items":..}: the field object is the type (schema.cpp)
        t = {k: v for k, v in f.items() if k not in ("name", "aliases", "default", "doc")}
        nt = evolve(t)
        out = {"name": f["name"], "type": nt}
        return out

    return json.dumps(record(j))


# The Kafka v2 reader of the tests and tools/bench_resolve.py (workloads.kafka_v2_schema).
from workloads import kafka_v2_schema as kafka_v2  # noqa: E402,F401
