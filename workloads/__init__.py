"""Synthetic benchmark workloads (BASELINE.json configs; SURVEY.md 8(d)).  Bench/test infrastructure.

    C1  10 k records, generate_avro.py schema, num_chunks = 8          (README bench)
    C2  flat primitives, 10 M                                           (benches/common/mod.rs:37-63)
    C3  generate_avro.py "Kafka" schema, 10 M                           (scripts/generate_avro.py:12-62)
    C4  wide 8-variant unions + three maps, 10 M                        (divergence stress)
    C5  C3 at 100 M over 2/4/8 GPUs
"""
from __future__ import annotations

import ctypes
import json
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(HERE, "libavrogen.so")
_SRC = os.path.join(HERE, "avrogen.c")

KAFKA_SCHEMA = json.dumps({  # scripts/generate_avro.py:12-41, verbatim structure
    "type": "record", "name": "User",
    "fields": [
        {"name": "name", "type": ["null", "string"], "default": None},
        {"name": "age", "type": ["null", "int"], "default": None},
        {"name": "emails", "type": {"type": "array", "items": "string"}},
        {"name": "address", "type": ["null", {"type": "record", "name": "Address", "fields": [
            {"name": "street", "type": "string"}, {"name": "city", "type": "string"}, {"name": "zipcode", "type": "string"}]}],
         "default": None},
        {"name": "phone_numbers", "type": {"type": "map", "values": "string"}},
        {"name": "preferences", "type": ["null", {"type": "record", "name": "Preferences", "fields": [
            {"name": "contact_method", "type": ["null", "string"], "default": None},
            {"name": "newsletter", "type": "boolean"}]}], "default": None},
        {"name": "status", "type": ["null", "string", "int", "boolean"], "default": None},
        {"name": "created_at", "type": "long"},
        {"name": "class", "type": {"type": "enum", "name": "enum_col", "symbols": ["A", "B", "C"]}},
    ]})

FLAT_SCHEMA = json.dumps({  # ruhvro/benches/common/mod.rs:37-50
    "type": "record", "name": "FlatPrim",
    "fields": [{"name": "i", "type": "int"}, {"name": "l", "type": "long"}, {"name": "f", "type": "float"},
               {"name": "d", "type": "double"}, {"name": "b", "type": "boolean"}, {"name": "s", "type": "string"}]})


def _wide_union(i):
    return ["null", "string", "int", "long", "float", "double", "boolean",
            {"type": "enum", "name": f"Kind{i}", "symbols": ["ALPHA", "BETA", "GAMMA", "DELTA"]}]


WIDE_SCHEMA = json.dumps({
    "type": "record", "name": "Wide",
    "fields": [{"name": "id", "type": "long"}] +
              [{"name": f"u{i}", "type": _wide_union(i)} for i in range(4)] +
              [{"name": "ms", "type": {"type": "map", "values": "string"}},
               {"name": "ml", "type": {"type": "map", "values": "long"}},
               {"name": "md", "type": {"type": "map", "values": "double"}}]})

ARRAY_MAP_SCHEMA = json.dumps({  # benches/common/mod.rs:137-147
    "type": "record", "name": "Collection",
    "fields": [{"name": "id", "type": "long"}, {"name": "tags", "type": {"type": "array", "items": "string"}},
               {"name": "props", "type": {"type": "map", "values": "string"}}]})

NESTED_SCHEMA = json.dumps({  # benches/common/mod.rs:102-119
    "type": "record", "name": "Outer",
    "fields": [{"name": "outer_id", "type": "long"},
               {"name": "inner", "type": {"type": "record", "name": "Inner", "fields": [
                   {"name": "x", "type": "int"}, {"name": "y", "type": "int"}, {"name": "label", "type": "string"}]}}]})

NULLABLE_SCHEMA = json.dumps({  # benches/common/mod.rs:67-79
    "type": "record", "name": "NullPrim",
    "fields": [{"name": "i", "type": ["null", "int"], "default": None}, {"name": "l", "type": ["null", "long"], "default": None},
               {"name": "d", "type": ["null", "double"], "default": None}, {"name": "b", "type": ["null", "boolean"], "default": None},
               {"name": "s", "type": ["null", "string"], "default": None}]})

def kafka_v2_schema(enum_symbols=("A", "B", "C", "D"), enum_default=None) -> str:
    """A reader of KAFKA_SCHEMA data ("Kafka v2", tools/bench_resolve.py): the bench's schema as a later version reads it: phone_numbers dropped, age widened to long, three new
    fields with defaults, more enum symbols, Address reshaped, created_at first."""
    enum = {"type": "enum", "name": "enum_col", "symbols": list(enum_symbols)}
    if enum_default is not None:
        enum["default"] = enum_default
    address = {"type": "record", "name": "Address", "fields": [
        {"name": "city", "type": "string"}, {"name": "street", "type": "string"},
        {"name": "country", "type": "string", "default": "US"}]}
    prefs = {"type": "record", "name": "Preferences", "fields": [
        {"name": "contact_method", "type": ["null", "string"], "default": None}, {"name": "newsletter", "type": "boolean"}]}
    return json.dumps({"type": "record", "name": "User", "fields": [
        {"name": "created_at", "type": "long"},
        {"name": "name", "type": ["null", "string"], "default": None},
        {"name": "age", "type": ["null", "long"], "default": None},
        {"name": "emails", "type": {"type": "array", "items": "string"}},
        {"name": "address", "type": ["null", address], "default": None},
        {"name": "preferences", "type": ["null", prefs], "default": None},
        {"name": "status", "type": ["null", "string", "int", "boolean"], "default": None},
        {"name": "class", "type": enum},
        {"name": "country", "type": ["null", "string"], "default": None},
        {"name": "score", "type": "double", "default": 0.0},
        {"name": "source", "type": "string", "default": "kafka"},
    ]})


CONFIGS = {
    "flat": (2, FLAT_SCHEMA), "kafka": (3, KAFKA_SCHEMA), "wide": (4, WIDE_SCHEMA),
    "array_map": (5, ARRAY_MAP_SCHEMA), "nested": (6, NESTED_SCHEMA), "nullable": (7, NULLABLE_SCHEMA),
}

_lib = None


def _load():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO) or os.path.getmtime(_SRC) > os.path.getmtime(_SO):
            subprocess.check_call(["gcc", "-O3", "-march=native", "-fPIC", "-shared", "-pthread", "-Wall", "-o", _SO, _SRC])
        _lib = ctypes.CDLL(_SO)
        _lib.avrogen_lens.argtypes = [ctypes.c_int, ctypes.c_int64, ctypes.c_int64, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_int]
        _lib.avrogen_fill.argtypes = [ctypes.c_int, ctypes.c_int64, ctypes.c_int64, ctypes.c_uint64, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
        _lib.avrogen_lens.restype = None
        _lib.avrogen_fill.restype = None
    return _lib


def build():
    _load()


def generate(name: str, n: int, seed: int = 42, r0: int = 0, threads: int = 0, alloc=None):
    """Returns (schema_json, data uint8[total], offsets int64[n+1]).  `alloc(nbytes) -> np.uint8 array`
    lets the caller provide pinned memory for the payload and offsets."""
    cfg, schema = CONFIGS[name]
    L = _load()
    threads = threads or min(32, os.cpu_count() or 1)
    lens = np.empty(n, dtype=np.int64)
    L.avrogen_lens(cfg, r0, n, seed, lens.ctypes.data, threads)
    if alloc is None:
        offsets = np.empty(n + 1, dtype=np.int64)
    else:
        offsets = alloc((n + 1) * 8).view(np.int64)
    offsets[0] = 0
    np.cumsum(lens, out=offsets[1:])
    total = int(offsets[n])
    data = np.empty(total + 64, dtype=np.uint8) if alloc is None else alloc(total + 64)
    L.avrogen_fill(cfg, r0, n, seed, offsets.ctypes.data, data.ctypes.data, threads)
    return schema, data[:total], offsets
