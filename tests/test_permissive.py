"""Permissive decodes (rv_schema_permissive / errors="null"): a damaged record becomes a null row and is reported, the
rest of the call decodes.  These CPU tests run the product's permissive plan and the kernel's per-lane protocol through
the host emulation (tests/emu/permissive.py) with the interpreter, the generated walker per lane and the generated walker
in lock-step warps, against the C oracle (tests/permissive_cases.py states the contract).  tests/test_gpu_permissive.py
runs the same cases on the device."""
import json
import random

import pyarrow as pa
import pytest

import pyruhvro_b200 as pr
from oracle import pyoracle as po
from tests import emu
from tests import mutation as M
from tests import permissive_cases as PC
from tests.emu import permissive as EP
from tests.emu import resolve as R
from tests.parity import gen_case

WALKERS = ["interp", "gen", "warp"]


def rec(*fields, name="R"):
    return json.dumps({"type": "record", "name": name, "fields": list(fields)})


def fld(name, t, **kw):
    return dict({"name": name, "type": t}, **kw)


ITEM = {"type": "record", "name": "It", "fields": [fld("x", "int"), fld("s", "string")]}
# a flat column, a nullable one, a string, an item-parallel list of records, a map, an N-variant union and an enum
PLACE_SCHEMA = rec(fld("a", "long"), fld("b", ["null", "string"]), fld("c", "string"), fld("l", {"type": "array", "items": ITEM}),
                   fld("m", {"type": "map", "values": "int"}), fld("u", ["int", "string", "null"]),
                   fld("e", {"type": "enum", "name": "E", "symbols": ["A", "B", "C"]}))


def place_records(n, bad, items=2):
    """n records of PLACE_SCHEMA with `items` list items each; the ones in `bad` truncated to one byte (EOF)."""
    s = po.parse_schema(PLACE_SCHEMA)
    out = []
    for i in range(n):
        v = {"a": i, "b": (0, None) if i % 3 == 0 else (1, f"b{i}"), "c": "c" * (i % 7), "l": [{"x": j, "s": "s"} for j in range(items)],
             "m": [("k", i)], "u": [(0, i), (1, "u"), (2, None)][i % 3], "e": i % 3}
        r = po.encode_datum(s, v)
        out.append(r[:1] if i in bad else r)
    return out


def run(coracle, sj, recs, k, walker, wide=False, columns=None, **kw):
    exp = PC.Expected(coracle, sj, recs, k, wide=wide)
    data, off = po.pack_records(recs)
    batches, bad = EP.decode(sj, data, off, len(recs), k, walker=walker, columns=columns, **kw)
    exp.check(batches, [(r, 6 if c == 13 else c) for r, c in bad], columns=columns)
    return exp, batches


@pytest.mark.parametrize("walker", WALKERS)
@pytest.mark.parametrize("seed", range(12))
def test_damaged_random(coracle, walker, seed):
    sj, recs, k = M.damaged_case(seed)
    run(coracle, sj, recs, k, walker)


@pytest.mark.parametrize("walker", WALKERS)
@pytest.mark.parametrize("seed", range(8))
def test_forged_varints(coracle, walker, seed):
    sj, recs, k = M.forged_case(seed)
    run(coracle, sj, recs, k, walker)


@pytest.mark.parametrize("seed", range(6))
def test_damaged_wide(seed):
    sj, recs, k = M.damaged_case_wide(seed)
    run(None, sj, recs, k, "interp", wide=True)


def test_clean_input_equals_read_as(coracle):
    """No bad record: the batches are Schema(R).read_as(R') of the same input, and the report is empty."""
    for seed in range(4):
        sj, recs, data, off = gen_case(seed, n=300)
        batches, bad = EP.decode(sj, data, off, len(recs), 3)
        assert bad == []
        want = R.decode(sj, PC.optional_json(sj), data, off, len(recs), 3)
        for b, w in zip(batches, want):
            assert po.canon_diff(po.canon_from_batch(b), po.canon_from_batch(w)) is None


PLACEMENTS = {
    "lanes": [0, 31, 32, 255, 256, 383, 384],
    "warp": list(range(64, 96)),
    "tile": list(range(512, 768)),
}


@pytest.mark.parametrize("walker", WALKERS)
@pytest.mark.parametrize("where", sorted(PLACEMENTS))
def test_placements(coracle, walker, where):
    bad = set(PLACEMENTS[where])
    recs = place_records(1000, bad)
    exp, _ = run(coracle, PLACE_SCHEMA, recs, 1, walker)
    assert [i for i, _ in exp.bad] == sorted(bad)   # the placements are reached: exactly these records are bad
    assert all(s == 1 for _, s in exp.bad)


@pytest.mark.parametrize("walker", WALKERS)
def test_chunk_entirely_bad(coracle, walker):
    n, k = 900, 3
    recs = place_records(n, set(range(300, 600)))
    exp, batches = run(coracle, PLACE_SCHEMA, recs, k, walker)
    assert [i for i, _ in exp.bad] == list(range(300, 600))
    b = batches[1]   # every column but the map (empty maps) and the union (type id 0) is null throughout
    assert b.num_rows == 300 and all(b.column(j).null_count == 300 for j in range(b.num_columns) if b.schema.names[j] not in ("m", "u"))
    assert b.column(b.schema.names.index("m")).offsets.to_pylist() == [0] * 301


@pytest.mark.parametrize("walker", ["gen", "warp"])
def test_bad_beside_item_parallel_warps(coracle, walker):
    """Warp 1 of the tile has a bad record; warps 0 and 2-7 hold lists of at most kItemSlots items, which the generated
    walker's FAST emit hands out item-parallel."""
    recs = place_records(256, {40}, items=3)
    exp, _ = run(coracle, PLACE_SCHEMA, recs, 1, walker)
    assert [i for i, _ in exp.bad] == [40]


def test_forged_varint_fast_accepts_precise_refuses(coracle):
    """A record whose bytes the FAST count only flags as not plain (a varint of more than ten bytes), which the
    precise walk then refuses: it is a bad row."""
    sj = rec(fld("a", "long"), fld("s", "string"))
    s = po.parse_schema(sj)
    recs = [po.encode_datum(s, {"a": i, "s": "x"}) for i in range(64)]
    recs[33] = b"\xff" * 10 + b"\x01" + recs[33][1:]   # an 11-byte varint
    assert PC.verdict(coracle, sj, recs[33]) == "varint"
    for walker in WALKERS:
        exp, _ = run(coracle, sj, recs, 1, walker)
        assert exp.bad == [(33, 2)]


@pytest.mark.parametrize("walker", WALKERS)
def test_projection_unselected_field_broken(coracle, walker):
    """Only an unselected field is broken: the record is still bad (the skipped field is validated as in a strict call)."""
    sj = rec(fld("a", "int"), fld("b", "string"), fld("c", "boolean"))
    s = po.parse_schema(sj)
    recs = [po.encode_datum(s, {"a": i, "b": "x" * (i % 5), "c": True}) for i in range(300)]
    for i in (3, 100, 299):
        recs[i] = recs[i][:-1] + b"\x07"   # not a boolean byte
    exp = PC.Expected(coracle, sj, recs, 2)
    data, off = po.pack_records(recs)
    batches, bad = EP.decode(sj, data, off, len(recs), 2, walker=walker, columns=["b", "a"])
    exp.check(batches, bad, columns=["b", "a"])
    assert bad == [(3, 3), (100, 3), (299, 3)]


@pytest.mark.parametrize("walker", WALKERS)
def test_resolved_unmapped_enum(walker):
    writer = rec(fld("a", "int"), fld("e", {"type": "enum", "name": "E", "symbols": ["A", "B", "C"]}))
    reader = rec(fld("e", {"type": "enum", "name": "E", "symbols": ["B", "A"]}), fld("a", "long"), fld("d", "string", default="z"))
    ws = po.parse_schema(writer)
    vals = [{"a": i, "e": i % 3} for i in range(260)]
    recs = [po.encode_datum(ws, v) for v in vals]
    data, off = po.pack_records(recs)
    batches, bad = EP.decode(writer, data, off, len(recs), 1, reader_json=reader, walker=walker)
    assert bad == [(i, 13) for i in range(260) if i % 3 == 2]
    (b,) = batches
    assert b.schema.field("e").nullable and b.schema.field("a").nullable and b.schema.field("d").nullable
    got = b.to_pydict()
    assert got["a"] == [None if i % 3 == 2 else i for i in range(260)]
    assert got["e"] == [None if i % 3 == 2 else "AB"[i % 3] for i in range(260)]
    assert got["d"] == [None if i % 3 == 2 else "z" for i in range(260)]


def _framed(recs, header):
    return [header + r for r in recs]


@pytest.mark.parametrize("walker", WALKERS)
def test_confluent_framing_errors(coracle, walker):
    sj = PLACE_SCHEMA
    plain = place_records(300, set())
    msgs = _framed(plain, b"\x00\x00\x00\x00\x07")
    msgs[5] = b"\x01" + msgs[5][1:]           # wrong magic byte
    msgs[256] = b"\x00\x00"                   # shorter than its header
    msgs[257] = b""                           # empty message
    msgs[290] = b"\x00\x00\x00\x00\x08" + plain[290]   # another schema id
    data, off = po.pack_records(msgs)
    batches, bad = EP.decode(sj, data, off, len(msgs), 3, walker=walker, frame=(5, 2, 7))
    assert bad == [(5, 12), (256, 12), (257, 12), (290, 12)]
    verdicts = [None] * len(plain)
    for i, _ in bad:
        verdicts[i] = "frame"
    PC.Expected(coracle, sj, plain, 3, verdicts=verdicts).check(batches, bad)


@pytest.mark.parametrize("walker", WALKERS)
def test_single_object_framing_errors(coracle, walker):
    sj = PLACE_SCHEMA
    fp = pr.Schema(sj).fingerprint
    plain = place_records(100, set())
    hdr = b"\xc3\x01" + fp.to_bytes(8, "little")
    msgs = _framed(plain, hdr)
    msgs[0] = b"\xc3\x01" + (fp ^ 1).to_bytes(8, "little") + plain[0]   # another writer
    msgs[31] = hdr[:9]
    msgs[32] = b"\xc3\x00" + hdr[2:] + plain[32]
    msgs[99] = hdr + plain[99][:1]   # the datum itself is truncated
    data, off = po.pack_records(msgs)
    batches, bad = EP.decode(sj, data, off, len(msgs), 1, walker=walker, frame=(10, EP.SINGLE_OBJECT, 0), fingerprint=fp)
    assert bad == [(0, 12), (31, 12), (32, 12), (99, 1)]
    verdicts = [None] * len(plain)
    for i, c in bad:
        verdicts[i] = "frame" if c == 12 else "eof"
    PC.Expected(coracle, sj, plain, 1, verdicts=verdicts).check(batches, bad)


def test_overflow_stays_fatal():
    """Two lists of 2^30 + 1 zero-width items overflow the batch's i32 offsets: RV_ERR_OVERFLOW, as in a strict call."""
    sj = rec(fld("l", {"type": "array", "items": "null"}))
    big = po.zigzag_bytes(2 ** 30 + 1) + b"\x00"
    recs = [big, b"", big]
    data, off = po.pack_records(recs)
    with pytest.raises(emu.EmuError) as e:
        EP.decode(sj, data, off, len(recs), 1)
    assert e.value.code == 8


# ---- the interface (no device needed) ---------------------------------------------------------------------------------
def test_errors_argument_is_checked():
    sj = rec(fld("a", "int"))
    for call in (lambda: pr.deserialize_array([b"\x02"], sj, errors="nope"),
                 lambda: pr.deserialize_array_threaded([b"\x02"], sj, 1, errors="nope"),
                 lambda: pr.deserialize_array_threaded_spawn([b"\x02"], sj, 1, errors="nope"),
                 lambda: pr.deserialize_arrow_array(pa.array([b"\x02"], pa.binary()), sj, errors="nope"),
                 lambda: pr.decode_packed(b"\x02", [0, 1], 1, sj, errors="nope"),
                 lambda: pr.deserialize_confluent([b"\x02"], sj, errors="nope"),
                 lambda: pr.deserialize_single_object([b"\x02"], sj, errors=None)):
        with pytest.raises(ValueError, match="errors"):
            call()


def test_permissive_schema():
    sj = rec(fld("a", "int"), fld("b", ["null", "string"]), fld("n", "null"), fld("u", ["int", "string", "boolean"]),
             fld("r", {"type": "record", "name": "In", "fields": [fld("x", "int")]}))
    p = pr.Schema(sj).permissive()
    s = p.arrow_schema
    assert [f.nullable for f in s] == [True, True, False, False, True]   # null and union fields stay as they are
    assert s.field("u").type == pr.Schema(sj).arrow_schema.field("u").type
    assert p.fingerprint == pr.Schema(sj).fingerprint and p.canonical_form == pr.Schema(sj).canonical_form
    assert "c.in_range && c.err == 0" in p.walker_source
    assert "c.in_range && c.err == 0" not in pr.Schema(sj).walker_source
    with pytest.raises(ValueError, match="already permissive"):
        p.permissive()
    q = pr.Schema(sj).project(["r", "a"]).permissive()
    assert q.arrow_schema.names == ["r", "a"] and all(f.nullable for f in q.arrow_schema)
    assert "c.in_range && c.err == 0" in p.project(["a"]).walker_source   # a projection of a permissive handle stays permissive


def test_permissive_handles_are_refused():
    sj = rec(fld("a", "int"))
    p = pr.Schema(sj).permissive()
    v = ctypes_versions_create(pr.Schema(sj), p)
    assert v[0] == 9 and "permissive" in v[1]
    v = ctypes_versions_create(p, pr.Schema(sj))
    assert v[0] == 9 and "permissive" in v[1]
    import ctypes
    c_arr, c_sch = pr._ArrowArray(), pr._ArrowSchema()
    pa.record_batch([pa.array([1], pa.int32())], names=["a"])._export_to_c(ctypes.addressof(c_arr), ctypes.addressof(c_sch))
    h = ctypes.c_void_p()
    assert pr.lib.rv_encode_host(p.handle, ctypes.addressof(c_arr), ctypes.addressof(c_sch), 1, ctypes.byref(h)) == 9
    assert "permissive" in pr._last_error()


def ctypes_versions_create(reader, writer):
    import ctypes
    h = ctypes.c_void_p()
    ids = (ctypes.c_int64 * 1)(1)
    ws = (ctypes.c_void_p * 1)(writer.handle)
    st = pr.lib.rv_versions_create(reader.handle, ids, ws, 1, None, 0, ctypes.byref(h))
    return st, pr._last_error()


def test_cache_key_has_the_mode():
    sj = rec(fld("a", "int"))
    assert pr._get_or_parse_schema(sj) is not pr._get_or_parse_schema(sj, permissive=True)
    assert pr._get_or_parse_schema(sj, permissive=True) is pr._get_or_parse_schema(sj, None, None, True)


def test_strict_walker_sources_are_unchanged():
    """A strict handle generates the same walker source as before permissive decoding existed: the reference schemas and
    the bench schemas, against hashes recorded from the code before the change (tests/golden/strict_walker_sources.json)."""
    import hashlib
    import os
    with open(os.path.join(os.path.dirname(__file__), "golden", "strict_walker_sources.json")) as f:
        golden = json.load(f)
    assert len(golden) == 37
    for g in golden:
        assert hashlib.sha256(pr.Schema(g["schema"]).walker_source.encode()).hexdigest() == g["walker_sha256"], g["schema"][:80]
