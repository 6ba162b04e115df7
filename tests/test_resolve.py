"""Schema resolution (rv_schema_resolve / Schema.read_as / `reader_schema=`): data written with one schema decoded into
another schema's Arrow form.  A resolved decode must equal, buffer for buffer, the oracle's decode of the values converted
by the rules (tests/resolution.py) and re-encoded with the reader's schema.  These CPU tests run the product's resolver,
plan and walkers through the host emulation (tests/emu/resolve.py); tests/test_gpu_resolve.py runs them on the device."""
import json
import random

import numpy as np
import pytest

import pyruhvro_b200 as pr
from oracle import pyoracle as po
from tests import emu
from tests import mutation as M
from tests import resolution as RS
from tests.emu import resolve as R
from tests.parity import expected_schema, expected_schema_wide


def rec(*fields, name="R", **kw):
    return json.dumps(dict({"type": "record", "name": name, "fields": list(fields)}, **kw))


def fld(name, t, **kw):
    return dict({"name": name, "type": t}, **kw)


def enum(syms, name="E", **kw):
    return dict({"type": "enum", "name": name, "symbols": syms}, **kw)


def inner(fields, name="In", **kw):
    return dict({"type": "record", "name": name, "fields": fields}, **kw)


TS_MS = {"type": "long", "logicalType": "timestamp-millis"}
DATE = {"type": "int", "logicalType": "date"}
DEC = {"type": "bytes", "logicalType": "decimal", "precision": 9, "scale": 2}
FIX4 = {"type": "fixed", "name": "F", "size": 4}

# (writer, reader, None: accepted | the path the RV_ERR_SCHEMA message must name)
RULES = [
    # records: names, aliases, order, writer-only and reader-only fields
    (rec(fld("a", "int")), rec(fld("a", "int")), None),
    (rec(fld("a", "int"), fld("b", "string")), rec(fld("b", "string"), fld("a", "int")), None),
    (rec(fld("a", "int"), fld("b", "string")), rec(fld("b", "string")), None),
    (rec(fld("a", "int")), rec(fld("x", "int", aliases=["a"])), None),
    (rec(fld("a", "int"), name="Old"), rec(fld("a", "int"), name="New", aliases=["Old"]), None),
    (rec(fld("a", "int"), name="ns.R"), rec(fld("a", "int"), name="other.R"), None),
    (rec(fld("a", "int"), name="Old"), rec(fld("a", "int"), name="New"), ""),
    (rec(fld("a", inner([fld("x", "int"), fld("y", "int")]))), rec(fld("a", inner([fld("y", "int")]))), None),
    (rec(fld("a", inner([fld("x", "int")]))), rec(fld("a", inner([fld("x", "int")], name="Other"))), "a"),
    # reader-only fields: defaults of every supported kind, and the errors
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", "string", default="x")), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", "bytes", default="ÿ\u0000")), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", "boolean", default=True)), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", "long", default=-(2 ** 63))), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", "float", default=0.1)), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", "double", default=1)), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", ["null", "int"], default=None)), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", ["int", "null"], default=4)), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", enum(["P", "Q"]), default="Q")), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", TS_MS, default=5)), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", DATE, default=3)), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", "null", default=None)), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", "string")), "b"),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", "int", default="x")), "b"),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", "int", default=2 ** 31)), "b"),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", ["null", "int"], default=3)), "b"),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", enum(["P"]), default="Z")), "b"),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", inner([fld("x", "int")]), default={"x": 1})), "b"),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", {"type": "array", "items": "int"}, default=[])), "b"),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", {"type": "map", "values": "int"}, default={})), "b"),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", FIX4, default="abcd")), "b"),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", DEC, default="\u0000")), "b"),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", {"type": "string", "logicalType": "uuid"}, default="")), "b"),
    # null defaults of optional fields of every kind: a null of the reader's type
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", ["null", inner([fld("x", "int"), fld("y", ["null", "string"])])], default=None)), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", ["null", {"type": "array", "items": "string"}], default=None)), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", ["null", FIX4], default=None)), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", ["null", DEC], default=None)), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", ["null", {"type": "string", "logicalType": "uuid"}], default=None)), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", ["null", "string", "int"], default=None)), None),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", ["string", "int", "null"], default="x")), "b"),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", ["null", "string", "int"], default="x")), "b"),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", [inner([fld("x", "int")]), "null"], default={"x": 1})), "b"),
    (rec(fld("a", "int")), rec(fld("a", "int"), fld("b", [{"type": "array", "items": "int"}, "null"], default=None)), "b"),
    (rec(fld("a", inner([fld("x", "int")], name="Address"))),
     rec(fld("a", inner([fld("x", "int"), fld("country", "string")], name="Address"))), "a.country"),
    # promotions
    (rec(fld("a", "int")), rec(fld("a", "long")), None),
    (rec(fld("a", "int")), rec(fld("a", "float")), None),
    (rec(fld("a", "int")), rec(fld("a", "double")), None),
    (rec(fld("a", "long")), rec(fld("a", "float")), None),
    (rec(fld("a", "long")), rec(fld("a", "double")), None),
    (rec(fld("a", "float")), rec(fld("a", "double")), None),
    (rec(fld("a", "string")), rec(fld("a", "bytes")), None),
    (rec(fld("a", "bytes")), rec(fld("a", "string")), None),
    (rec(fld("a", "long")), rec(fld("a", "int")), "a"),
    (rec(fld("a", "double")), rec(fld("a", "float")), "a"),
    (rec(fld("a", "int")), rec(fld("a", "string")), "a"),
    (rec(fld("a", "int")), rec(fld("a", DATE)), "a"),
    (rec(fld("a", DATE)), rec(fld("a", "int")), "a"),
    (rec(fld("a", "long")), rec(fld("a", TS_MS)), "a"),
    (rec(fld("a", TS_MS)), rec(fld("a", {"type": "long", "logicalType": "timestamp-micros"})), "a"),
    (rec(fld("a", DATE)), rec(fld("a", DATE)), None),
    (rec(fld("a", DEC)), rec(fld("a", DEC)), None),
    (rec(fld("a", DEC)), rec(fld("a", dict(DEC, scale=3))), "a"),
    (rec(fld("a", FIX4)), rec(fld("a", FIX4)), None),
    (rec(fld("a", FIX4)), rec(fld("a", dict(FIX4, size=5))), "a"),
    (rec(fld("a", FIX4)), rec(fld("a", dict(FIX4, name="G"))), "a"),
    # enums
    (rec(fld("a", enum(["A", "B"]))), rec(fld("a", enum(["B", "A", "C"]))), None),
    (rec(fld("a", enum(["A", "B", "C"]))), rec(fld("a", enum(["A", "B"]))), None),
    (rec(fld("a", enum(["A", "B", "C"]))), rec(fld("a", enum(["A", "B"], default="A"))), None),
    (rec(fld("a", enum(["A"]))), rec(fld("a", enum(["A"], name="Other"))), "a"),
    # arrays / maps
    (rec(fld("a", {"type": "array", "items": "int"})), rec(fld("a", {"type": "array", "items": "double"})), None),
    (rec(fld("a", {"type": "map", "values": inner([fld("x", "int")])})),
     rec(fld("a", {"type": "map", "values": inner([fld("y", "string", default="d"), fld("x", "long")])})), None),
    (rec(fld("a", {"type": "array", "items": "int"})), rec(fld("a", {"type": "map", "values": "int"})), "a"),
    (rec(fld("a", {"type": "array", "items": inner([fld("z", "null")])})),
     rec(fld("a", {"type": "array", "items": inner([fld("z", "null"), fld("s", "string", default="x")])})), "a"),
    # unions
    (rec(fld("a", ["null", "int"])), rec(fld("a", ["long", "null"])), None),
    (rec(fld("a", "int")), rec(fld("a", ["null", "long"])), None),
    (rec(fld("a", inner([fld("x", "int")]))), rec(fld("a", ["null", inner([fld("x", "int")])])), None),
    (rec(fld("a", ["int", "string", "null"])), rec(fld("a", ["long", "bytes", "null"])), None),
    (rec(fld("a", ["null", "int"])), rec(fld("a", "int")), "a"),
    (rec(fld("a", ["int", "string"])), rec(fld("a", ["string", "int"])), "a"),
    (rec(fld("a", ["int", "string"])), rec(fld("a", ["int", "string", "null"])), "a"),
    (rec(fld("a", ["null", "int", "string"])), rec(fld("a", ["null", "int"])), "a"),
    (rec(fld("a", "null")), rec(fld("a", ["null", "int"])), "a"),
]


@pytest.mark.parametrize("i", range(len(RULES)))
def test_rule_table(i):
    w, r, path = RULES[i]
    if path is None:
        s = pr.Schema(w).read_as(r)
        assert s.arrow_schema.equals(pr.Schema(r).arrow_schema, check_metadata=True)
        assert s.walker_source
    else:
        with pytest.raises(ValueError, match="schema resolution") as ei:
            pr.Schema(w).read_as(r)
        if path:
            assert f"field '{path}'" in str(ei.value), str(ei.value)


def test_name_before_alias(coracle):
    """A reader field binds to the writer field of its own name even when one of its aliases names an earlier field."""
    wj = rec(fld("old_x", "int"), fld("x", "int"), fld("y", "int"))
    rj = rec(fld("x", "long", aliases=["old_x"]), fld("z", "int", aliases=["nope", "y", "old_x"]))
    vals = [{"old_x": i, "x": 100 + i, "y": 200 + i} for i in range(300)]
    ws = po.parse_schema(wj)
    data, off = po.pack_records([po.encode_datum(ws, v) for v in vals])
    for walker in ("interp", "gen"):
        got = R.decode(wj, rj, data, off, len(vals), 2, walker=walker)
        assert [r for b in got for r in b.to_pylist()] == [{"x": 100 + i, "z": 200 + i} for i in range(300)]
    _check(coracle, wj, rj, 300, 2, ["interp"], random.Random(1))


def test_null_defaults_of_every_kind(coracle):
    """Optional reader-only fields of every kind with a null default: buffer for buffer a null of the reader's type."""
    base = [fld("a", "int"), fld("xs", {"type": "array", "items": inner([fld("q", "string")], name="It")})]
    added = [fld("r", ["null", inner([fld("x", "int"), fld("y", ["null", "string"]), fld("z", {"type": "array", "items": "long"})], name="NR")], default=None),
             fld("l", ["null", {"type": "array", "items": "string"}], default=None),
             fld("u", ["null", "string", "int"], default=None)]
    inner_added = [fld("n", ["null", inner([fld("k", "boolean")], name="NK")], default=None), fld("q", "string")]
    wj = rec(*base)
    rj = rec(*added[:2], fld("xs", {"type": "array", "items": inner(inner_added, name="It")}), fld("a", "long"), added[2])
    rng = random.Random(3)
    for n, k in ((1, 1), (257, 3), (600, 3)):
        _check(coracle, wj, rj, n, k, ["interp", "gen", "warp"], rng)
    # the wider subset: fixed, decimal, uuid
    wide_added = [fld("f", ["null", FIX4], default=None), fld("d", ["null", DEC], default=None),
                  fld("g", ["null", {"type": "string", "logicalType": "uuid"}], default=None)]
    rjw = rec(fld("a", "int"), *wide_added, base[1])
    _check(coracle, wj, rjw, 300, 3, ["interp", "gen"], rng, wide=True)


def test_rule_table_is_large_enough():
    assert len(RULES) >= 40
    assert sum(p is not None for _, _, p in RULES) >= 15


def test_resolved_handles_are_refused_where_they_do_not_belong():
    import workloads
    s = pr.Schema(workloads.KAFKA_SCHEMA).read_as(RS.kafka_v2())
    with pytest.raises(ValueError, match="full schemas"):
        s.read_as(RS.kafka_v2())
    with pytest.raises(ValueError, match="full schemas"):
        pr.Schema(workloads.KAFKA_SCHEMA).read_as(pr.Schema(workloads.KAFKA_SCHEMA).project(["name"]))
    # the same documents parse as before: a default is only checked when a resolution uses it
    pr.Schema(rec(fld("a", "int", default="not an int")))
    assert pr.Schema(workloads.KAFKA_SCHEMA).read_as(RS.kafka_v2()).project(["source", "age"]).arrow_schema.names == ["source", "age"]


# ---- identity: a schema read as itself is the plain plan --------------------------------------------------------------
def test_identity_walker_source():
    import workloads
    for sj in (workloads.KAFKA_SCHEMA, workloads.FLAT_SCHEMA, workloads.WIDE_SCHEMA):
        assert pr.Schema(sj).read_as(sj).walker_source == pr.Schema(sj).walker_source
    for wide in (False, True):
        rng = random.Random(77 + wide)
        for _ in range(400):
            sj = po.random_schema_json(rng, wide=wide)
            s = pr.Schema(sj)
            if not s.is_supported:
                continue
            assert s.read_as(sj).walker_source == s.walker_source, sj


# ---- emulated parity with the oracle ---------------------------------------------------------------------------------
def _values(sj, n, rng, wide):
    s = po.parse_schema(sj, wide=wide)
    return [po.random_value(s, rng) for _ in range(n)], s


def _check(coracle, wj, rj, n, k, walkers, rng, wide=False, columns=None):
    vals, ws = _values(wj, n, rng, wide)
    recs = [po.encode_datum(ws, v) for v in vals]
    data, off = po.pack_records(recs)
    want = RS.expected_batches(coracle, wj, rj, vals, k, wide=wide)
    exp = expected_schema_wide(rj) if wide else expected_schema(rj)
    for walker in walkers:
        if isinstance(want, tuple):
            with pytest.raises(emu.EmuError) as ei:
                R.decode(wj, rj, data, off, n, k, columns=columns, walker=walker)
            assert (ei.value.code, ei.value.record) == (6, want[1]), (walker, ei.value)
            continue
        got = R.decode(wj, rj, data, off, n, k, columns=columns, walker=walker)
        assert len(got) == len(want)
        for i, (b, w) in enumerate(zip(got, want)):
            assert b.schema.equals(exp, check_metadata=True), (walker, b.schema, exp)
            b.validate(full=not wide)   # (bytes read as string are not checked for UTF-8, as in any decode)
            d = po.canon_diff(po.canon_from_batch(b), w, f"{walker} batch[{i}]")
            assert d is None, (d, wj, rj)


# Every evolution goes through the interpreter; every sixth (fifth, wide) also through the generated walker, per lane and
# in lock-step warps (each of those compiles a host library of its own).
@pytest.mark.parametrize("seed", range(60))
def test_emulated_parity_narrow(coracle, seed):
    rng = random.Random(seed * 31 + 1)
    wj = po.random_schema_json(rng)
    rj = RS.random_evolution(rng, wj, unmapped_ok=seed % 5 == 0)
    n = [1, 255, 256, 257, 600][seed % 5]
    _check(coracle, wj, rj, n, [1, 3][seed % 2], ["interp", "gen", "warp"] if seed % 6 == 0 else ["interp"], rng)


@pytest.mark.parametrize("seed", range(30))
def test_emulated_parity_wide(coracle, seed):
    rng = random.Random(seed * 37 + 2)
    wj = po.random_schema_json(rng, wide=True)
    rj = RS.random_evolution(rng, wj, wide=True)
    n = [1, 255, 256, 257, 600][seed % 5]
    _check(coracle, wj, rj, n, [3, 1][seed % 2], ["interp", "gen", "warp"] if seed % 5 == 0 else ["interp"], rng, wide=True)


def test_kafka_v2_values(coracle):
    import workloads
    W = workloads.KAFKA_SCHEMA
    rng = random.Random(5)
    for rj in (RS.kafka_v2(), RS.kafka_v2(("A", "B"), "A")):
        _check(coracle, W, rj, 600, 3, ["interp", "gen", "warp"], rng)
    ws = po.parse_schema(W)
    vals = [po.random_value(ws, rng) for _ in range(300)]
    data, off = po.pack_records([po.encode_datum(ws, v) for v in vals])
    plain = emu.decode(W, data, off, 300, 1)[0].to_pylist()
    for rj, classes in ((RS.kafka_v2(), None), (RS.kafka_v2(("A", "B"), "A"), {"A": "A", "B": "B", "C": "A"})):
        got = R.decode(W, rj, data, off, 300, 1, walker="gen")[0]
        assert got.schema.names[0] == "created_at" and got.schema.names[-3:] == ["country", "score", "source"]
        for p, g in zip(plain, got.to_pylist()):
            assert g["created_at"] == p["created_at"] and g["name"] == p["name"] and g["age"] == p["age"]
            assert "phone_numbers" not in g
            assert (g["country"], g["score"], g["source"]) == (None, 0.0, "kafka")
            assert g["class"] == (classes[p["class"]] if classes else p["class"])
            if p["address"] is None:
                assert g["address"] is None
            else:
                assert g["address"] == {"city": p["address"]["city"], "street": p["address"]["street"], "country": "US"}
    # the projection names reader fields
    got = R.decode(W, RS.kafka_v2(), data, off, 300, 2, columns=["source", "age"], walker="warp")
    assert got[0].schema.names == ["source", "age"]
    assert [r["age"] for b in got for r in b.to_pylist()] == [p["age"] for p in plain]


def test_promotions_round_once(coracle):
    """long -> float / double with one rounding step: values just above a float's halfway point."""
    wj = rec(fld("a", "long"), fld("b", "long"), fld("c", "int"))
    rj = rec(fld("a", "float"), fld("b", "double"), fld("c", "float"))
    vals = [{"a": v, "b": v, "c": c} for v, c in [((1 << 60) + (1 << 36) + 1, 16777217), (2 ** 63 - 1, -(2 ** 31)), (-(2 ** 63), 2 ** 31 - 1),
                                                     ((1 << 53) + 1, 16777219), (0, 0)]]
    ws = po.parse_schema(wj)
    data, off = po.pack_records([po.encode_datum(ws, v) for v in vals])
    got = R.decode(wj, rj, data, off, len(vals), 1, walker="gen")[0].to_pydict()
    assert got["a"] == [float(np.array([v["a"]]).astype(np.float32)[0]) for v in vals]
    assert got["b"] == [float(np.array([v["b"]]).astype(np.float64)[0]) for v in vals]
    assert got["c"] == [float(np.array([v["c"]]).astype(np.float32)[0]) for v in vals]


# ---- damaged inputs: the writer-schema decode's verdict --------------------------------------------------------------
def _verdict(fn):
    try:
        fn()
        return None
    except emu.EmuError as e:
        return (e.code, e.record)


@pytest.mark.parametrize("seed", range(200))
def test_damaged_inputs_match_writer_decode(seed):
    rng = random.Random(seed * 13 + 7)
    wj = po.random_schema_json(rng)
    rj = RS.random_evolution(rng, wj)
    ws = po.parse_schema(wj)
    recs = M.damage(rng, [po.encode_datum(ws, po.random_value(ws, rng)) for _ in range(rng.choice([3, 40, 257]))])
    data, off = po.pack_records(recs)
    n, k = len(recs), rng.choice([1, 2, 3])
    want = _verdict(lambda: emu.decode(wj, data, off, n, k))
    walker = ["gen", "warp"][seed // 10 % 2] if seed % 10 == 0 else "interp"
    got = _verdict(lambda: R.decode(wj, rj, data, off, n, k, walker=walker))
    if want is not None and want[0] == 8:   # RV_ERR_OVERFLOW: only produced columns overflow
        return
    assert got == want, (wj, rj)
