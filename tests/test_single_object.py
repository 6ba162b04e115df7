"""Avro single-object encoding without a GPU: the Parsing Canonical Form and CRC-64-AVRO fingerprint of a schema
(Schema.canonical_form / Schema.fingerprint) against the restatement of the specification in tests/single_object.py, the
registry errors of rv_versions_create_single_object (all raised before any CUDA call), and the partition's 64-bit header
check through the host emulation (tests/emu/single_object.py).  tests/test_gpu_single_object.py runs the decodes and the
encode on the device."""
import ctypes
import json
import random

import pytest

import pyruhvro_b200 as pr
import workloads
from oracle import pyoracle as po
from tests import emu
from tests import resolution as RS
from tests import single_object as SO
from tests.emu import single_object as E


def _same(sj: str):
    s = pr.Schema(sj)
    want = SO.canonical_form(sj)
    assert s.canonical_form == want, (sj, s.canonical_form, want)
    assert s.fingerprint == SO.fingerprint(sj)


def test_known_answers():
    assert SO.fingerprint('"null"') == 0x63DD24E7CC258F8A == 7195948357588979594
    assert SO.fingerprint('"int"') == 0x7275D51A3F395C8F
    assert pr.Schema('"null"').fingerprint == 0x63DD24E7CC258F8A
    assert pr.Schema('"int"').fingerprint == 0x7275D51A3F395C8F
    assert pr.Schema('{"type": "int"}').canonical_form == '"int"'


# one per rule of the canonical form
RULE_CASES = {
    "primitives": ['"string"', '{"type": "long"}', '["null", {"type": "double"}, "boolean", "bytes", "float"]'],
    "fullnames": ['{"type": "record", "name": "R", "namespace": "a.b", "fields": [{"name": "x", "type": "int"}]}',
                  '{"type": "record", "name": "a.b.R", "namespace": "ignored", "fields": [{"name": "e", "type": {"type": "enum", "name": "E", "symbols": ["X"]}}]}',
                  '{"type": "record", "name": "R", "namespace": "n", "fields": [{"name": "f", "type": {"type": "fixed", "name": "F", "namespace": "", "size": 3}}]}'],
    "strip": ['{"type": "record", "name": "R", "doc": "d", "aliases": ["Q"], "fields": [{"name": "x", "type": "int", "doc": "f", "default": 3, "aliases": ["y"], "order": "descending"}]}',
              '{"type": "enum", "name": "E", "symbols": ["A", "B"], "default": "A", "doc": "x"}'],
    "logical": ['{"type": "record", "name": "R", "fields": ['
                '{"name": "d", "type": {"type": "int", "logicalType": "date"}},'
                '{"name": "tm", "type": {"type": "int", "logicalType": "time-millis"}},'
                '{"name": "tu", "type": {"type": "long", "logicalType": "time-micros"}},'
                '{"name": "ts", "type": {"type": "long", "logicalType": "timestamp-millis"}},'
                '{"name": "tsu", "type": {"type": "long", "logicalType": "timestamp-micros"}},'
                '{"name": "u", "type": {"type": "string", "logicalType": "uuid"}},'
                '{"name": "db", "type": {"type": "bytes", "logicalType": "decimal", "precision": 9, "scale": 2}},'
                '{"name": "df", "type": {"type": "fixed", "name": "D", "size": 8, "logicalType": "decimal", "precision": 10}}]}'],
    "order": ['{"fields": [{"type": "int", "name": "x"}], "name": "R", "type": "record"}',
              '{"size": 4, "name": "F", "type": "fixed"}', '{"values": "int", "type": "map"}', '{"items": "int", "type": "array"}'],
    "named_once": ['{"type": "record", "name": "R", "namespace": "n", "fields": ['
                   '{"name": "a", "type": {"type": "record", "name": "In", "fields": [{"name": "v", "type": "int"}]}},'
                   '{"name": "b", "type": "In"}, {"name": "c", "type": ["null", "n.In"]},'
                   '{"name": "e", "type": {"type": "enum", "name": "E", "symbols": ["P", "Q"]}}, {"name": "e2", "type": {"type": "array", "items": "E"}}]}'],
    "whitespace": ['{ "type" : "record" , "name" : "R" ,\n "fields" : [ { "name" : "x" , "type" : [ "null" , "int" ] } ] }'],
}


@pytest.mark.parametrize("rule", sorted(RULE_CASES))
def test_canonical_form_rules(rule):
    for sj in RULE_CASES[rule]:
        _same(sj)


def test_canonical_form_of_reference_schemas():
    with open(po.__file__.replace("oracle/pyoracle.py", "tests/golden/reference_schemas.json")) as f:
        schemas = json.load(f)
    assert len(schemas) >= 20
    for sj in schemas:
        _same(sj if isinstance(sj, str) else json.dumps(sj))


@pytest.mark.parametrize("wide", [False, True], ids=["narrow", "wide"])
def test_canonical_form_of_random_schemas(wide):
    rng = random.Random(2024 + wide)
    for _ in range(200):
        _same(po.random_schema_json(rng, wide=wide))


def test_canonical_form_is_idempotent():
    rng = random.Random(7)
    # (not a name in the null namespace inside a namespaced type: the form writes it bare, and a bare name there reads
    # as one of the enclosing namespace — the specification's form cannot say otherwise)
    cases = [sj for v in RULE_CASES.values() for sj in v if '"namespace": ""' not in sj]
    cases += [po.random_schema_json(rng, wide=True) for _ in range(50)]
    for sj in cases:
        c = pr.Schema(sj).canonical_form
        assert pr.Schema(c).canonical_form == c
        assert pr.Schema(c).fingerprint == pr.Schema(sj).fingerprint


BASE = {"type": "record", "name": "R", "namespace": "ns", "fields": [
    {"name": "a", "type": "int"}, {"name": "b", "type": {"type": "enum", "name": "E", "symbols": ["X", "Y"]}},
    {"name": "c", "type": {"type": "fixed", "name": "F", "size": 4}}, {"name": "d", "type": "long"}]}


def _fp(doc) -> int:
    return pr.Schema(doc if isinstance(doc, str) else json.dumps(doc)).fingerprint


def test_equal_canonical_form_equal_fingerprint():
    import copy
    same = []
    d = copy.deepcopy(BASE); d["doc"] = "docs"; d["fields"][0]["doc"] = "x"; same.append(d)
    d = copy.deepcopy(BASE); d["aliases"] = ["Old"]; d["fields"][1]["aliases"] = ["bee"]; same.append(d)
    d = copy.deepcopy(BASE); d["fields"][0]["default"] = 5; d["fields"][1]["type"]["default"] = "Y"; same.append(d)
    d = copy.deepcopy(BASE); d["fields"][3]["type"] = {"type": "long", "logicalType": "timestamp-micros"}; same.append(d)
    same.append(json.dumps(BASE, indent=3))                                           # whitespace
    same.append(json.dumps(dict(reversed(list(BASE.items())))))                       # key order
    d = copy.deepcopy(BASE); del d["namespace"]; d["name"] = "ns.R"; same.append(d)   # a dotted name instead of "namespace"
    want = _fp(BASE)
    for doc in same:
        assert _fp(doc) == want, doc


def test_different_canonical_form_different_fingerprint():
    import copy
    diff = []
    d = copy.deepcopy(BASE); d["fields"][0], d["fields"][3] = d["fields"][3], d["fields"][0]; diff.append(d)   # field order
    d = copy.deepcopy(BASE); d["fields"][1]["type"]["symbols"] = ["X", "Z"]; diff.append(d)                   # an enum symbol
    d = copy.deepcopy(BASE); d["fields"][2]["type"]["size"] = 5; diff.append(d)                               # a fixed size
    d = copy.deepcopy(BASE); d["name"] = "S"; diff.append(d)                                                  # a record name
    fps = {_fp(BASE)} | {_fp(doc) for doc in diff}
    assert len(fps) == len(diff) + 1


def test_projected_and_resolved_handles_name_the_writer():
    v1, v2 = workloads.KAFKA_SCHEMA, workloads.kafka_v2_schema()
    w = pr.Schema(v1)
    names = [f.name for f in w.arrow_schema][:2]
    for h in (w.project(names), w.read_as(v2), w.read_as(v2).project([f.name for f in pr.Schema(v2).arrow_schema][:1])):
        assert h.canonical_form == w.canonical_form == SO.canonical_form(v1)
        assert h.fingerprint == w.fingerprint


def test_schema_without_canonical_form_is_refused():
    sj = json.dumps({"type": "record", "name": "R", "fields": [{"name": "d", "type": {"type": "fixed", "name": "D", "size": 12, "logicalType": "duration"}}]})
    with pytest.raises(ValueError, match="Canonical Form"):
        pr.Schema(sj).fingerprint


# ---- registry errors: raised before any CUDA call (this machine may have none) ------------------------------------------
def test_registry_errors():
    v1 = workloads.KAFKA_SCHEMA
    doc = json.loads(v1)
    doc["doc"] = "the same schema with a doc"
    with pytest.raises(ValueError, match="same fingerprint"):
        pr.Versions([v1, json.dumps(doc)], v1, single_object=True)
    many = []
    for i in range(257):
        many.append(json.dumps({"type": "record", "name": f"R{i}", "fields": [{"name": "a", "type": "int"}]}))
    with pytest.raises(ValueError, match="more than 256"):
        pr.Versions(many, many[0], single_object=True)
    with pytest.raises(ValueError, match="no writer"):
        pr.Versions([], v1, single_object=True)
    w = pr.Schema(v1)
    reader = pr.Schema(v1)
    out = ctypes.c_void_p()
    for bad in (w.project([f.name for f in w.arrow_schema][:1]), w.read_as(v1)):
        hs = (ctypes.c_void_p * 1)(bad.handle)
        assert pr.lib.rv_versions_create_single_object(reader.handle, hs, 1, None, 0, ctypes.byref(out)) == 9   # RV_ERR_INVALID
        assert "full schema" in pr._last_error()
        hs = (ctypes.c_void_p * 1)(w.handle)
        assert pr.lib.rv_versions_create_single_object(bad.handle, hs, 1, None, 0, ctypes.byref(out)) == 9
    with pytest.raises(TypeError):
        pr.deserialize_single_object_versions([], {1: v1}, v1)


# ---- the partition's header check, emulated -------------------------------------------------------------------------
def _writers():
    rj = RS.kafka_v2()
    return rj, [workloads.KAFKA_SCHEMA, rj]


def _messages(rng, n, sel):
    """n single-object messages of the two Kafka writers (writer sel(i) for message i) -> (recs, fps)"""
    _, ws = _writers()
    parsed = [po.parse_schema(sj) for sj in ws]
    fps = [SO.fingerprint(sj) for sj in ws]
    recs = []
    for i in range(n):
        w = sel(i)
        recs.append(SO.frame(fps[w], po.encode_datum(parsed[w], po.random_value(parsed[w], rng))))
    return recs, fps


@pytest.mark.parametrize("mix", ["alternate", "runs", "one"])
def test_partition_groups_every_message_by_its_writer(mix):
    rng = random.Random(len(mix))
    sel = {"alternate": lambda i: i % 2, "runs": lambda i: (i // 300) % 2, "one": lambda i: 1}[mix]
    n = 1000
    recs, fps = _messages(rng, n, sel)
    data, off = po.pack_records(recs)
    order = sorted(range(2), key=lambda w: fps[w])
    got = E.partition(data, off, n, 3, fps)
    assert [order[g] for g in got] == [sel(i) for i in range(n)]


def test_partition_header_errors():
    rng = random.Random(9)
    n = 700
    recs, fps = _messages(rng, n, lambda i: i % 2)
    other = SO.fingerprint(json.dumps({"type": "record", "name": "X", "fields": [{"name": "a", "type": "int"}]}))
    for at, bad, code in (
            (5, SO.frame(other, recs[5][10:]), 14),                         # unregistered fingerprint
            (6, b"\xc2" + recs[6][1:], 12),                                 # wrong C3
            (7, recs[7][:1] + b"\x02" + recs[7][2:], 12),                   # wrong 01
            (8, recs[8][:2] + bytes([recs[8][2] ^ 0x10]) + recs[8][3:], 14),  # one flipped fingerprint byte: another key
            (9, recs[9][:9] + bytes([recs[9][9] ^ 0x80]) + recs[9][10:], 14)):
        r = list(recs)
        r[at] = bad
        data, off = po.pack_records(r)
        with pytest.raises(emu.EmuError) as ei:
            E.partition(data, off, n, 3, fps)
        assert (ei.value.code, ei.value.record) == (code, at)
    for length in range(10):                                                # 0-9 bytes: shorter than the header
        r = list(recs)
        r[300] = SO.header(fps[0])[:length]
        data, off = po.pack_records(r)
        with pytest.raises(emu.EmuError) as ei:
            E.partition(data, off, n, 3, fps)
        assert (ei.value.code, ei.value.record) == (12, 300)
    r = list(recs)                                                           # a bare 10-byte header is a message of an empty datum
    r[300] = SO.header(fps[0])
    data, off = po.pack_records(r)
    E.partition(data, off, n, 3, fps)


@pytest.mark.parametrize("k", [1, 3, 8])
def test_partition_lowest_failing_message_wins(k):
    """Damage in a later tile and chunk is found first by the emulation (it runs last tile first); the lowest index wins."""
    rng = random.Random(k)
    n = 2500
    recs, fps = _messages(rng, n, lambda i: (i // 7) % 2)
    for first, second in ((255, 2400), (256, 1300), (383, 384), (1299, 1300)):
        r = list(recs)
        r[second] = b"\xc3"
        r[first] = SO.frame(fps[0] ^ 1, recs[first][10:])
        data, off = po.pack_records(r)
        with pytest.raises(emu.EmuError) as ei:
            E.partition(data, off, n, k, fps)
        assert (ei.value.code, ei.value.record) == (14, first)

