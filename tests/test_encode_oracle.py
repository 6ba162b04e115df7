"""The encode oracle (oracle.pyoracle.py_encode) on Arrow layouts this library's decoder never produces, and the layout
perturber (tests/arrow_layouts.py) that the GPU encode tests feed it.  CPU only.

pyarrow's `StructArray.field(i)` and sparse `UnionArray.field(i)` already apply the parent's offset, and a map's
`keys` / `items` ignore the entries struct's offset; the oracle once added parent offsets twice and dropped the
entries' offset.  It also took union children by position where the reference takes them by type code, and accepted
Arrow types the reference's exact downcasts reject."""
import random

import pyarrow as pa
import pytest

from oracle import pyoracle as po
from tests import arrow_layouts as L


def _flat(chunks):
    return [d for c in chunks for d in c]


def _random_batch(seed, n=None):
    rng = random.Random(seed)
    sj = po.random_schema_json(rng)
    s = po.parse_schema(sj)
    n = rng.choice([1, 7, 40]) if n is None else n
    vals = [po.random_value(s, rng) for _ in range(n)]
    recs = [po.encode_datum(s, v) for v in vals]
    return s, recs, po.canon_to_batch(po.py_decode(s, recs), po.to_arrow_schema(s))


def test_sliced_record_and_union_encode_their_logical_rows():
    sj = ('{"type":"record","name":"T","fields":[{"name":"r","type":{"type":"record","name":"R","fields":'
          '[{"name":"a","type":"long"}]}},{"name":"u","type":["int","string","null"]}]}')
    s = po.parse_schema(sj)
    n = 12
    u = pa.UnionArray.from_sparse(pa.array([i % 3 for i in range(n)], pa.int8()),
                                  [pa.array(range(100, 100 + n), pa.int32()), pa.array([f"s{i}" for i in range(n)]), pa.nulls(n)])
    b = pa.record_batch({"r": pa.StructArray.from_arrays([pa.array(range(100, 100 + n), pa.int64())], ["a"]), "u": u})
    got = _flat(po.py_encode(s, b.slice(5, 6)))
    want = [po.encode_datum(s, {"r": {"a": 100 + i}, "u": [(0, 100 + i), (1, f"s{i}"), (2, None)][i % 3]}) for i in range(5, 11)]
    assert got == want


def test_list_of_records_over_a_sliced_struct():
    sj = ('{"type":"record","name":"T","fields":[{"name":"l","type":{"type":"array","items":'
          '{"type":"record","name":"R","fields":[{"name":"a","type":"long"}]}}}]}')
    s = po.parse_schema(sj)
    items = pa.StructArray.from_arrays([pa.array(range(10), pa.int64())], ["a"]).slice(4)   # values at offset 4
    lst = pa.ListArray.from_arrays(pa.array([0, 2, 2, 6], pa.int32()), items)
    got = _flat(po.py_encode(s, pa.record_batch({"l": lst})))
    assert got == [po.encode_datum(s, {"l": v}) for v in ([{"a": 4}, {"a": 5}], [], [{"a": x} for x in (6, 7, 8, 9)])]


def test_map_entries_at_an_offset():
    sj = '{"type":"record","name":"T","fields":[{"name":"m","type":{"type":"map","values":"long"}}]}'
    s = po.parse_schema(sj)
    ent = pa.StructArray.from_arrays([pa.array(["x", "y", "a", "b", "c"]), pa.array([9, 9, 1, 2, 3])],
                                     fields=[pa.field("keys", pa.string(), False), pa.field("values", pa.int64())]).slice(2)
    m = pa.Array.from_buffers(pa.map_(pa.string(), pa.int64()), 2, [None, pa.py_buffer(pa.array([0, 2, 3], pa.int32()).buffers()[1])],
                              children=[ent])
    m.validate(full=True)
    assert _flat(po.py_encode(s, pa.record_batch({"m": m}))) == [po.encode_datum(s, {"m": [("a", 1), ("b", 2)]}),
                                                                 po.encode_datum(s, {"m": [("c", 3)]})]


def test_union_children_are_taken_by_type_code():
    sj = '{"type":"record","name":"T","fields":[{"name":"u","type":["string","int"]}]}'
    s = po.parse_schema(sj)
    u = pa.UnionArray.from_sparse(pa.array([1, 0, 0], pa.int8()), [pa.array([7, 8, 9], pa.int32()), pa.array(["a", "b", "c"])],
                                  type_codes=[1, 0])   # +us:1,0: the int32 child has code 1 = Avro branch "int"
    assert _flat(po.py_encode(s, pa.record_batch({"u": u}))) == [b"\x02\x0e", b"\x00\x02b", b"\x00\x02c"]
    for codes in ([5, 7], [0, 0]):
        bad = pa.UnionArray.from_sparse(pa.array([codes[0]] * 3, pa.int8()), [pa.array(["a", "b", "c"]), pa.array([7, 8, 9], pa.int32())],
                                        type_codes=codes)
        with pytest.raises(po.EncodeError, match="type codes"):
            po.py_encode(s, pa.record_batch({"u": bad}))


@pytest.mark.parametrize("avro,ok,rejected", [
    ("int", pa.int32(), [pa.date32(), pa.int64()]),
    ('{"type":"int","logicalType":"date"}', pa.date32(), [pa.int32()]),
    ("long", pa.int64(), [pa.timestamp("ms"), pa.int32()]),
    ('{"type":"long","logicalType":"timestamp-millis"}', pa.timestamp("ms", "UTC"), [pa.timestamp("us"), pa.timestamp("s"), pa.int64()]),
    ('{"type":"long","logicalType":"timestamp-micros"}', pa.timestamp("us"), [pa.timestamp("ms"), pa.timestamp("ns", "UTC"), pa.int64()]),
])
def test_exact_downcasts(avro, ok, rejected):
    s = po.parse_schema('{"type":"record","name":"T","fields":[{"name":"x","type":%s}]}' % (avro if avro[0] == "{" else f'"{avro}"'))
    assert _flat(po.py_encode(s, pa.record_batch({"x": pa.array([3], ok)}))) == [b"\x06"]
    for t in rejected:
        with pytest.raises(po.EncodeError, match="downcast failed"):
            po.py_encode(s, pa.record_batch({"x": pa.array([3], t)}))


@pytest.mark.parametrize("seed", range(30))
def test_slices_encode_their_rows(seed):
    s, recs, batch = _random_batch(seed, 40)
    assert _flat(po.py_encode(s, batch)) == recs
    rng = random.Random(seed)
    for a, m in ((0, 40), (1, 30), (rng.randrange(1, 40), None), (39, 1), (17, 0)):
        m = rng.randrange(0, 41 - a) if m is None else m
        assert _flat(po.py_encode(s, batch.slice(a, m))) == recs[a:a + m]    # recs: encode_datum of the values


@pytest.mark.parametrize("variation", L.VARIATIONS + ("all",))
@pytest.mark.parametrize("seed", range(12))
def test_relayout_keeps_values_and_datums(seed, variation):
    s, recs, batch = _random_batch(seed)
    var = L.KEEPS_DATUMS if variation == "all" else (variation,)
    b2 = L.relayout_batch(batch, random.Random(1000 * seed + 7), var)
    b2.validate(full=True)
    if variation == "nonnull_junk":      # raw values of non-nullable null slots change the datums: only the oracle runs
        po.py_encode(s, b2)
        return
    for x, y in zip(b2.columns, batch.columns):
        if x.type == y.type:            # permuted union codes change the type; the datums below still pin the values
            assert x.equals(y)
    assert _flat(po.py_encode(s, b2)) == recs
