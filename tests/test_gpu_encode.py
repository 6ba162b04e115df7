"""GPU parity of the Arrow -> Avro direct encode (serialize_record_batch, SURVEY.md 8(f) rank 1) against the
pure-Python restatement of fast_encode.rs (oracle.pyoracle.py_encode) and against the round-trip property the
reference's own tests use (fast_encode.rs:616-637: avro -> decode -> encode gives the datums back)."""
import random

import numpy as np
import pyarrow as pa
import pytest

import pyruhvro_b200 as pr
from oracle import pyoracle as po
from tests import arrow_layouts as L
from tests.golden import reference_datums as G

pytestmark = pytest.mark.gpu


def _datums(arrays):
    return [bytes(x.as_py()) for a in arrays for x in a]


@pytest.mark.parametrize("seed", range(40))
def test_round_trip_and_oracle(coracle, seed):
    rng = random.Random(seed)
    sj = po.random_schema_json(rng)
    s = po.parse_schema(sj)
    n = rng.choice([1, 33, 257, 700])
    recs = [po.encode_datum(s, po.random_value(s, rng)) for _ in range(n)]
    batch = pr.deserialize_array(recs, sj)
    k = rng.choice([1, 2, 5])
    out = pr.serialize_record_batch(batch, sj, k)
    assert len(out) == po.clamp_chunks(k, n) and all(a.type == pa.binary() for a in out)
    assert [len(a) for a in out] == [b - a for a, b in po.chunk_bounds(n, po.clamp_chunks(k, n))]
    assert _datums(out) == recs                                     # avro -> arrow -> avro is the identity
    want = po.py_encode(s, po.canon_to_batch(coracle.decode(sj, recs), po.to_arrow_schema(s)), k)
    assert [[bytes(x.as_py()) for x in a] for a in out] == want     # and equals the fast_encode.rs restatement


def test_reference_golden_datums():
    recs = [bytes.fromhex(h) for h in (G.G3_HEX, G.G4_HEX, G.G5_HEX)]
    batch = pr.deserialize_array(recs, G.G345_SCHEMA)
    out = _datums(pr.serialize_record_batch(batch, G.G345_SCHEMA, 1))   # what lib.rs:174-178 does (asserting only "no error")
    assert out[0] == recs[0][:157] and out[1] == recs[1] and out[2] == recs[2]
    for sj, hx in ((G.G1_SCHEMA, G.G1_HEX), (G.G2_SCHEMA, G.G2_HEX)):
        r = bytes.fromhex(hx)
        assert _datums(pr.serialize_record_batch(pr.deserialize_array([r, r], sj), sj, 2)) == [r, r]


def test_columns_matched_by_name_and_slices():
    import workloads
    sj, data, off = workloads.generate("kafka", 3000, seed=3)
    recs = [bytes(data[off[i]:off[i + 1]]) for i in range(3000)]
    batch = pr.deserialize_array(recs, sj)
    names = list(batch.schema.names)
    shuffled = pa.RecordBatch.from_arrays([batch.column(n) for n in reversed(names)], names=list(reversed(names)))
    assert _datums(pr.serialize_record_batch(shuffled, sj, 3)) == recs       # fast_encode.rs:157-181
    sl = batch.slice(100, 1234)                                              # offsets / slices are honoured
    assert _datums(pr.serialize_record_batch(sl, sj, 4)) == recs[100:1334]
    extra = shuffled.append_column("unused", pa.array(range(3000)))
    assert _datums(pr.serialize_record_batch(extra, sj, 1)) == recs


def test_large_batch_takes_the_staged_upload_and_round_trips():
    """A decoded batch of more than 16 MiB, whole and sliced, encodes back to the input datums (decode -> encode
    identity).  Its buffers are the decoder's pinned slabs, so encode_group copies them directly; the staged upload of
    pageable buffers is test_pageable_buffers_are_staged_in_pieces."""
    import numpy as np
    import workloads
    n = 200_000
    sj, data, off = workloads.generate("kafka", n, seed=11)
    batch = pr.decode_packed(data, off, n, sj, 1)[0]
    assert batch.nbytes > (16 << 20)
    for b, lo, k in ((batch, 0, 3), (batch.slice(12_345, 150_000), 12_345, 2)):
        out = pr.serialize_record_batch(b, sj, k)
        offs = [np.frombuffer(a.buffers()[1], dtype=np.int32)[:len(a) + 1] for a in out]
        got = np.concatenate([np.frombuffer(a.buffers()[2], dtype=np.uint8)[:o[-1]] for a, o in zip(out, offs)])
        assert got.tobytes() == data[off[lo]:off[lo + b.num_rows]].tobytes()
        lens = np.concatenate([np.diff(o) for o in offs])
        assert np.array_equal(lens, np.diff(off[lo:lo + b.num_rows + 1]))


def test_row_groups_keep_each_chunk_alive_on_its_own():
    """From 2^18 rows the chunks are encoded in concurrent row groups (encode.cu: rv_encode_host).  Every exported array
    must own ITS chunk's memory: drop all but one array, churn the pinned cache with further calls, and the survivor
    still holds its datums."""
    import gc
    import numpy as np
    import workloads
    n, k = 600_000, 8
    sj, data, off = workloads.generate("kafka", n, seed=5)
    batch = pr.decode_packed(data, off, n, sj, 1)[0]
    rows = n // k
    for keep in (0, 3, 7):
        out = pr.serialize_record_batch(batch, sj, k)
        assert [len(a) for a in out] == [rows] * (k - 1) + [n - rows * (k - 1)]
        survivor = out[keep]
        del out
        gc.collect()
        for _ in range(2):                                          # re-uses whatever the dropped arrays gave back
            pr.serialize_record_batch(batch.slice(17, 300_000), sj, 5)
        lo = keep * rows
        o = np.frombuffer(survivor.buffers()[1], dtype=np.int32)[:len(survivor) + 1]
        got = np.frombuffer(survivor.buffers()[2], dtype=np.uint8)[:o[-1]]
        assert got.tobytes() == data[off[lo]:off[lo + len(survivor)]].tobytes()
        assert np.array_equal(np.diff(o), np.diff(off[lo:lo + len(survivor) + 1]))


def test_error_surface():
    recs = [bytes.fromhex(G.G2_HEX)]
    batch = pr.deserialize_array(recs, G.G2_SCHEMA)
    with pytest.raises(ValueError) as e:
        pr.serialize_record_batch(batch.drop_columns(["age"]), G.G2_SCHEMA, 1)
    assert "Arrow struct missing column 'age' required by Avro schema. Available columns:" in str(e.value)   # :171-179
    with pytest.raises(ValueError):
        pr.serialize_record_batch(batch.set_column(2, "age", pa.array(["x"])), G.G2_SCHEMA, 1)               # downcast failure
    sj = '{"type":"record","name":"E","fields":[{"name":"e","type":{"type":"enum","name":"S","symbols":["A","B"]}}]}'
    with pytest.raises(ValueError) as e:
        pr.serialize_record_batch(pa.record_batch({"e": ["A", "Z", "B"]}), sj, 1)
    assert "enum symbol" in str(e.value) and "(row 1)" in str(e.value)                                        # :573-576
    assert _datums(pr.serialize_record_batch(pa.record_batch({"e": ["A", "B", "B"]}), sj, 1)) == [b"\x00", b"\x02", b"\x02"]
    out = pr.serialize_record_batch(batch.slice(0, 0), G.G2_SCHEMA, 8)
    assert len(out) == 1 and len(out[0]) == 0                                                                  # n = 0 -> one empty chunk


def test_null_slots_of_non_nullable_fields_encode_their_raw_value():
    """`array.value(row)` ignores validity for non-nullable Avro fields (fast_encode.rs:401-409)."""
    sj = '{"type":"record","name":"N","fields":[{"name":"a","type":"long"},{"name":"b","type":["null","long"]}]}'
    b = pa.record_batch({"a": pa.array([1, None, 3], pa.int64()), "b": pa.array([None, 5, None], pa.int64())})
    got = _datums(pr.serialize_record_batch(b, sj, 1))
    want = [d for ch in po.py_encode(po.parse_schema(sj), b, 1) for d in ch]
    assert got == want == [b"\x02\x00", b"\x00\x02\x0a", b"\x06\x00"]


# --------------------------------------------------------------------------------------------------------------------
# Arrow layouts the decoder never produces, and the encoder's own tile, window and error paths
# --------------------------------------------------------------------------------------------------------------------
TILE = 256                 # rows per CTA tile (kBlock)
STAGE_CAP = 100 * 1024     # encode_write_kernel assembles a tile in at most this much shared memory


def _chunks(out):
    return [[bytes(x.as_py()) for x in a] for a in out]


def _random_case(seed, n):
    rng = random.Random(seed)
    sj = po.random_schema_json(rng)
    s = po.parse_schema(sj)
    recs = [po.encode_datum(s, po.random_value(s, rng)) for _ in range(n)]
    return sj, s, recs, pr.deserialize_array(recs, sj)


@pytest.mark.parametrize("variation", L.VARIATIONS + ("all",))
@pytest.mark.parametrize("seed", range(6))
def test_relaid_batches_match_the_oracle(monkeypatch, seed, variation):
    sj, s, recs, batch = _random_case(seed, 300)
    var = L.KEEPS_DATUMS if variation == "all" else (variation,)
    b2 = L.relayout_batch(batch, random.Random(seed * 13 + 1), var)
    for k in (1, 2, 5):
        for groups in (None, "3"):
            if groups:
                monkeypatch.setenv("RV_ENC_GROUPS", groups)       # read on every call: groups at a small n
            else:
                monkeypatch.delenv("RV_ENC_GROUPS", raising=False)
            got = _chunks(pr.serialize_record_batch(b2, sj, k))
            assert got == po.py_encode(s, b2, k), (k, groups)
            if variation != "nonnull_junk":
                assert [d for c in got for d in c] == recs


@pytest.mark.parametrize("seed", range(4))
def test_slices_of_relaid_batches(monkeypatch, seed):
    sj, s, recs, batch = _random_case(100 + seed, 600)
    b2 = L.relayout_batch(batch, random.Random(seed), L.KEEPS_DATUMS)
    rng = random.Random(seed)
    monkeypatch.setenv("RV_ENC_GROUPS", "2")
    for o in list(range(10)) + [rng.randrange(10, 600) for _ in range(3)]:
        m = rng.randrange(0, 600 - o + 1)
        k = rng.choice([1, 2, 3])
        sl = b2.slice(o, m)
        got = _chunks(pr.serialize_record_batch(sl, sj, k))
        assert [d for c in got for d in c] == recs[o:o + m]
        if m <= 400:
            assert got == po.py_encode(s, sl, k)


@pytest.mark.parametrize("name", ["kafka", "wide"])
def test_benchmark_batches_relaid_at_every_level(name):
    import workloads
    n = 1500
    sj, data, off = workloads.generate(name, n, seed=21)
    recs = [bytes(data[off[i]:off[i + 1]]) for i in range(n)]
    b2 = L.relayout_batch(pr.deserialize_array(recs, sj), random.Random(5), L.KEEPS_DATUMS)
    for k in (1, 4):
        assert _datums(pr.serialize_record_batch(b2, sj, k)) == recs
    assert _chunks(pr.serialize_record_batch(b2.slice(0, 300), sj, 2)) == po.py_encode(po.parse_schema(sj), b2.slice(0, 300), 2)


FLAT = ('{"type":"record","name":"F","fields":[{"name":"i","type":"int"},{"name":"s","type":["null","string"]},'
        '{"name":"b","type":"boolean"},{"name":"u","type":["long","string","null"]}]}')


def _flat_batch(n, seed=0):
    rng = random.Random(seed)
    s = po.parse_schema(FLAT)
    recs = [po.encode_datum(s, po.random_value(s, rng)) for _ in range(n)]
    return s, recs, pr.deserialize_array(recs, FLAT) if n else None


@pytest.mark.parametrize("n", [1, 255, 256, 257, 511, 513])
def test_tile_and_chunk_edges(n):
    s, recs, batch = _flat_batch(n, n)
    b2 = L.relayout_batch(batch, random.Random(n), L.KEEPS_DATUMS)
    for k in (1, 2, 3, n, n + 5):
        out = pr.serialize_record_batch(b2, FLAT, k)
        kk = po.clamp_chunks(k, n)
        assert [len(a) for a in out] == [b - a for a, b in po.chunk_bounds(n, kk)]
        assert _chunks(out) == po.py_encode(s, b2, k) and _datums(out) == recs


@pytest.mark.parametrize("n", [0, 1, 256, 257, 700])
def test_rows_of_zero_bytes(monkeypatch, n):
    """Every row encodes to nothing: every tile has tile_total == 0 and every chunk's data is empty.  (No Avro value but
    null, or records of nulls, encodes to zero bytes, so such rows cannot share a batch with non-empty ones.)"""
    sj = ('{"type":"record","name":"Z","fields":[{"name":"a","type":"null"},{"name":"r","type":{"type":"record",'
          '"name":"R","fields":[{"name":"x","type":"null"},{"name":"y","type":"null"}]}}]}')
    b = pa.record_batch({"a": pa.nulls(n), "r": pa.StructArray.from_arrays([pa.nulls(n), pa.nulls(n)], ["x", "y"])})
    monkeypatch.setenv("RV_ENC_GROUPS", "2")
    for k in (1, 3):
        out = pr.serialize_record_batch(b, sj, k)
        assert sum(len(a) for a in out) == n and all(x.as_py() == b"" for a in out for x in a)
        assert _chunks(out) == po.py_encode(po.parse_schema(sj), b, k)
        for a in out:
            assert np.all(np.frombuffer(a.buffers()[1], dtype=np.int32)[:len(a) + 1] == 0)


def test_tiles_above_the_staging_cap_are_written_unstaged():
    """Tiles of 1-8 KB rows exceed the 100 KiB staging cap and are written straight to global memory; tiles of short
    rows are assembled in shared memory.  The test recomputes which tiles take which path and requires both."""
    sj = '{"type":"record","name":"W","fields":[{"name":"s","type":"string"},{"name":"x","type":"long"}]}'
    s = po.parse_schema(sj)
    rng = random.Random(3)
    n = 8 * TILE + 77
    big = lambda i: (i // TILE) % 2 == 0                                       # noqa: E731
    vals = [{"s": "x" * (rng.randint(1024, 8192) if big(i) else rng.randint(0, 300)), "x": i} for i in range(n)]
    recs = [po.encode_datum(s, v) for v in vals]
    batch = L.relayout_batch(pa.record_batch({"s": [v["s"] for v in vals], "x": pa.array(range(n), pa.int64())}),
                             random.Random(1), ("offset", "unaligned"))
    for k in (1, 3):
        out = pr.serialize_record_batch(batch, sj, k)
        assert _chunks(out) == po.py_encode(s, batch, k) and _datums(out) == recs
        kinds = set()
        for c0, c1 in po.chunk_bounds(n, po.clamp_chunks(k, n)):
            lens = [len(r) for r in recs[c0:c1]]
            tiles = [sum(lens[t:t + TILE]) for t in range(0, len(lens), TILE)]
            cap = (min(max(tiles) + 32, STAGE_CAP) + 63) // 64 * 64
            base = 0
            for tot in tiles:                            # staged iff the tile plus its 16-byte misalignment fits
                kinds.add(tot + (base & 15) <= cap)
                base += tot
        assert kinds == {True, False}, k


def test_pageable_buffers_are_staged_in_pieces(monkeypatch):
    """numpy-built buffers are ordinary pageable memory: above 4 MiB per row group the upload is staged through pinned
    memory in 16 MiB pieces.  The string data of each row group spans more than one piece."""
    n = 60_000
    rng = np.random.default_rng(7)
    lens = rng.integers(600, 1400, n).astype(np.int32)
    offs = np.zeros(n + 1, dtype=np.int32)
    np.cumsum(lens, out=offs[1:])
    data = rng.integers(97, 123, int(offs[-1]), dtype=np.uint8)
    x = rng.integers(-1000, 1000, n).astype(np.int64)
    s_col = pa.Array.from_buffers(pa.string(), n, [None, pa.py_buffer(offs), pa.py_buffer(data)])
    batch = pa.record_batch({"s": s_col, "x": pa.array(x)})
    sj = '{"type":"record","name":"P","fields":[{"name":"s","type":"string"},{"name":"x","type":"long"}]}'
    s = po.parse_schema(sj)
    lo, m, k = 1234, 56_000, 4
    monkeypatch.setenv("RV_ENC_GROUPS", "2")
    bounds = po.chunk_bounds(m, k)
    for g0, g1 in ((bounds[0][0], bounds[1][1]), (bounds[2][0], bounds[3][1])):   # each row group's string window
        assert offs[lo + g1] - offs[lo + g0] > (16 << 20)
    out = pr.serialize_record_batch(batch.slice(lo, m), sj, k)
    got_lens = np.concatenate([np.diff(np.frombuffer(a.buffers()[1], dtype=np.int32)[:len(a) + 1]) for a in out])
    zz = lambda v: len(po.zigzag_bytes(int(v)))                                  # noqa: E731
    assert np.array_equal(got_lens, [zz(lens[i]) + lens[i] + zz(x[i]) for i in range(lo, lo + m)])
    flat = _datums(out)
    for i in list(range(0, m, 997)) + [m - 1]:
        r = lo + i
        assert flat[i] == po.encode_datum(s, {"s": data[offs[r]:offs[r + 1]].tobytes(), "x": int(x[r])})


def test_columns_sharing_one_array_merge_their_windows(monkeypatch):
    sj = ('{"type":"record","name":"S","fields":[{"name":"a","type":"string"},{"name":"b","type":["null","string"]},'
          '{"name":"c","type":"long"},{"name":"d","type":"long"}]}')
    s = po.parse_schema(sj)
    n = 1000
    base = pa.array([None if i % 7 == 3 else "v%d" % (i * 37 % 1000) for i in range(n + 400)])
    nums = pa.array(range(n + 400), pa.int64())
    a, b = base.slice(0, n), base.slice(300, n)
    assert a.buffers()[2].address == b.buffers()[2].address              # one buffer, two windows to merge
    batch = pa.record_batch({"a": a, "b": b, "c": nums.slice(400, n), "d": nums.slice(0, n)})
    for groups in ("1", "3"):
        monkeypatch.setenv("RV_ENC_GROUPS", groups)
        for k in (1, 3):
            assert _chunks(pr.serialize_record_batch(batch, sj, k)) == po.py_encode(s, batch, k)


ENUM_UNION = ('{"type":"record","name":"E","fields":[{"name":"i","type":"long"},'
              '{"name":"e","type":{"type":"enum","name":"S","symbols":["A","BB","C"]}},'
              '{"name":"u","type":["int","string","null"]}]}')


def _enum_union_batch(n, bad_sym=(), bad_tid=()):
    tids = [i % 3 for i in range(n)]
    for r, t in bad_tid:
        tids[r] = t
    syms = ["A", "BB", "C"]
    e = [syms[i % 3] for i in range(n)]
    for r in bad_sym:
        e[r] = "ZZ"
    u = pa.UnionArray.from_sparse(pa.array(tids, pa.int8()), [pa.array(range(n), pa.int32()), pa.array([f"s{i}" for i in range(n)]), pa.nulls(n)])
    return pa.record_batch({"i": pa.array(range(n), pa.int64()), "e": e, "u": u})


@pytest.mark.parametrize("bad", [("sym", 0), ("sym", 255), ("sym", 256), ("sym", -1), ("tid", -1), ("tid", 3), ("tid", 127)])
def test_first_error_is_reported_with_its_row(monkeypatch, bad):
    n = 1200
    s = po.parse_schema(ENUM_UNION)
    rows = [0, 255, 256, n - 1] if bad[0] == "tid" else [bad[1] % n]
    for first in rows:
        more = sorted({first, min(n - 1, first + 300), n - 1})          # later bad rows, in other chunks and groups
        b = _enum_union_batch(n, bad_sym=more if bad[0] == "sym" else (), bad_tid=[(r, bad[1]) for r in more] if bad[0] == "tid" else ())
        with pytest.raises(po.EncodeError, match="enum symbol" if bad[0] == "sym" else "type_id"):
            po.py_encode(s, b)
        for groups, k in (("1", 1), ("3", 5)):
            monkeypatch.setenv("RV_ENC_GROUPS", groups)
            with pytest.raises(ValueError) as e:
                pr.serialize_record_batch(b, ENUM_UNION, k)
            assert ("enum symbol" if bad[0] == "sym" else "type_id out of range") in str(e.value)
            assert f"(row {first})" in str(e.value), (groups, k, str(e.value))


def test_bad_values_that_are_not_encoded_raise_nothing():
    sj = ('{"type":"record","name":"N","fields":[{"name":"e","type":["null",{"type":"enum","name":"S","symbols":["A","B"]}]},'
          '{"name":"u","type":["int",{"type":"enum","name":"T","symbols":["X"]}]},'
          '{"name":"l","type":{"type":"array","items":{"type":"enum","name":"V","symbols":["P"]}}}]}')
    s = po.parse_schema(sj)
    n = 600
    e = pa.Array.from_buffers(pa.string(), n, [pa.array([i % 5 != 2 for i in range(n)]).buffers()[1],
                                               *pa.array(["A" if i % 5 != 2 else "junk" for i in range(n)]).buffers()[1:]])
    u = pa.UnionArray.from_sparse(pa.array([0] * n, pa.int8()), [pa.array(range(n), pa.int32()), pa.array(["nope"] * n)])
    items = pa.array(["bad", "P", "P", "bad"])                              # the rows' range is items 1..2
    lst = pa.ListArray.from_arrays(pa.array([1, 3] + [3] * (n - 1), pa.int32()), items)
    b = pa.record_batch({"e": e, "u": u, "l": lst})
    want = po.py_encode(s, b, 3)                                              # the oracle raises nothing either
    assert _chunks(pr.serialize_record_batch(b, sj, 3)) == want


def test_one_chunk_over_the_i32_limit_is_an_error():
    """Needs about 1.1 GB of host input, 1.1 GB of pinned staging and 2.2 GB of encoded output (host and device).
    One 1.1 GB Utf8 array serves as two columns, so one chunk would hold 2.2 GB of datums: more than i32 offsets can
    address.  Split in two chunks it fits."""
    n, w = 1_100_000, 1000
    offs = np.arange(n + 1, dtype=np.int32) * w
    data = np.full(n * w, ord("q"), dtype=np.uint8)
    data[::w] = np.arange(n * w // w, dtype=np.int64) % 26 + 65
    col = pa.Array.from_buffers(pa.string(), n, [None, pa.py_buffer(offs), pa.py_buffer(data)])
    sj = '{"type":"record","name":"O","fields":[{"name":"a","type":"string"},{"name":"b","type":"string"}]}'
    b = pa.record_batch({"a": col, "b": col})
    with pytest.raises(ValueError, match="i32 offset overflow"):
        pr.serialize_record_batch(b, sj, 1)
    out = pr.serialize_record_batch(b, sj, 2)
    assert [len(a) for a in out] == [n // 2, n - n // 2]
    d = 2 * (2 + w)                                   # zigzag(1000) is two bytes
    s = po.parse_schema(sj)
    for a, r0 in zip(out, (0, n // 2)):
        o = np.frombuffer(a.buffers()[1], dtype=np.int32)[:len(a) + 1]
        assert np.all(np.diff(o) == d) and o[0] == 0
        body = np.frombuffer(a.buffers()[2], dtype=np.uint8)
        for i in (0, 1, len(a) // 2, len(a) - 1):
            txt = data[(r0 + i) * w:(r0 + i + 1) * w].tobytes()
            assert body[o[i]:o[i + 1]].tobytes() == po.encode_datum(s, {"a": txt, "b": txt})


LEAVES = ["int", '{"type":"int","logicalType":"date"}', "long", '{"type":"long","logicalType":"timestamp-millis"}',
          '{"type":"long","logicalType":"timestamp-micros"}', "float", "double", "boolean", "string",
          '{"type":"enum","name":"S","symbols":["A","B"]}']
ARROW_TYPES = [pa.int32(), pa.date32(), pa.int64()] + [pa.timestamp(u, tz) for u in "s ms us ns".split() for tz in (None, "UTC")] + \
    [pa.float32(), pa.float64(), pa.bool_(), pa.utf8(), pa.large_utf8()]


def _column(t, n=5):
    if pa.types.is_boolean(t):
        return pa.array([i % 2 == 0 for i in range(n)])
    if pa.types.is_string(t) or pa.types.is_large_string(t):
        return pa.array(["AB"[i % 2] for i in range(n)], t)
    if pa.types.is_floating(t):
        return pa.array([i * 1.5 - 2 for i in range(n)], t)
    return pa.array([i * 1000 - 2 for i in range(n)], pa.int64()).cast(t) if not pa.types.is_date32(t) else pa.array([i - 2 for i in range(n)], pa.int32()).cast(t)


@pytest.mark.parametrize("leaf", LEAVES)
def test_type_matrix(leaf):
    for nullable in (False, True):
        typ = leaf if leaf[0] in "{" else f'"{leaf}"'
        sj = '{"type":"record","name":"T","fields":[{"name":"x","type":%s}]}' % (f'["null",{typ}]' if nullable else typ)
        s = po.parse_schema(sj)
        for t in ARROW_TYPES:
            b = pa.record_batch({"x": _column(t)})
            try:
                want = po.py_encode(s, b, 2)
            except po.EncodeError:
                with pytest.raises(ValueError):
                    pr.serialize_record_batch(b, sj, 2)
                continue
            assert _chunks(pr.serialize_record_batch(b, sj, 2)) == want, (leaf, nullable, t)


def test_union_layouts_and_type_codes():
    """Sparse unions take their Avro variants by type code; dense unions, and codes that are not 0..N-1, are errors."""
    sj = '{"type":"record","name":"U","fields":[{"name":"u","type":["string",{"type":"enum","name":"S","symbols":["A","B"]},"int"]}]}'
    s = po.parse_schema(sj)
    n = 300
    tids = pa.array([i % 3 for i in range(n)], pa.int8())
    strs, syms, ints = pa.array([f"s{i}" for i in range(n)]), pa.array(["AB"[i % 2] for i in range(n)]), pa.array(range(n), pa.int32())
    want = [po.encode_datum(s, {"u": [(0, f"s{i}"), (1, i % 2), (2, i)][i % 3]}) for i in range(n)]
    for order in ([0, 1, 2], [1, 0, 2], [2, 1, 0], [1, 2, 0]):       # string and enum share Utf8: only the code tells them apart
        kids = [[strs, syms, ints][c] for c in order]
        b = pa.record_batch({"u": pa.UnionArray.from_sparse(tids, kids, type_codes=order)})
        assert _chunks(pr.serialize_record_batch(b, sj, 2)) == po.py_encode(s, b, 2)
        assert _datums(pr.serialize_record_batch(b, sj, 2)) == want
    for codes in ([5, 7, 0], [0, 0, 1]):
        b = pa.record_batch({"u": pa.UnionArray.from_sparse(pa.array([codes[0]] * n, pa.int8()), [strs, syms, ints], type_codes=codes)})
        with pytest.raises(po.EncodeError):
            po.py_encode(s, b)
        with pytest.raises(ValueError, match="type codes"):
            pr.serialize_record_batch(b, sj, 1)
    dense = pa.UnionArray.from_dense(tids, pa.array([i // 3 for i in range(n)], pa.int32()), [strs, syms, ints])
    with pytest.raises(po.EncodeError):
        po.py_encode(s, pa.record_batch({"u": dense}))
    with pytest.raises(ValueError):
        pr.serialize_record_batch(pa.record_batch({"u": dense}), sj, 1)
