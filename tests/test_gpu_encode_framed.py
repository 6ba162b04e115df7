"""GPU tests of the framed encodes: Object Container Files (serialize_ocf) byte for byte against the container writer of
the tests (tests/ocf_files.py) and against an assembly from serialize_record_batch's datums, and Confluent-framed
messages (serialize_confluent) against serialize_record_batch's datums with the 5-byte header."""
import random

import numpy as np
import pyarrow as pa
import pytest

import pyruhvro_b200 as pr
from oracle import pyoracle as po
from tests import arrow_layouts as L
from tests import ocf_files as O

pytestmark = pytest.mark.gpu

BLOCKS = (1, 7, 255, 256, 257, 1000)


def _counts(n, r):
    return [min(r, n - i) for i in range(0, n, r)]


def _meta(rng):
    return {"user.name": bytes(rng.randrange(256) for _ in range(rng.randrange(6))), "k": b"", "z" * 40: b"\x00\x01"}


def _assemble(sj, datums_arrays, r, sync, meta):
    """The expected file from serialize_record_batch's datums (one chunk), assembled with numpy."""
    (a,) = datums_arrays
    n = len(a)
    off = np.frombuffer(a.buffers()[1], dtype=np.int32)[:n + 1]
    data = np.frombuffer(a.buffers()[2], dtype=np.uint8) if n else np.zeros(0, np.uint8)
    parts = [np.frombuffer(O.ocf_header(sj, sync, meta), dtype=np.uint8)]
    s = np.frombuffer(sync, dtype=np.uint8)
    for i in range(0, n, r):
        j = min(n, i + r)
        parts += [np.frombuffer(O.zz(j - i) + O.zz(int(off[j] - off[i])), dtype=np.uint8), data[off[i]:off[j]], s]
    return np.concatenate(parts)


def _same_decode(f, recs, sj, k):
    got = pr.deserialize_ocf(f, k)
    want = pr.deserialize_array_threaded(recs, sj, k) if recs else [pr.deserialize_array([], sj)]
    assert len(got) == len(want)
    for g, w in zip(got, want):
        d = po.canon_diff(po.canon_from_batch(g), po.canon_from_batch(w))
        assert d is None, d


@pytest.mark.parametrize("seed", range(40))
def test_ocf_matches_the_container_writer(seed):
    rng = random.Random(seed)
    sj = po.random_schema_json(rng)
    s = po.parse_schema(sj)
    n = rng.choice([1, 33, 257, 700])
    recs = [po.encode_datum(s, po.random_value(s, rng)) for _ in range(n)]
    batch = pr.deserialize_array(recs, sj)
    datums = po.py_encode(s, batch, 1)[0]
    for r in BLOCKS + (n, n + 5):
        sync = bytes(rng.randrange(256) for _ in range(16))
        meta = _meta(rng)
        f = pr.serialize_ocf(batch, sj, r, sync_marker=sync, metadata=meta)
        assert isinstance(f, pa.Buffer)
        want = O.ocf_file(sj, datums, counts=_counts(n, r), sync=sync, meta_extra=meta)
        assert f.to_pybytes() == want, r
        got_sj, got_datums, blocks = po.ocf_read(f.to_pybytes())
        assert got_sj == sj and got_datums == recs and [c for _, c in blocks] == _counts(n, r)
    _same_decode(f, recs, sj, rng.choice([1, 3, 8]))


@pytest.mark.parametrize("variation", L.VARIATIONS)
def test_ocf_of_relaid_batches(monkeypatch, variation):
    rng = random.Random(L.VARIATIONS.index(variation))
    sj = po.random_schema_json(random.Random(7))
    s = po.parse_schema(sj)
    recs = [po.encode_datum(s, po.random_value(s, rng)) for _ in range(600)]
    b2 = L.relayout_batch(pr.deserialize_array(recs, sj), rng, (variation,))
    want_datums = po.py_encode(s, b2, 1)[0]
    for groups in ("1", "3"):
        monkeypatch.setenv("RV_ENC_GROUPS", groups)
        for r in (1, 257, 600):
            sync = bytes(range(16, 32))
            f = pr.serialize_ocf(b2, sj, r, sync_marker=sync, metadata={"m": b"v"})
            assert f.to_pybytes() == O.ocf_file(sj, want_datums, counts=_counts(600, r), sync=sync, meta_extra={"m": b"v"})
            sl = b2.slice(17, 400)
            f = pr.serialize_ocf(sl, sj, r, sync_marker=sync)
            assert f.to_pybytes() == O.ocf_file(sj, want_datums[17:417], counts=_counts(400, r), sync=sync)


def test_ocf_of_no_rows_one_row_and_one_row_blocks():
    import workloads
    sj, data, off = workloads.generate("kafka", 5000, seed=4)
    recs = [bytes(data[off[i]:off[i + 1]]) for i in range(5000)]
    batch = pr.deserialize_array(recs, sj)
    sync = bytes(range(100, 116))
    f0 = pr.serialize_ocf(batch.slice(0, 0), sj, sync_marker=sync)
    assert f0.to_pybytes() == O.ocf_header(sj, sync) == O.ocf_file(sj, [], counts=[], sync=sync)
    assert sum(b.num_rows for b in pr.deserialize_ocf(f0, 2)) == 0
    f1 = pr.serialize_ocf(batch.slice(4999, 1), sj, sync_marker=sync)
    assert f1.to_pybytes() == O.ocf_file(sj, recs[4999:], counts=[1], sync=sync)
    f = pr.serialize_ocf(batch, sj, 1, sync_marker=sync)
    assert f.to_pybytes() == O.ocf_file(sj, recs, counts=[1] * 5000, sync=sync)
    assert len(O.block_spans(f.to_pybytes())) == 5000
    _same_decode(f, recs, sj, 3)
    assert pr.lib.rv_last_encode_timings((pr.ctypes.c_float * 5)(), 5) == 5


def test_default_sync_marker_is_random_and_repeated_after_every_block():
    import workloads
    sj, data, off = workloads.generate("kafka", 3000, seed=5)
    batch = pr.decode_packed(data, off, 3000, sj, 1)[0]
    a, b = pr.serialize_ocf(batch, sj).to_pybytes(), pr.serialize_ocf(batch, sj).to_pybytes()
    spans = O.block_spans(a)
    assert [c for *_, c in spans] == [1024, 1024, 952]
    marker = a[spans[0][0] - 16:spans[0][0]]
    assert all(a[p + sz:p + sz + 16] == marker for _, p, sz, _ in spans)
    assert a != b and len(a) == len(b)


@pytest.mark.parametrize("groups", ["1", "4"])
def test_ocf_row_groups_match_the_assembly_from_datums(monkeypatch, groups):
    """300 000 Kafka rows take the row-group path (two phases: sizes of every group first, then the file)."""
    import workloads
    n = 300_000
    sj, data, off = workloads.generate("kafka", n, seed=9)
    batch = pr.decode_packed(data, off, n, sj, 1)[0]
    monkeypatch.setenv("RV_ENC_GROUPS", groups)
    sync = bytes(range(40, 56))
    meta = {"writer": b"test"}
    for r, b in ((1024, batch), (1000, batch.slice(1234, 250_000))):
        f = pr.serialize_ocf(b, sj, r, sync_marker=sync, metadata=meta)
        want = _assemble(sj, pr.serialize_record_batch(b, sj, 1), r, sync, meta)
        assert np.array_equal(np.frombuffer(f, dtype=np.uint8), want), r
    t = (pr.ctypes.c_float * 5)()
    pr.lib.rv_last_encode_timings(t, 5)
    assert all(x > 0 for x in t)


def _errors_batch(n, bad_sym=(), bad_tid=()):
    tids = [i % 3 for i in range(n)]
    for r in bad_tid:
        tids[r] = 3
    e = [["A", "BB", "C"][i % 3] for i in range(n)]
    for r in bad_sym:
        e[r] = "ZZ"
    u = pa.UnionArray.from_sparse(pa.array(tids, pa.int8()), [pa.array(range(n), pa.int32()), pa.array(["s"] * n), pa.nulls(n)])
    return pa.record_batch({"i": pa.array(range(n), pa.int64()), "e": e, "u": u})


ENUM_UNION = ('{"type":"record","name":"E","fields":[{"name":"i","type":"long"},'
              '{"name":"e","type":{"type":"enum","name":"S","symbols":["A","BB","C"]}},'
              '{"name":"u","type":["int","string","null"]}]}')


@pytest.mark.parametrize("kind", ["sym", "tid"])
def test_errors_in_a_later_block_and_row_group(monkeypatch, kind):
    n = 300_000
    first = 200_123
    bad = [first, first + 5, 280_000]
    b = _errors_batch(n, bad_sym=bad if kind == "sym" else (), bad_tid=bad if kind == "tid" else ())
    monkeypatch.setenv("RV_ENC_GROUPS", "4")
    with pytest.raises(ValueError) as plain:
        pr.serialize_record_batch(b, ENUM_UNION, 8)
    for r in (1000, 1024, 77_777):
        with pytest.raises(ValueError) as e:
            pr.serialize_ocf(b, ENUM_UNION, r)
        assert str(e.value) == str(plain.value) and f"(row {first})" in str(e.value)
        with pytest.raises(ValueError) as e:
            pr.serialize_confluent(b, ENUM_UNION, 12, 8)
        assert str(e.value) == str(plain.value)


def _big_string_batch(n, w, cols):
    offs = np.arange(n + 1, dtype=np.int32) * w
    data = np.full(n * w, ord("q"), dtype=np.uint8)
    data[::w] = np.arange(n, dtype=np.int64) % 26 + 65
    col = pa.Array.from_buffers(pa.string(), n, [None, pa.py_buffer(offs), pa.py_buffer(data)])
    sj = '{"type":"record","name":"O","fields":[%s]}' % ",".join('{"name":"c%d","type":"string"}' % i for i in range(cols))
    return sj, pa.record_batch({f"c{i}": col for i in range(cols)}), data


def test_ocf_past_4_gib_places_every_block_with_64_bit_offsets():
    """4 x 1.1 GB of string columns: a file just past 4 GiB, in blocks of about 400 MB, checked block by block in place."""
    n, w, cols, r = 1_075_000, 1000, 4, 100_000
    sj, batch, data = _big_string_batch(n, w, cols)
    sync = bytes(range(200, 216))
    f = pr.serialize_ocf(batch, sj, r, sync_marker=sync)
    head = len(O.ocf_header(sj, sync))
    row = cols * (2 + w)
    assert len(f) == head + sum(len(O.zz(c)) + len(O.zz(c * row)) + c * row + 16 for c in _counts(n, r)) > (4 << 30)
    buf = np.frombuffer(f, dtype=np.uint8)
    assert buf[:head].tobytes() == O.ocf_header(sj, sync)
    spans = O.block_spans(memoryview(f))
    assert [c for *_, c in spans] == _counts(n, r)
    txt = data.reshape(n, w)
    for j, (_, p, size, count) in enumerate(spans):
        assert size == count * row
        body = buf[p:p + size].reshape(count, cols, 2 + w)
        assert np.all(body[:, :, 0] == 0xD0) and np.all(body[:, :, 1] == 0x0F)        # zigzag(1000)
        for c in range(cols):
            assert np.array_equal(body[:, c, 2:], txt[j * r:j * r + count]), (j, c)
        assert buf[p + size:p + size + 16].tobytes() == sync
    assert spans[-1][1] + spans[-1][2] + 16 == len(f)


def test_ocf_block_over_2_gib_is_an_overflow_with_its_row():
    n, w = 1_100_000, 1000
    sj, batch, _ = _big_string_batch(n, w, 2)
    with pytest.raises(ValueError, match=r"block.*2 GiB \(row 0\)"):
        pr.serialize_ocf(batch, sj, n)
    f = pr.serialize_ocf(batch, sj, n // 2)                     # two blocks of 1.1 GB each fit
    assert [c for *_, c in O.block_spans(memoryview(f))] == [n // 2, n // 2]


# --------------------------------------------------------------------------------------------------------------------
# Confluent
# --------------------------------------------------------------------------------------------------------------------
def _header(sid):
    return b"\x00" + sid.to_bytes(4, "big")


@pytest.mark.parametrize("sid", [0, 1, (1 << 32) - 1])
def test_confluent_is_the_header_and_the_datum(sid):
    import workloads
    n = 3000
    sj, data, off = workloads.generate("kafka", n, seed=sid & 0xFF)
    recs = [bytes(data[off[i]:off[i + 1]]) for i in range(n)]
    batch = pr.deserialize_array(recs, sj)
    for k in (1, 3, 8):
        plain = pr.serialize_record_batch(batch, sj, k)
        out = pr.serialize_confluent(batch, sj, sid, k)
        assert [a.type for a in out] == [pa.binary()] * k and [len(a) for a in out] == [len(a) for a in plain]
        assert [[x.as_py() for x in a] for a in out] == [[_header(sid) + x.as_py() for x in a] for a in plain]
        msgs = [x.as_py() for a in out for x in a]
        got = pr.deserialize_confluent(msgs, sj, k, schema_id=sid)
        want = pr.deserialize_array_threaded(recs, sj, k)
        for g, w in zip(got, want):
            assert po.canon_diff(po.canon_from_batch(g), po.canon_from_batch(w)) is None
    h = pr._encode(pr.lib.rv_encode_host_confluent, batch, sj, 2, sid)
    try:
        assert pr.lib.rv_encoded_file(h, pr.ctypes.byref(pr.ctypes.c_void_p()), pr.ctypes.byref(pr.ctypes.c_int64())) == 9
    finally:
        pr.lib.rv_encoded_free(h)


@pytest.mark.parametrize("groups", ["1", "4"])
def test_confluent_row_groups(monkeypatch, groups):
    import workloads
    n, sid = 300_000, 0x01020304
    sj, data, off = workloads.generate("kafka", n, seed=12)
    batch = pr.decode_packed(data, off, n, sj, 1)[0]
    monkeypatch.setenv("RV_ENC_GROUPS", groups)
    for k in (1, 8):
        out, plain = pr.serialize_confluent(batch, sj, sid, k), pr.serialize_record_batch(batch, sj, k)
        for a, p in zip(out, plain):
            m = len(a)
            o = np.frombuffer(a.buffers()[1], dtype=np.int32)[:m + 1]
            po_ = np.frombuffer(p.buffers()[1], dtype=np.int32)[:m + 1]
            assert np.array_equal(o, po_ + 5 * np.arange(m + 1, dtype=np.int32))
            got = np.frombuffer(a.buffers()[2], dtype=np.uint8)[:o[-1]]
            pd = np.frombuffer(p.buffers()[2], dtype=np.uint8)
            heads = (o[:-1, None] + np.arange(5)).ravel()
            assert np.array_equal(got[heads], np.tile(np.frombuffer(_header(sid), np.uint8), m))
            mask = np.ones(len(got), dtype=bool)
            mask[heads] = False
            assert np.array_equal(got[mask], pd[:po_[-1]])


def test_confluent_headers_count_towards_the_chunk_limit():
    """Rows of 2 x (2 + 510) bytes: 2 097 151 of them are 1 KiB short of 2^31 bytes, and 10 MB over with the headers."""
    n, w = 2_097_151, 510
    sj, batch, _ = _big_string_batch(n, w, 2)
    plain = pr.serialize_record_batch(batch, sj, 1)
    assert np.frombuffer(plain[0].buffers()[1], dtype=np.int32)[n] == n * 2 * (2 + w) == (1 << 31) - 1024
    del plain
    with pytest.raises(ValueError, match=r"i32 offset overflow.*\(row 0\)"):
        pr.serialize_confluent(batch, sj, 1, 1)
    out = pr.serialize_confluent(batch, sj, 1, 2)
    assert [len(a) for a in out] == [n // 2, n - n // 2]
