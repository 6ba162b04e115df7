"""Avro single-object messages on the GPU (deserialize_single_object, rv_decode_*_single_object,
deserialize_single_object_versions, serialize_single_object).  A decode must equal, buffer for buffer, the oracle's decode
of the bare datums; a several-writer decode must equal the oracle's decode of each message resolved with its own writer
and re-encoded with the reader (tests/versions_cases.py); an encode must equal the header plus serialize_record_batch's
datum, byte for byte.  Headers are those of the restatement in tests/single_object.py."""
import ctypes
import json
import random

import numpy as np
import pyarrow as pa
import pytest

import pyruhvro_b200 as pr
import workloads
from oracle import pyoracle as po
from tests import resolution as RS
from tests import single_object as SO
from tests import versions_cases as VC
from tests.parity import assert_matches_oracle, gen_case

pytestmark = pytest.mark.gpu


@pytest.fixture(params=[1, 0], ids=["jit", "interp"])
def walker(request):
    pr.set_jit_enabled(request.param)
    yield request.param
    pr.set_jit_enabled(-1)


def _framed(sj, recs):
    fp = SO.fingerprint(sj)
    return [SO.frame(fp, r) for r in recs]


@pytest.mark.parametrize("n", [0, 1, 255, 256, 257, 383, 384, 385, 2500])
def test_counts(coracle, walker, n):
    sj, recs, data, off = gen_case(n + 17, n=n)
    msgs = _framed(sj, recs)
    for k in (1, 3, 8):
        got = pr.deserialize_single_object(msgs, sj, k)
        if n == 0:
            assert len(got) == 1 and got[0].num_rows == 0 and got[0].schema.equals(pr.Schema(sj).arrow_schema)
            continue
        assert_matches_oracle(coracle, got, sj, data, off, n, k)


def test_kafka_at_384_row_tiles(coracle):
    n = 20_011
    sj, data, off = workloads.generate("kafka", n, seed=9)
    msgs = _framed(sj, [data[off[i]:off[i + 1]].tobytes() for i in range(n)])
    pr.set_jit_enabled(1)
    try:
        for k in (1, 3, 8):
            pr.deserialize_single_object(msgs, sj, k)
            got = pr.deserialize_single_object(msgs, sj, k)
            assert pr.last_walker() == "jit" and pr.lib.rv_last_tile() == 384
            assert_matches_oracle(coracle, got, sj, data, off, n, k, full_validate=False)
    finally:
        pr.set_jit_enabled(-1)


def test_reader_schema_and_columns(walker):
    n = 3000
    v1, v2 = workloads.KAFKA_SCHEMA, RS.kafka_v2()
    _, data, off = workloads.generate("kafka", n, seed=5)
    bare = [data[off[i]:off[i + 1]].tobytes() for i in range(n)]
    msgs = _framed(v1, bare)
    cols1 = pr.Schema(v1).arrow_schema.names[1::2]
    cols2 = pr.Schema(v2).arrow_schema.names[::2]
    for kw in ({"reader_schema": v2}, {"columns": cols1}, {"reader_schema": v2, "columns": cols2}):
        want = pr.deserialize_array_threaded(bare, v1, 3, **kw)
        got = pr.deserialize_single_object(msgs, v1, 3, **kw)
        assert len(got) == len(want)
        for g, w in zip(got, want):
            assert g.equals(w)
    with pytest.raises(ValueError, match=r"single-object message.*record 0"):   # the header names v1, not v2
        pr.deserialize_single_object(msgs, v2, 1)


def test_device_entry_point(coracle, walker):
    import torch
    sj, recs, data, off = gen_case(77, n=2500)
    fd, fo = po.pack_records(_framed(sj, recs))
    dev = torch.device("cuda", 0)
    d_data = torch.zeros(len(fd) + 64, dtype=torch.uint8, device=dev)
    d_data[:len(fd)].copy_(torch.from_numpy(np.ascontiguousarray(fd)))
    d_off = torch.from_numpy(np.ascontiguousarray(fo, dtype=np.int64)).to(dev)
    s = pr._get_or_parse_schema(sj)
    for k in (1, 3):
        h = ctypes.c_void_p()
        pr._check(pr.lib.rv_decode_device_single_object(s.handle, d_data.data_ptr(), d_off.data_ptr(), len(recs), k,
                                                        torch.cuda.current_stream(dev).cuda_stream, ctypes.byref(h)))
        pr._check(pr.lib.rv_result_to_host(h.value))
        assert_matches_oracle(coracle, pr._export_batches(h.value, s), sj, data, off, len(recs), k)


def _damage(msg, how, fp):
    if how == "c3":
        return b"\xc4" + msg[1:]
    if how == "01":
        return msg[:1] + b"\x00" + msg[2:]
    if how == "fp":
        return msg[:5] + bytes([msg[5] ^ 0x01]) + msg[6:]
    if how == "short":
        return SO.header(fp)[:9]
    raise ValueError(how)


@pytest.mark.parametrize("k", [1, 3, 8])
def test_damaged_headers_at_tile_and_chunk_edges(walker, k):
    n = 2500
    sj, data, off = workloads.generate("kafka", n, seed=3)
    fp = SO.fingerprint(sj)
    msgs = _framed(sj, [data[off[i]:off[i + 1]].tobytes() for i in range(n)])
    cr = n // k
    edges = sorted(e for e in {255, 256, 383, 384, cr - 1, cr, n - 1} if e < n)
    for j, at in enumerate(edges):
        how = ("c3", "01", "fp", "short")[j % 4]
        bad = list(msgs)
        bad[at] = _damage(bad[at], how, fp)
        later = min(n - 1, at + 300)
        if later != at:
            bad[later] = _damage(bad[later], "short", fp)
        with pytest.raises(ValueError, match=r"single-object message.*\(record %d\)" % at):
            pr.deserialize_single_object(bad, sj, k)


# ---- several writers -------------------------------------------------------------------------------------------------
def _so_messages(rng, writers, seq, wide=False):
    """writers: {key: json}; seq: the key of every message -> (single-object messages, [(key, value)])"""
    parsed = {i: po.parse_schema(sj, wide=wide) for i, sj in writers.items()}
    fps = {i: SO.fingerprint(sj) for i, sj in writers.items()}
    vals = [(i, po.random_value(parsed[i], rng)) for i in seq]
    return [SO.frame(fps[i], po.encode_datum(parsed[i], v)) for i, v in vals], vals


def _distinct(writers):
    """Drop writers whose canonical form repeats an earlier one's (the registry refuses them)."""
    out, seen = {}, set()
    for i, sj in writers.items():
        fp = SO.fingerprint(sj)
        if fp not in seen:
            seen.add(fp)
            out[i] = sj
    return out


def _run_versions(coracle, writers, rj, seq, k, rng, wide=False):
    recs, vals = _so_messages(rng, writers, seq, wide)
    want = VC.expected(coracle, writers, rj, vals, k, wide)
    ws = list(writers.values())
    if isinstance(want, tuple):
        with pytest.raises(ValueError, match=r"\(record %d\)" % want[1]):
            pr.deserialize_single_object_versions(recs, ws, rj, k)
        return
    got = pr.deserialize_single_object_versions(recs, ws, rj, k)
    for b in got:
        assert b.schema.equals(pr.Schema(rj).arrow_schema)
        b.validate(full=not wide)
    VC.compare(got, want, rj)


@pytest.mark.parametrize("seed", range(8))
def test_several_writers(coracle, walker, seed):
    rng = random.Random(seed * 211 + 1)
    rj, writers = VC.writer_chain(rng, wide=seed >= 6)
    writers = dict(list(_distinct(writers).items())[:2 + seed % 3])   # 2-4 writers
    k = [1, 3, 8][seed % 3]
    n = rng.choice([257, 385, 600])
    kind = ["alternate", "runs"][seed % 2]
    _run_versions(coracle, writers, rj, VC.mix(rng, writers, n, kind, k), k, rng, wide=seed >= 6)


def test_several_writers_errors(walker):
    rng = random.Random(4)
    rj, ws = RS.kafka_v2(), [workloads.KAFKA_SCHEMA, RS.kafka_v2()]
    writers = {0: ws[0], 1: ws[1]}
    recs, _ = _so_messages(rng, writers, [i % 2 for i in range(1200)])
    other = SO.fingerprint(json.dumps({"type": "record", "name": "X", "fields": [{"name": "a", "type": "int"}]}))
    bad = list(recs)
    bad[700] = SO.frame(other, recs[700][10:])
    bad[900] = b"\xc3\x01"
    with pytest.raises(ValueError, match=r"schema fingerprint 0x%016x is not registered \(record 700\)" % other):
        pr.deserialize_single_object_versions(bad, ws, rj, 3)
    bad = list(recs)
    bad[300] = b"\xc3\x02" + recs[300][2:]
    with pytest.raises(ValueError, match=r"single-object message.*\(record 300\)"):
        pr.deserialize_single_object_versions(bad, ws, rj, 3)


def test_one_fingerprint_takes_the_direct_path(coracle):
    rng = random.Random(8)
    rj, ws = RS.kafka_v2(), [workloads.KAFKA_SCHEMA, RS.kafka_v2()]
    writers = {0: ws[0], 1: ws[1]}
    recs, vals = _so_messages(rng, writers, [0] * 1500)
    want = VC.expected(coracle, writers, rj, vals, 3)
    got = pr.deserialize_single_object_versions(recs, ws, rj, 3)
    assert pr.last_versions_timings()["take"] == 0.0
    VC.compare(got, want, rj)


# ---- encode ----------------------------------------------------------------------------------------------------------
def _check_encode(batch, sj, k):
    fp_hdr = SO.header(SO.fingerprint(sj))
    got = pr.serialize_single_object(batch, sj, k)
    want = pr.serialize_record_batch(batch, sj, k)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.type == pa.binary() and len(g) == len(w)
        assert g.to_pylist() == [fp_hdr + d for d in w.to_pylist()]
    return got


@pytest.mark.parametrize("seed", range(6))
def test_encode_random_schemas_at_chunk_edges(seed):
    sj, recs, data, off = gen_case(300 + seed, n=[1, 255, 256, 257, 513, 1000][seed])
    batch = pr.deserialize_array(recs, sj)
    n = len(recs)
    for k in sorted({1, 2, 3, max(1, n // 256), n}):
        got = _check_encode(batch, sj, k)
        back = pr.deserialize_single_object([m for a in got for m in a.to_pylist()], sj, 1)[0]
        assert back.equals(batch)


def test_encode_row_groups_round_trip():
    n = 1 << 18
    sj, data, off = workloads.generate("kafka", n + 123, seed=2)
    batch = pr.decode_packed(data, off, n + 123, sj, 1)[0]
    got = _check_encode(batch, sj, 8)
    msgs = [m for a in got for m in a.to_pylist()]
    back = pr.deserialize_single_object(msgs, sj, 1)[0]
    assert back.equals(batch)


# ---- bench scale -----------------------------------------------------------------------------------------------------
def test_kafka_10m_parity(coracle):
    import os
    n = 10_000_000
    sj, data, off = workloads.generate("kafka", n, seed=42)
    batch_src = pr.decode_packed(data, off, n, sj, 8)
    msgs = pa.concat_arrays([a.cast(pa.large_binary()) for b in batch_src for a in pr.serialize_single_object(b, sj, 1)])
    md, mo, _ = pr._packed_view(msgs)
    s = pr._get_or_parse_schema(sj)
    h = ctypes.c_void_p()
    pr._check(pr.lib.rv_decode_host_single_object(s.handle, md.ctypes.data, np.ascontiguousarray(mo).ctypes.data, n, 8, ctypes.byref(h)))
    got = pr._export_batches(h.value, s)
    want = coracle.decode_threaded_packed(sj, data, off, n, 8, threads=os.cpu_count() or 4)
    assert len(got) == len(want)
    for i, (b, w) in enumerate(zip(got, want)):
        d = po.canon_diff(po.canon_from_batch(b), w, f"batch[{i}]")
        assert d is None, d
