"""Permissive decodes on the device (errors="null", Schema.permissive): the cases of tests/test_permissive.py through the
product with both walkers, k = 1, 3 and 8, the host and device-resident entry points, every Python entry point, and a
bench-scale Kafka input with every 1000th message damaged.  The contract is stated in tests/permissive_cases.py."""
import ctypes
import json

import numpy as np
import pyarrow as pa
import pytest

import pyruhvro_b200 as pr
from oracle import pyoracle as po
from tests import mutation as M
from tests import permissive_cases as PC
from tests.test_permissive import PLACE_SCHEMA, PLACEMENTS, fld, place_records, rec

pytestmark = pytest.mark.gpu


@pytest.fixture(params=["jit", "interp"])
def walker(request):
    pr.set_jit_enabled(1 if request.param == "jit" else 0)
    yield request.param
    pr.set_jit_enabled(-1)


PROJ_SCHEMA = rec(fld("a", "int"), fld("b", "string"), fld("c", "boolean"))
ENUM_WRITER = rec(fld("a", "int"), fld("e", {"type": "enum", "name": "E", "symbols": ["A", "B", "C"]}))
ENUM_READER = rec(fld("e", {"type": "enum", "name": "E", "symbols": ["B", "A"]}), fld("a", "long"), fld("d", "string", default="z"))


def jit_permissive():
    """(schema, columns, reader) of every permissive handle these tests decode with the generated walker
    (tools/warm_jit_cache.py compiles them ahead)."""
    import workloads
    from tests.parity import gen_case
    out = [(M.damaged_case(seed)[0], None, None) for seed in range(6)]
    out += [(M.forged_case(seed)[0], None, None) for seed in range(6)]
    out += [(gen_case(seed, n=1)[0], None, None) for seed in range(3)]
    out += [(PLACE_SCHEMA, None, None), (WIDE_PLACE_SCHEMA, None, None), (PROJ_SCHEMA, ("b", "a"), None), (ENUM_WRITER, None, ENUM_READER),
            (workloads.KAFKA_SCHEMA, None, None)]
    return out


def bad_list(bad: pa.RecordBatch):
    assert bad.schema.names == ["record", "status", "error"]
    assert bad.schema.field("record").type == pa.int64() and bad.schema.field("status").type == pa.int32()
    return list(zip(bad.column(0).to_pylist(), bad.column(1).to_pylist()))


def host(sj, recs, k, **kw):
    data, off = po.pack_records(recs)
    batches, bad = pr.decode_packed(data, off, len(recs), sj, k, errors="null", **kw)
    return batches, bad_list(bad), bad


def device(sj, recs, k):
    import torch
    data, off = po.pack_records(recs)
    s = pr._get_or_parse_schema(sj, permissive=True)
    total = int(off[len(recs)])
    d_data = torch.zeros(total + 64, dtype=torch.uint8, device="cuda")
    d_data[:total].copy_(torch.from_numpy(np.array(data[:total], dtype=np.uint8)))
    d_off = torch.from_numpy(np.ascontiguousarray(off, dtype=np.int64)).cuda()
    h = ctypes.c_void_p()
    pr._check(pr.lib.rv_decode_device(s.handle, d_data.data_ptr(), d_off.data_ptr(), len(recs), k,
                                      torch.cuda.current_stream().cuda_stream, ctypes.byref(h)))
    pr._check(pr.lib.rv_result_to_host(h))
    batches, bad = pr._export_batches(h.value, s, True)
    return batches, bad_list(bad)


@pytest.mark.parametrize("k", [1, 3, 8])
@pytest.mark.parametrize("seed", range(6))
def test_gpu_damaged_random(coracle, walker, seed, k):
    sj, recs, _ = M.damaged_case(seed)
    exp = PC.Expected(coracle, sj, recs, k)
    batches, bad, report = host(sj, recs, k)
    exp.check(batches, bad)
    assert all(t and "(record" not in t for t in report.column(2).to_pylist())
    batches, bad = device(sj, recs, k)
    exp.check(batches, bad)


@pytest.mark.parametrize("seed", range(6))
def test_gpu_forged_varints(coracle, walker, seed):
    sj, recs, k = M.forged_case(seed)
    exp = PC.Expected(coracle, sj, recs, k)
    batches, bad, _ = host(sj, recs, k)
    exp.check(batches, bad)


# nine streams or more: the generated walker takes 384-row tiles (engine.cu choose_tile)
WIDE_PLACE_SCHEMA = json.dumps(dict(json.loads(PLACE_SCHEMA), fields=json.loads(PLACE_SCHEMA)["fields"] + [fld("c2", "string"), fld("c3", "string")]))


def wide_place_records(n, bad):
    tail = po.parse_schema(rec(fld("c2", "string"), fld("c3", "string")))
    out = []
    for i, r in enumerate(place_records(n, set())):
        r = r + po.encode_datum(tail, {"c2": "x" * (i % 3), "c3": "y"})
        out.append(r[:1] if i in bad else r)
    return out


@pytest.mark.parametrize("schema", ["256", "384"])
@pytest.mark.parametrize("where", sorted(PLACEMENTS))
def test_gpu_placements(coracle, walker, where, schema):
    bad = set(PLACEMENTS[where])
    sj, recs = (PLACE_SCHEMA, place_records(1000, bad)) if schema == "256" else (WIDE_PLACE_SCHEMA, wide_place_records(1000, bad))
    exp = PC.Expected(coracle, sj, recs, 1)
    assert [i for i, _ in exp.bad] == sorted(bad)
    batches, got, _ = host(sj, recs, 1)
    exp.check(batches, got)
    if walker == "jit":
        assert pr.last_walker() == "jit" and pr.lib.rv_last_tile() == int(schema)


def test_gpu_chunk_entirely_bad(coracle, walker):
    recs = place_records(900, set(range(300, 600)))
    exp = PC.Expected(coracle, PLACE_SCHEMA, recs, 3)
    batches, bad, _ = host(PLACE_SCHEMA, recs, 3)
    exp.check(batches, bad)
    batches, bad = device(PLACE_SCHEMA, recs, 3)
    exp.check(batches, bad)


def test_gpu_projection_and_resolution(coracle, walker):
    sj = PROJ_SCHEMA
    s = po.parse_schema(sj)
    recs = [po.encode_datum(s, {"a": i, "b": "x" * (i % 5), "c": True}) for i in range(300)]
    for i in (3, 100, 299):
        recs[i] = recs[i][:-1] + b"\x07"
    exp = PC.Expected(coracle, sj, recs, 2)
    batches, bad, report = host(sj, recs, 2, columns=["b", "a"])
    exp.check(batches, bad, columns=["b", "a"])
    assert report.column(2).to_pylist() == ["invalid boolean byte"] * 3
    writer, reader = ENUM_WRITER, ENUM_READER
    ws = po.parse_schema(writer)
    recs = [po.encode_datum(ws, {"a": i, "e": i % 3}) for i in range(600)]
    batches, bad, report = host(writer, recs, 3, reader_schema=reader)
    assert bad == [(i, 6) for i in range(600) if i % 3 == 2]
    assert set(report.column(2).to_pylist()) == {"enum symbol has neither a reader symbol nor a reader default"}
    got = pa.Table.from_batches(batches).to_pydict()
    assert got["a"] == [None if i % 3 == 2 else i for i in range(600)]
    assert got["e"] == [None if i % 3 == 2 else "AB"[i % 3] for i in range(600)]
    assert got["d"] == [None if i % 3 == 2 else "z" for i in range(600)]


def test_gpu_framing(coracle, walker):
    plain = place_records(600, set())
    msgs = [b"\x00\x00\x00\x00\x07" + r for r in plain]
    msgs[5] = b"\x01" + msgs[5][1:]
    msgs[256], msgs[257] = b"\x00\x00", b""
    msgs[590] = b"\x00\x00\x00\x00\x08" + plain[590]
    for k in (1, 3, 8):
        batches, bad = pr.deserialize_confluent(msgs, PLACE_SCHEMA, k, schema_id=7, errors="null")
        assert bad_list(bad) == [(5, 12), (256, 12), (257, 12), (590, 12)]
        verdicts = [None] * len(plain)
        for i, _ in bad_list(bad):
            verdicts[i] = "frame"
        PC.Expected(coracle, PLACE_SCHEMA, plain, k, verdicts=verdicts).check(batches, bad_list(bad))
    fp = pr.Schema(PLACE_SCHEMA).fingerprint
    hdr = b"\xc3\x01" + fp.to_bytes(8, "little")
    msgs = [hdr + r for r in plain]
    msgs[0] = b"\xc3\x01" + (fp ^ 1).to_bytes(8, "little") + plain[0]
    msgs[300] = hdr[:9]
    msgs[599] = hdr + plain[599][:1]
    batches, bad = pr.deserialize_single_object(msgs, PLACE_SCHEMA, 3, errors="null")
    assert bad_list(bad) == [(0, 12), (300, 12), (599, 1)]
    assert bad.column(2).to_pylist()[0].startswith("single-object message")
    verdicts = [None] * len(plain)
    verdicts[0] = verdicts[300] = "frame"
    verdicts[599] = "eof"
    PC.Expected(coracle, PLACE_SCHEMA, plain, 3, verdicts=verdicts).check(batches, bad_list(bad))


def test_gpu_python_surface(coracle):
    recs = place_records(700, {1, 400, 699})
    exp = PC.Expected(coracle, PLACE_SCHEMA, recs, 3)
    b, bad = pr.deserialize_array(recs, PLACE_SCHEMA, errors="null")
    PC.Expected(coracle, PLACE_SCHEMA, recs, 1).check([b], bad_list(bad))
    for fn in (pr.deserialize_array_threaded, pr.deserialize_array_threaded_spawn):
        batches, bad = fn(recs, PLACE_SCHEMA, 3, errors="null")
        exp.check(batches, bad_list(bad))
    batches, bad = pr.deserialize_arrow_array(pa.array(recs, pa.binary()), PLACE_SCHEMA, 3, errors="null")
    exp.check(batches, bad_list(bad))
    assert bad.column(2).to_pylist() == ["unexpected end of buffer"] * 3
    assert isinstance(pr.deserialize_array_threaded(recs[2:5], PLACE_SCHEMA, 1), list)   # errors="raise" is unchanged
    with pytest.raises(ValueError, match=r"\(record 1\)"):
        pr.deserialize_array_threaded(recs, PLACE_SCHEMA, 3)


def test_gpu_clean_input_is_read_as(coracle, walker):
    for seed in range(3):
        from tests.parity import gen_case
        sj, recs, data, off = gen_case(seed, n=700)
        batches, bad = pr.decode_packed(data, off, len(recs), sj, 3, errors="null")
        assert bad.num_rows == 0
        want = pr.decode_packed(data, off, len(recs), sj, 3, reader_schema=PC.optional_json(sj))
        for b, w in zip(batches, want):
            assert b.schema.equals(w.schema)
            assert po.canon_diff(po.canon_from_batch(b), po.canon_from_batch(w)) is None


def test_gpu_overflow_stays_fatal():
    sj = rec(fld("l", {"type": "array", "items": "null"}))
    big = po.zigzag_bytes(2 ** 30 + 1) + b"\x00"
    data, off = po.pack_records([big, b"", big])
    with pytest.raises(ValueError, match="overflow"):
        pr.decode_packed(data, off, 3, sj, 1, errors="null")


def _union_type_ids(col):
    return np.concatenate([np.frombuffer(c.buffers()[1], dtype=np.int8)[c.offset:c.offset + len(c)] for c in col.chunks])


def _check_kafka(strict, batches, bad, damaged, status):
    n = strict.num_rows
    assert bad.column(0).to_numpy().tolist() == damaged.tolist()
    assert set(bad.column(1).to_pylist()) == {status}
    assert [b.num_rows for b in batches] == [b.num_rows for b in strict.to_batches()]
    got = pa.Table.from_batches(batches)
    good = np.ones(n, dtype=bool)
    good[damaged] = False
    for name in strict.column_names:
        g, w = got.column(name), strict.column(name)
        if pa.types.is_union(g.type):   # no validity: type id 0 at a bad row
            gt, wt = _union_type_ids(g), _union_type_ids(w)
            assert np.array_equal(gt[good], wt[good]) and not gt[~good].any(), name
            continue
        if pa.types.is_map(g.type):     # no validity: an empty map at a bad row
            assert g.filter(pa.array(good)).equals(w.filter(pa.array(good))), name
            o = g.filter(pa.array(~good)).combine_chunks().offsets.to_numpy()
            assert o[0] == o[-1], name
            continue
        assert g.filter(pa.array(good)).equals(w.filter(pa.array(good))), name
        assert g.filter(pa.array(~good)).null_count == len(damaged), name


def test_gpu_kafka_bench_scale():
    """10 M Kafka messages with every 1000th damaged: Confluent frames with a wrong magic byte (RV_ERR_FRAME), and plain
    datums replaced by empty messages (RV_ERR_EOF).  Good rows equal the strict decode of the undamaged input."""
    import workloads
    n, k = 10_000_000, 8
    sj, data, off = workloads.generate("kafka", n, seed=42)
    data, off = np.ascontiguousarray(data), np.ascontiguousarray(off, dtype=np.int64)
    strict = pa.Table.from_batches(pr.decode_packed(data, off, n, sj, k))
    damaged = np.arange(0, n, 1000)
    msgs, moff = frame_kafka(data, off, damaged)
    batches, bad = pr.decode_packed(msgs, moff, n, sj, k, pr.Framing(5, 1, -1), errors="null")
    _check_kafka(strict, batches, bad, damaged, 12)
    cut, coff = empty_messages(data, off, damaged)
    batches, bad = pr.decode_packed(cut, coff, n, sj, k, errors="null")
    _check_kafka(strict, batches, bad, damaged, 1)


def frame_kafka(data, off, wrong_magic):
    """Confluent frames (schema id 7) around each datum; the messages `wrong_magic` start with 0x01."""
    lens = np.diff(off)
    moff = np.concatenate([[0], np.cumsum(lens + 5)]).astype(np.int64)
    out = np.zeros(int(moff[-1]), dtype=np.uint8)
    starts = moff[:-1]
    out[starts + 4] = 7
    out[np.repeat(starts + 5 - off[:-1], lens) + np.arange(int(off[0]), int(off[-1]))] = data[int(off[0]):int(off[-1])]
    out[starts[wrong_magic]] = 1
    return out, moff


def empty_messages(data, off, which):
    """The packed datums with the messages `which` made empty."""
    lens = np.diff(off)
    keep = np.ones(len(lens), dtype=bool)
    keep[which] = False
    out = np.ascontiguousarray(data[int(off[0]):int(off[-1])][np.repeat(keep, lens)])
    return out, np.concatenate([[0], np.cumsum(np.where(keep, lens, 0))]).astype(np.int64)
