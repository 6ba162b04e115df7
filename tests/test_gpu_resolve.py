"""Schema resolution on the GPU: every entry point with `reader_schema=` (and `columns=`), both walkers, against the
oracle's decode of the converted, re-encoded values (tests/resolution.py)."""
import ctypes
import json
import random
import re

import numpy as np
import pyarrow as pa
import pytest

import pyruhvro_b200 as pr
from oracle import pyoracle as po
from tests import mutation as M
from tests import resolution as RS
from tests.parity import expected_schema, expected_schema_wide

pytestmark = pytest.mark.gpu


class _GpuError(Exception):
    def __init__(self, status, message):
        super().__init__(message)
        m = re.search(r"\(record (-?\d+)\)", message)
        self.status, self.category, self.record = status, po.ERR_NAMES.get(status, str(status)), int(m.group(1)) if m else -1


def _gpu_host(s, data, off, n, k):
    data = np.ascontiguousarray(data, dtype=np.uint8)
    off = np.ascontiguousarray(off, dtype=np.int64)
    h = ctypes.c_void_p()
    rc = pr.lib.rv_decode_host(s.handle, data.ctypes.data if data.size else None, off.ctypes.data, n, k, ctypes.byref(h))
    if rc:
        raise _GpuError(rc, pr._last_error())
    return pr._export_batches(h.value, s)


@pytest.fixture(params=["jit", "interp"])
def walker(request):
    pr.set_jit_enabled(1 if request.param == "jit" else 0)
    yield request.param
    pr.set_jit_enabled(-1)


def _assert_batches(got, want, rj, wide=False, cols=None, full_validate=True):
    exp = expected_schema_wide(rj) if wide else expected_schema(rj)
    idx = list(range(len(exp))) if cols is None else [exp.names.index(c) for c in cols]
    exp = pa.schema([exp.field(i) for i in idx])
    assert len(got) == len(want)
    for i, (b, w) in enumerate(zip(got, want)):
        assert b.schema.equals(exp, check_metadata=True), (b.schema, exp)
        if full_validate:
            b.validate(full=not wide)   # (bytes read as string are not checked for UTF-8, as in any decode)
        d = po.canon_diff(po.canon_from_batch(b), [w[j] for j in idx], f"batch[{i}]")
        assert d is None, d


def _case(seed, n, wide):
    rng = random.Random(seed)
    wj = po.random_schema_json(rng, wide=wide)
    rj = RS.random_evolution(rng, wj, wide=wide)
    ws = po.parse_schema(wj, wide=wide)
    vals = [po.random_value(ws, rng) for _ in range(n)]
    data, off = po.pack_records([po.encode_datum(ws, v) for v in vals])
    return wj, rj, vals, data, off


@pytest.mark.parametrize("n", [1, 255, 256, 257, 383, 384, 385, 2500])
def test_gpu_random_evolutions(coracle, walker, n):
    for i, k in enumerate((1, 3, 8)):
        wide = i == 2
        wj, rj, vals, data, off = _case(n * 10 + i, n, wide)
        s = pr.Schema(wj).read_as(rj)
        got = _gpu_host(s, data, off, n, k)
        assert pr.last_walker() == walker
        _assert_batches(got, RS.expected_batches(coracle, wj, rj, vals, k, wide=wide), rj, wide)


def _kafka_values(n, seed):
    import workloads
    ws = po.parse_schema(workloads.KAFKA_SCHEMA)
    rng = random.Random(seed)
    vals = [po.random_value(ws, rng) for _ in range(n)]
    return workloads.KAFKA_SCHEMA, vals, [po.encode_datum(ws, v) for v in vals]


def test_gpu_every_entry_point(coracle):
    from tests.ocf_files import ocf_file
    from tests.test_gpu_framed import _confluent
    W, vals, recs = _kafka_values(3000, 1)
    data, off = po.pack_records(recs)
    n = len(recs)
    for rj in (RS.kafka_v2(), RS.kafka_v2(("A", "B"), "A")):
        want = {k: RS.expected_batches(coracle, W, rj, vals, k) for k in (1, 3)}
        for cols in (None, ["source", "age", "address"], ["created_at"]):
            kw = dict(reader_schema=rj, columns=cols)
            _assert_batches([pr.deserialize_array(recs, W, **kw)], want[1], rj, cols=cols)
            _assert_batches(pr.deserialize_array_threaded(recs, W, 3, **kw), want[3], rj, cols=cols)
            _assert_batches(pr.deserialize_array_threaded_spawn(recs, W, 3, **kw), want[3], rj, cols=cols)
            _assert_batches(pr.deserialize_arrow_array(pa.array(recs, pa.binary()), W, 3, **kw), want[3], rj, cols=cols)
            _assert_batches(pr.decode_packed(data, off, n, W, 3, **kw), want[3], rj, cols=cols)
            _assert_batches(pr.deserialize_confluent(_confluent(recs, 9), W, 3, schema_id=9, **kw), want[3], rj, cols=cols)
            _assert_batches(pr.deserialize_ocf(ocf_file(W, recs, [1, 300, 1000], random.Random(1)), 3, **kw), want[3], rj, cols=cols)
    with pytest.raises(ValueError, match="schema resolution"):
        pr.deserialize_array(recs[:3], W, reader_schema=json.dumps({"type": "record", "name": "User", "fields": [
            {"name": "nope", "type": "int"}]}))
    with pytest.raises(ValueError, match="no top-level field"):
        pr.deserialize_ocf(ocf_file(W, recs[:10], [10], random.Random(1)), 1, reader_schema=RS.kafka_v2(), columns=["phone_numbers"])


def test_gpu_kafka_v2_takes_384_row_tiles():
    W, vals, recs = _kafka_values(5000, 2)
    s = pr.Schema(W).read_as(RS.kafka_v2())
    assert pr.lib.rv_schema_max_tile(s.handle) == 384
    pr.set_jit_enabled(1)
    try:
        pr.deserialize_array_threaded(recs, W, 2, reader_schema=RS.kafka_v2())
        assert pr.last_walker() == "jit" and pr.lib.rv_last_tile() == 384
    finally:
        pr.set_jit_enabled(-1)


@pytest.mark.parametrize("items", [(0, 4), (0, 9)])
def test_gpu_defaults_inside_list_items(coracle, walker, items):
    """Item-parallel (at most four items per record) and per-lane (more) list warps whose items gain default fields."""
    wj = json.dumps({"type": "record", "name": "T", "fields": [
        {"name": "xs", "type": {"type": "array", "items": {"type": "record", "name": "It", "fields": [
            {"name": "a", "type": "int"}, {"name": "b", "type": "string"}]}}},
        {"name": "m", "type": {"type": "map", "values": "long"}}]})
    rj = json.dumps({"type": "record", "name": "T", "fields": [
        {"name": "m", "type": {"type": "map", "values": "double"}},
        {"name": "xs", "type": {"type": "array", "items": {"type": "record", "name": "It", "fields": [
            {"name": "tag", "type": "string", "default": "dflt-tag"}, {"name": "b", "type": "string"},
            {"name": "a", "type": ["null", "long"]}, {"name": "z", "type": ["null", "string"], "default": None},
            {"name": "w", "type": "float", "default": 2.5}]}}}]})
    rng = random.Random(items[1])
    vals = [{"xs": [{"a": rng.randint(-99, 99), "b": "s" * rng.randint(0, 9)} for _ in range(rng.randint(*items))],
             "m": [("k%d" % j, rng.randint(-5, 5)) for j in range(rng.randint(0, 3))]} for _ in range(1000)]
    ws = po.parse_schema(wj)
    data, off = po.pack_records([po.encode_datum(ws, v) for v in vals])
    for k in (1, 3):
        _assert_batches(_gpu_host(pr.Schema(wj).read_as(rj), data, off, len(vals), k), RS.expected_batches(coracle, wj, rj, vals, k), rj)


def test_gpu_null_defaults_of_every_kind(coracle, walker):
    """Optional reader-only fields of every kind whose default is null (records, lists, unions, fixed, decimal, uuid; at
    the top level and inside list items): buffer for buffer a null of the reader's type."""
    def rec(*fields, name="R"):
        return json.dumps({"type": "record", "name": name, "fields": list(fields)})

    def fld(name, t, **kw):
        return dict({"name": name, "type": t}, **kw)

    item_w = {"type": "record", "name": "It", "fields": [fld("q", "string")]}
    item_r = {"type": "record", "name": "It", "fields": [
        fld("n", ["null", {"type": "record", "name": "NK", "fields": [fld("k", "boolean")]}], default=None), fld("q", "string")]}
    wj = rec(fld("a", "int"), fld("xs", {"type": "array", "items": item_w}))
    nr = {"type": "record", "name": "NR", "fields": [fld("x", "int"), fld("y", ["null", "string"]), fld("z", {"type": "array", "items": "long"})]}
    rj = rec(fld("r", ["null", nr], default=None), fld("l", ["null", {"type": "array", "items": "string"}], default=None),
             fld("xs", {"type": "array", "items": item_r}), fld("a", "long"), fld("u", ["null", "string", "int"], default=None))
    rjw = rec(fld("a", "int"), fld("f", ["null", {"type": "fixed", "name": "F", "size": 4}], default=None),
              fld("d", ["null", {"type": "bytes", "logicalType": "decimal", "precision": 9, "scale": 2}], default=None),
              fld("g", ["null", {"type": "string", "logicalType": "uuid"}], default=None), fld("xs", {"type": "array", "items": item_w}))
    rng = random.Random(9)
    ws = po.parse_schema(wj)
    for n, k in ((1, 1), (385, 3), (2500, 8)):
        vals = [po.random_value(ws, rng) for _ in range(n)]
        data, off = po.pack_records([po.encode_datum(ws, v) for v in vals])
        _assert_batches(_gpu_host(pr.Schema(wj).read_as(rj), data, off, n, k), RS.expected_batches(coracle, wj, rj, vals, k), rj)
        _assert_batches(_gpu_host(pr.Schema(wj).read_as(rjw), data, off, n, k), RS.expected_batches(coracle, wj, rjw, vals, k, wide=True),
                        rjw, wide=True)


def test_gpu_device_resident_kafka_2m_twice(coracle):
    """2 M Kafka records decoded as Kafka v2 straight from device memory, twice: the second call plans from the first
    (one pass), and every buffer matches the oracle.  (20 000 distinct records, repeated.)"""
    import torch
    W, vals, recs = _kafka_values(20_000, 3)
    reps = 100
    d1, o1 = po.pack_records(recs)
    data = np.tile(d1, reps)
    off = np.concatenate([o1[:-1] + r * o1[-1] for r in range(reps)] + [np.array([o1[-1] * reps])]).astype(np.int64)
    n = len(off) - 1
    rj = RS.kafka_v2()
    ws, rs = po.parse_schema(W), po.parse_schema(rj)
    meta = RS.ReaderMeta(rj)
    rd, ro = po.pack_records([po.encode_datum(rs, RS.resolve_value(ws, rs, v, meta)) for v in vals])
    rdata = np.tile(rd, reps)
    roff = np.concatenate([ro[:-1] + r * ro[-1] for r in range(reps)] + [np.array([ro[-1] * reps])]).astype(np.int64)
    want = coracle.decode_threaded_packed(rj, rdata, roff, n, 4, threads=8)
    dev = torch.device("cuda", 0)
    d_data = torch.zeros(len(data) + 64, dtype=torch.uint8, device=dev)
    d_data[:len(data)] = torch.from_numpy(data).to(dev)
    d_off = torch.from_numpy(off).to(dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    s = pr._get_or_parse_schema(W, None, rj)
    for call in range(2):
        h = ctypes.c_void_p()
        pr._check(pr.lib.rv_decode_device(s.handle, d_data.data_ptr(), d_off.data_ptr(), n, 4, stream, ctypes.byref(h)))
        if call == 1:
            assert pr.lib.rv_last_passes() == 1
        pr._check(pr.lib.rv_result_to_host(h.value))
        got = pr._export_batches(h.value, s)
    _assert_batches(got, want, rj, full_validate=False)


def test_gpu_unmapped_enum_reports_the_lowest_record(walker):
    W, vals, recs = _kafka_values(4000, 4)
    rj = RS.kafka_v2(("A", "B"))   # no default: a "C" cannot be read
    ws = po.parse_schema(W)
    c_rows = [i for i, v in enumerate(vals) if v["class"] == 2]
    for first in (3999, 2100, 700):   # only records >= `first` keep their "C"
        fixed = [po.encode_datum(ws, dict(v, **{"class": 0})) if (v["class"] == 2 and i < first) else recs[i] for i, v in enumerate(vals)]
        data, off = po.pack_records(fixed)
        want = min(i for i in c_rows if i >= first) if any(i >= first for i in c_rows) else None
        for k in (1, 3, 8):
            if want is None:
                _gpu_host(pr.Schema(W).read_as(rj), data, off, len(fixed), k)
                continue
            with pytest.raises(_GpuError) as ei:
                _gpu_host(pr.Schema(W).read_as(rj), data, off, len(fixed), k)
            assert (ei.value.status, ei.value.record) == (6, want), str(ei.value)
            assert "neither a reader symbol nor a reader default" in str(ei.value)


@pytest.mark.timeout(900, method="thread")
def test_gpu_damaged_inputs(coracle):
    seen = {"decoded": 0, "error": 0}
    for seed in range(100):
        rng = random.Random(seed + 5000)
        wj = po.random_schema_json(rng)
        rj = RS.random_evolution(rng, wj)
        ws = po.parse_schema(wj)
        recs = M.damage(rng, [po.encode_datum(ws, po.random_value(ws, rng)) for _ in range(rng.choice([3, 40, 257, 300]))])
        data, off = po.pack_records(recs)
        k = rng.choice([1, 2, 3, 8])
        want = M.expected(coracle, wj, recs)
        if seed % 2:
            pr.set_jit_enabled(0)
        try:
            _gpu_host(pr.Schema(wj).read_as(rj), data, off, len(recs), k)
        except _GpuError as e:
            assert (e.category, e.record) == want, (wj, rj)
            seen["error"] += 1
            continue
        finally:
            pr.set_jit_enabled(-1)
        assert want is None or want[0] == "overflow", want
        seen["decoded"] += 1
    assert seen["decoded"] > 5 and seen["error"] > 5


def test_gpu_resolved_gather_on_one_device(coracle):
    import torch
    from pyruhvro_b200 import distributed as D
    from tests.test_gpu_gather import _split, _to_device
    W, vals, recs = _kafka_values(30_000, 6)
    data, off = po.pack_records(recs)
    rj = RS.kafka_v2(("A", "B"), "A")
    L = D._lib()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    handles, g = [], ctypes.c_void_p()
    try:
        for d, o in _split(data, off, [9_984, 10_240, 9_776]):
            d_data, d_off = _to_device(d, o, dev)
            s, h = D.decode_sharded(W, d_data, d_off, len(o) - 1, 1, reader_schema=rj)
            handles.append(h)
        m = int(L.rv_gather_meta_len(s.handle))
        metas = np.zeros((len(handles), max(m, 1)), dtype=np.int64)
        for r, h in enumerate(handles):
            pr._check(L.rv_result_gather_meta(h, 0, metas[r].ctypes.data, m))
        pr._check(L.rv_gather_plan(s.handle, metas.ctypes.data, len(handles), ctypes.byref(g)))
        assert L.rv_gather_num_groups(g) == 1
        base = ctypes.c_void_p()
        pr._check(L.rv_gather_alloc(g, 0, stream, ctypes.byref(base)))
        for r, h in enumerate(handles):
            pr._check(L.rv_gather_push(g, 0, r, h, 0, base, stream))
        res = ctypes.c_void_p()
        pr._check(L.rv_gather_finish(g, 0, ctypes.byref(res)))
        pr._check(L.rv_result_to_host(res))
        got = pr._export_batches(res.value, s)
    finally:
        L.rv_gather_free(g)
        for h in handles:
            L.rv_result_free(h)
    _assert_batches(got, RS.expected_batches(coracle, W, rj, vals, 1), rj)
