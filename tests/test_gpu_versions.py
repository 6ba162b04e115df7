"""deserialize_confluent_versions / rv_decode_*_versions on the GPU: the matrix of tests/test_versions.py through both
walkers and through the device entry point on torch-allocated input, two threads sharing one registry, an output column
that overflows only when its writers' parts are added, and 10 M Kafka messages of two schema versions."""
import ctypes
import json
import random
import threading

import numpy as np
import pytest

import pyruhvro_b200 as pr
import workloads
from oracle import pyoracle as po
from tests import resolution as RS
from tests import versions_cases as VC

pytestmark = pytest.mark.gpu
MIXES = ["runs", "alternate", "absent", "single"]


@pytest.fixture(params=[1, 0], ids=["jit", "interp"])
def walker(request):
    pr.set_jit_enabled(request.param)
    yield request.param
    pr.set_jit_enabled(-1)


def _device_decode(writers, rj, recs, k, columns=None):
    import torch
    data, off = po.pack_records(recs)
    n = len(recs)
    dev = torch.device("cuda", 0)
    d_data = torch.zeros(max(len(data), 1) + 64, dtype=torch.uint8, device=dev)
    if len(data):
        d_data[:len(data)].copy_(torch.from_numpy(np.ascontiguousarray(data)))
    d_off = torch.from_numpy(np.ascontiguousarray(off, dtype=np.int64)).to(dev)
    v = pr._get_or_create_versions(writers, rj, columns)
    h = ctypes.c_void_p()
    pr._check(pr.lib.rv_decode_device_versions(v.handle, d_data.data_ptr(), d_off.data_ptr(), n, k,
                                               torch.cuda.current_stream(dev).cuda_stream, ctypes.byref(h)))
    pr._check(pr.lib.rv_result_to_host(h.value))
    return pr._export_batches(h.value, v.reader)


def _run(coracle, writers, rj, ids, k, rng, wide=False):
    recs, vals = VC.messages(rng, writers, ids, wide)
    want = VC.expected(coracle, writers, rj, vals, k, wide)
    for decode in (lambda: pr.deserialize_confluent_versions(recs, writers, rj, k), lambda: _device_decode(writers, rj, recs, k)):
        if isinstance(want, tuple):
            with pytest.raises(ValueError, match=r"\(record %d\)" % want[1]):
                decode()
            continue
        got = decode()
        for b in got:
            assert b.schema.equals(pr.Schema(rj).arrow_schema)
            b.validate(full=not wide)
        VC.compare(got, want, rj)


@pytest.mark.parametrize("seed", range(24))
def test_mixes_narrow(coracle, walker, seed):
    rng = random.Random(seed * 101 + 3)
    rj, writers = VC.writer_chain(rng, unmapped_ok=seed % 6 == 5)
    k = [1, 3, 8][seed % 3]
    n = rng.choice([1, 40, 255, 256, 257, 600])
    _run(coracle, writers, rj, VC.mix(rng, writers, n, MIXES[seed % 4], k), k, rng)


@pytest.mark.parametrize("seed", range(12))
def test_mixes_wide(coracle, walker, seed):
    rng = random.Random(seed * 103 + 5)
    rj, writers = VC.writer_chain(rng, wide=True)
    k = [3, 1, 8][seed % 3]
    _run(coracle, writers, rj, VC.mix(rng, writers, rng.choice([40, 257, 500]), MIXES[seed % 4], k), k, rng, wide=True)


@pytest.mark.parametrize("size", [255, 256, 257, 383, 384, 385])
def test_group_sizes_at_tile_edges(coracle, walker, size):
    rng = random.Random(size)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    seq = []
    for _ in range(3):
        part = [3] * size + [4] * rng.randint(1, 70)
        rng.shuffle(part)
        seq += part
    _run(coracle, writers, rj, seq, 3, rng)


def test_absent_subtrees_maps_and_depth3(coracle, walker):
    rng = random.Random(11)
    writers = {7: VC.ABSENT_W, 8: VC.ABSENT_R}
    for kind in MIXES:
        _run(coracle, writers, VC.ABSENT_R, VC.mix(rng, writers, 300, kind, 3), 3, rng)


def test_one_id_equals_reader_schema_decode(walker):
    rng = random.Random(9)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    recs, _ = VC.messages(rng, writers, [3] * 3000, False)
    got = pr.deserialize_confluent_versions(recs, writers, rj, 3)
    want = pr.deserialize_confluent(recs, workloads.KAFKA_SCHEMA, 3, schema_id=3, reader_schema=rj)
    assert pr.last_versions_timings()["take"] == 0.0   # the single-id path: no partition copy, no take
    assert all(g.equals(w) for g, w in zip(got, want))


def test_projection_and_empty_input():
    rng = random.Random(12)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    recs, _ = VC.messages(rng, writers, VC.mix(rng, writers, 2000, "runs"), False)
    full = pr.deserialize_confluent_versions(recs, writers, rj, 3)
    cols = ["source", "address", "age"]
    got = pr.deserialize_confluent_versions(recs, writers, rj, 3, columns=cols)
    for f, g in zip(full, got):
        assert g.schema.names == cols and all(g.column(c).equals(f.column(c)) for c in cols)
    empty = pr.deserialize_confluent_versions([], writers, rj, 4)
    assert len(empty) == 1 and empty[0].num_rows == 0 and empty[0].schema.names == pr.Schema(rj).arrow_schema.names


def test_errors():
    rng = random.Random(22)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    recs, _ = VC.messages(rng, writers, VC.mix(rng, writers, 3000, "alternate"), False)
    for bad, at, msg in ((b"\x00\x00\x00", 40, "framed message"), (b"\x01" + recs[41][1:], 41, "framed message"),
                         (VC.frame(99, recs[1042][5:]), 1042, "schema id 99 is not registered")):
        r = list(recs)
        r[at] = bad
        with pytest.raises(ValueError, match=r"%s.*\(record %d\)" % (msg, at)):
            pr.deserialize_confluent_versions(r, writers, rj, 3)
    for damaged, framed in ((500, 1200), (1200, 500)):
        r = list(recs)
        r[damaged] = r[damaged][:6]
        r[framed] = VC.frame(12345, r[framed][5:])
        with pytest.raises(ValueError, match=r"\(record %d\)" % min(damaged, framed)):
            pr.deserialize_confluent_versions(r, writers, rj, 3)
    ev1 = json.dumps({"type": "record", "name": "R", "fields": [{"name": "e", "type": {"type": "enum", "name": "E", "symbols": ["A", "B", "C"]}}]})
    ev2 = json.dumps({"type": "record", "name": "R", "fields": [{"name": "e", "type": {"type": "enum", "name": "E", "symbols": ["A", "B"]}}]})
    msgs = [VC.frame(2, b"\x02")] * 10 + [VC.frame(1, b"\x00"), VC.frame(1, b"\x04")] + [VC.frame(2, b"\x00")] * 5
    with pytest.raises(ValueError, match=r"enum.*\(record 11\)"):
        pr.deserialize_confluent_versions(msgs, {1: ev1, 2: ev2}, ev2, 2)


@pytest.mark.parametrize("seed", range(40))
def test_damaged_inputs_match_emulation(seed):
    """The device's verdict equals the host emulation's (tests/test_versions.py checks that one against the writers')."""
    from tests import emu
    from tests import mutation as M
    from tests.emu import versions as V
    rng = random.Random(seed * 17 + 1)
    rj, writers = VC.writer_chain(rng)
    recs, _ = VC.messages(rng, writers, VC.mix(rng, writers, rng.choice([3, 40, 257]), rng.choice(MIXES), 3), False)
    msgs = [r[:5] + b for r, b in zip(recs, M.damage(rng, [r[5:] for r in recs]))]
    n, k = len(msgs), rng.choice([1, 2, 3])
    data, off = po.pack_records(msgs)
    try:
        V.decode(writers, rj, data, off, n, k)
        want = None
    except emu.EmuError as e:
        want = (e.code, e.record)
    if want is not None and want[0] == 8:
        return
    if want is None:
        pr.deserialize_confluent_versions(msgs, writers, rj, k)
    else:
        with pytest.raises(ValueError, match=r"\(record %d\)" % want[1]):
            pr.deserialize_confluent_versions(msgs, writers, rj, k)


def test_two_threads_share_one_registry(coracle):
    rng = random.Random(31)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    cases = []
    for t in range(2):
        recs, vals = VC.messages(rng, writers, VC.mix(rng, writers, 5000, ["runs", "alternate"][t]), False)
        cases.append((recs, VC.expected(coracle, writers, rj, vals, 4)))
    errors = []

    def work(recs, want):
        try:
            for _ in range(5):
                VC.compare(pr.deserialize_confluent_versions(recs, writers, rj, 4), want)
        except Exception as e:  # noqa: BLE001 - reported below
            errors.append(e)
    th = [threading.Thread(target=work, args=c) for c in cases]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors


def test_batch_overflows_only_when_parts_add_up():
    """Two writers' parts of one batch each fit i32 offsets, together they do not."""
    w1 = json.dumps({"type": "record", "name": "R", "fields": [{"name": "s", "type": "string"}]})
    w2 = json.dumps({"type": "record", "name": "R", "fields": [{"name": "s", "type": "string"}, {"name": "x", "type": "int", "default": 1}]})
    big = b"a" * (1 << 20)
    ws = po.parse_schema(w1)
    m1, m2 = VC.frame(1, po.encode_datum(ws, {"s": big.decode()})), VC.frame(2, po.encode_datum(ws, {"s": big.decode()}))
    msgs = [m1, m2] * 1100   # 2.2 GiB of string bytes in one batch, 1.1 GiB per writer
    with pytest.raises(ValueError) as ei:
        pr.deserialize_confluent_versions(msgs, {1: w1, 2: w1}, w2, 1)
    assert "overflow" in str(ei.value)
    got = pr.deserialize_confluent_versions(msgs[:200], {1: w1, 2: w1}, w2, 1)[0]
    assert got.num_rows == 200 and got.column("s")[5].as_py() == big.decode()


@pytest.mark.parametrize("mix", ["alternate", ("runs", 100_000)], ids=["alternate", "runs"])
def test_bench_scale_kafka(mix):
    """10 M Kafka messages of v1 and v2, read as v2 with k = 8, through the device entry point; every buffer checked."""
    import torch
    n, k = 10_000_000, 8
    data, off, h_data, h_off, v1, v2 = VC.kafka_versions_input(n, mix, k=k)
    dev = torch.device("cuda", 0)
    d_data = torch.zeros(len(data) + 64, dtype=torch.uint8, device=dev)
    d_data[:len(data)].copy_(torch.from_numpy(data))
    d_off = torch.from_numpy(off).to(dev)
    v = pr._get_or_create_versions({3: v1, 4: v2}, v2, None)
    h = ctypes.c_void_p()
    pr._check(pr.lib.rv_decode_device_versions(v.handle, d_data.data_ptr(), d_off.data_ptr(), n, k,
                                               torch.cuda.current_stream(dev).cuda_stream, ctypes.byref(h)))
    pr._check(pr.lib.rv_result_to_host(h.value))
    got = pr._export_batches(h.value, v.reader)
    VC.check_kafka_v2(got, v1, v2, h_data, h_off, n, k)
