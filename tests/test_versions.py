"""Confluent messages written with several schema versions, decoded into one reader schema in message order
(rv_versions_create / rv_decode_*_versions / deserialize_confluent_versions).  Batch i must equal, buffer for buffer, the
oracle's decode of its messages each resolved with its own writer and re-encoded with the reader.  These CPU tests run the
product's header check, layout, take job tables and per-row take steps through the host emulation (tests/emu/versions.py);
tests/test_gpu_versions.py runs the same cases on the device."""
import json
import random

import pytest

import pyruhvro_b200 as pr
import workloads
from oracle import pyoracle as po
from tests import emu
from tests import mutation as M
from tests import resolution as RS
from tests import versions_cases as VC
from tests.emu import versions as V


def _run(coracle, writers, rj, id_seq, k, rng, wide=False, columns=None):
    recs, vals = VC.messages(rng, writers, id_seq, wide)
    data, off = po.pack_records(recs)
    want = VC.expected(coracle, writers, rj, vals, k, wide)
    if isinstance(want, tuple):
        with pytest.raises(emu.EmuError) as ei:
            V.decode(writers, rj, data, off, len(recs), k, columns)
        assert (ei.value.code, ei.value.record) == (6, want[1])
        return None
    got = V.decode(writers, rj, data, off, len(recs), k, columns)
    if columns is None:
        VC.compare(got, want, rj)
    return got


MIXES = ["runs", "alternate", "absent", "single"]


@pytest.mark.parametrize("seed", range(24))
def test_mixes_narrow(coracle, seed):
    rng = random.Random(seed * 101 + 3)
    rj, writers = VC.writer_chain(rng, unmapped_ok=seed % 6 == 5)
    k = [1, 3, 8][seed % 3]
    n = rng.choice([1, 40, 255, 256, 257, 600])
    _run(coracle, writers, rj, VC.mix(rng, writers, n, MIXES[seed % 4], k), k, rng)


@pytest.mark.parametrize("seed", range(12))
def test_mixes_wide(coracle, seed):
    rng = random.Random(seed * 103 + 5)
    rj, writers = VC.writer_chain(rng, wide=True)
    k = [3, 1, 8][seed % 3]
    _run(coracle, writers, rj, VC.mix(rng, writers, rng.choice([40, 257, 500]), MIXES[seed % 4], k), k, rng, wide=True)


@pytest.mark.parametrize("size", [255, 256, 257, 383, 384, 385])
def test_group_sizes_at_tile_edges(coracle, size):
    """A group of exactly `size` messages between the other writer's messages, in each of 3 chunks."""
    rng = random.Random(size)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    seq = []
    for _ in range(3):
        part = [3] * size + [4] * rng.randint(1, 70)
        rng.shuffle(part)
        seq += part
    _run(coracle, writers, rj, seq, 3, rng)


def test_one_id_is_the_resolved_decode(coracle):
    rng = random.Random(9)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    recs, vals = VC.messages(rng, writers, [3] * 600, False)
    data, off = po.pack_records(recs)
    from tests.emu import resolve as R
    bare = [r[5:] for r in recs]
    bd, bo = po.pack_records(bare)
    got = V.decode(writers, rj, data, off, 600, 3)
    want = R.decode(workloads.KAFKA_SCHEMA, rj, bd, bo, 600, 3)
    assert [b.equals(w) for b, w in zip(got, want)] == [True] * 3


def test_absent_subtrees_maps_and_depth3(coracle):
    rng = random.Random(11)
    writers = {7: VC.ABSENT_W, 8: VC.ABSENT_R}
    for kind in MIXES:
        _run(coracle, writers, VC.ABSENT_R, VC.mix(rng, writers, 300, kind, 3), 3, rng)


def test_projection(coracle):
    rng = random.Random(12)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    recs, _ = VC.messages(rng, writers, VC.mix(rng, writers, 500, "runs"), False)
    data, off = po.pack_records(recs)
    full = V.decode(writers, rj, data, off, 500, 3)
    cols = ["source", "address", "age"]
    got = V.decode(writers, rj, data, off, 500, 3, columns=cols)
    for f, g in zip(full, got):
        assert g.schema.names == cols
        for c in cols:
            assert g.column(c).equals(f.column(c))


def test_coverage_of_the_matrix():
    """The cases above reach every slot role, list depth 3, maps and nullable fields."""
    cov = {"roles": set(), "depth": 0, "map": False}
    for seed in range(24):
        rj, _ = VC.writer_chain(random.Random(seed * 101 + 3))
        VC.schema_roles(rj, cov)
    for seed in range(12):
        rj, _ = VC.writer_chain(random.Random(seed * 103 + 5), wide=True)
        VC.schema_roles(rj, cov)
    VC.schema_roles(VC.ABSENT_R, cov)
    assert cov["roles"] >= {"Validity", "Bits", "Values32", "Values64", "ValuesW", "Offsets", "Data", "TypeIds"}, cov
    assert cov["depth"] >= 3 and cov["map"]


# ---- errors ----------------------------------------------------------------------------------------------------------
def _verdict(fn):
    try:
        fn()
        return None
    except emu.EmuError as e:
        return (e.code, e.record)


def test_registry_errors():
    K, R2 = workloads.KAFKA_SCHEMA, RS.kafka_v2()
    cases = [({}, R2, None, "no writer"), ({1: K, -1: K}, R2, None, "not a u32"), ({2 ** 32: K}, R2, None, "not a u32"),
             ({i: K for i in range(257)}, R2, None, "more than 256"), ({1: K}, R2, ["nope"], "no top-level field")]
    for ws, rj, cols, msg in cases:
        with pytest.raises(ValueError, match=msg):
            pr.Versions(ws, rj, cols)
    with pytest.raises(ValueError, match="schema id 3: schema resolution: field .age."):
        pr.Versions({3: R2, 5: K, 6: workloads.FLAT_SCHEMA}, K)
    # a projected or resolved handle as reader or writer
    lib, full, proj = pr.lib, pr.Schema(R2), pr.Schema(R2).project(["age"])
    import ctypes
    for reader, writer in ((proj, full), (full, proj), (full, pr.Schema(K).read_as(R2))):
        h = ctypes.c_void_p()
        ids = (ctypes.c_int64 * 1)(1)
        ws = (ctypes.c_void_p * 1)(writer.handle)
        assert lib.rv_versions_create(reader.handle, ids, ws, 1, None, 0, ctypes.byref(h)) == 9
    # a repeated id can only come through the C ABI (a dict has unique keys)
    h = ctypes.c_void_p()
    ids = (ctypes.c_int64 * 2)(4, 4)
    ws = (ctypes.c_void_p * 2)(full.handle, full.handle)
    assert lib.rv_versions_create(full.handle, ids, ws, 2, None, 0, ctypes.byref(h)) == 9
    assert b"registered twice" in lib.rv_last_error()


def test_frame_errors():
    rng = random.Random(21)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    recs, _ = VC.messages(rng, writers, VC.mix(rng, writers, 300, "alternate"), False)
    for bad, at in ((b"\x00\x00\x00", 40), (b"\x01" + recs[41][1:], 41), (VC.frame(99, recs[42][5:]), 42)):
        r = list(recs)
        r[at] = bad
        data, off = po.pack_records(r)
        assert _verdict(lambda: V.decode(writers, rj, data, off, 300, 3)) == (12, at)


def test_lowest_message_wins():
    """A damaged datum of one writer before or after a frame error in another."""
    rng = random.Random(22)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    recs, _ = VC.messages(rng, writers, VC.mix(rng, writers, 300, "alternate"), False)
    for damaged, framed in ((50, 120), (120, 50), (51, 251)):
        r = list(recs)
        r[damaged] = r[damaged][:6]   # truncated datum: the writer's decode fails on it
        r[framed] = VC.frame(12345, r[framed][5:])
        data, off = po.pack_records(r)
        got = _verdict(lambda: V.decode(writers, rj, data, off, 300, 3))
        assert got[1] == min(damaged, framed), got
        assert got[0] == (12 if framed < damaged else 1)


def test_unmapped_enum_in_one_writer():
    ev1 = json.dumps({"type": "record", "name": "R", "fields": [{"name": "e", "type": {"type": "enum", "name": "E", "symbols": ["A", "B", "C"]}}]})
    ev2 = json.dumps({"type": "record", "name": "R", "fields": [{"name": "e", "type": {"type": "enum", "name": "E", "symbols": ["A", "B"]}}]})
    writers = {1: ev1, 2: ev2}
    msgs = [VC.frame(2, b"\x02")] * 10 + [VC.frame(1, b"\x00"), VC.frame(1, b"\x04")] + [VC.frame(2, b"\x00")] * 5
    data, off = po.pack_records(msgs)
    assert _verdict(lambda: V.decode(writers, ev2, data, off, len(msgs), 2)) == (6, 11)


@pytest.mark.parametrize("seed", range(200))
def test_damaged_inputs_over_several_writers(seed):
    """The verdict is the lowest failing message of the writers' own decodes of their messages."""
    rng = random.Random(seed * 17 + 1)
    rj, writers = VC.writer_chain(rng)
    recs, vals = VC.messages(rng, writers, VC.mix(rng, writers, rng.choice([3, 40, 257]), rng.choice(MIXES), 3), False)
    heads, bodies = [r[:5] for r in recs], M.damage(rng, [r[5:] for r in recs])
    msgs = [h + b for h, b in zip(heads, bodies)]
    n, k = len(msgs), rng.choice([1, 2, 3])
    data, off = po.pack_records(msgs)
    want = None
    for sid, wj in writers.items():
        idx = [i for i in range(n) if vals[i][0] == sid]
        if not idx:
            continue
        bd, bo = po.pack_records([bodies[i] for i in idx])
        from tests.emu import resolve as R
        v = _verdict(lambda: R.decode(wj, rj, bd, bo, len(idx), 1))
        if v is not None and (want is None or idx[v[1]] < want[1]):
            want = (v[0], idx[v[1]])
    got = _verdict(lambda: V.decode(writers, rj, data, off, n, k))
    if want is not None and want[0] == 8:
        return
    assert got == want, (rj, writers)
