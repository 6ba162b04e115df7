"""Permissive multi-version decodes (rv_versions_permissive) through the host emulation
(tests/emu/versions_permissive.py): the product's header classification, permissive resolved plans, layout, take job
tables and take steps with the null-row path.  Each case checks the batches against the permissive single-schema decode of the rebuilt
list L' (tests/versions_permissive_cases.py states the contract), emulated with the interpreter, and the report against
each message's verdict alone.  tests/test_gpu_versions_permissive.py runs the same kind of cases on the device."""
import ctypes
import random
import struct

import numpy as np
import pytest

import pyruhvro_b200 as pr
import workloads
from oracle import pyoracle as po
from tests import emu
from tests import resolution as RS
from tests import versions_cases as VC
from tests import versions_permissive_cases as VP
from tests.emu import permissive as EP
from tests.emu import resolve as R
from tests.emu import versions_permissive as VPE


def verdict(case, m: bytes):
    """The status of the strict versions decode of `m` alone: the partition's header check restated, then the writer's
    resolved decode of the datum (emulated).  None: the message decodes."""
    if case.so:
        if len(m) < 10 or m[:2] != b"\xc3\x01":
            return 12
        fp = struct.unpack("<Q", m[2:10])[0]
        wj = {f: case.writers[i] for i, f in case.fps.items()}.get(fp)
    else:
        if len(m) < 5 or m[0] != 0:
            return 12
        wj = case.writers.get(struct.unpack(">I", m[1:5])[0])
    if wj is None:
        return 12
    body = m[case.hdr:]
    data, off = po.pack_records([body])
    try:
        R.decode(wj, case.rj, data, off, 1, 1)
        return None
    except emu.EmuError as e:
        return e.code


def run(case, k):
    want_bad = []
    for i, m in enumerate(case.recs):
        v = verdict(case, m)
        if v is None and m != case.orig[i]:
            case.recs[i] = case.orig[i]
            v = verdict(case, m)
        if v is not None:
            want_bad.append((i, v))
    rs = po.parse_schema(case.rj)
    parsed = {i: po.parse_schema(sj) for i, sj in case.writers.items()}
    meta = RS.ReaderMeta(case.rj)
    bad_at = {i for i, _ in want_bad}
    lp = [b"\x01\x00\x00\x00\x00" if i in bad_at else VC.frame(1, po.encode_datum(rs, RS.resolve_value(parsed[sid], rs, v, meta)))
          for i, (sid, v) in enumerate(case.vals)]
    ld, lo = po.pack_records(lp)
    want, _ = EP.decode(case.rj, ld, lo, len(lp), k, columns=case.columns, frame=(5, 1, 0))
    data, off = po.pack_records(case.recs)
    fps = {case.fps[i]: sj for i, sj in case.writers.items()} if case.so else None
    got, bad = VPE.decode(case.writers, case.rj, data, off, len(case.recs), k, case.columns, fingerprints=fps)
    assert bad == want_bad, (bad[:6], want_bad[:6])
    VP.compare(got, want, case.rj)
    return bad


@pytest.mark.parametrize("single_object", [False, True], ids=["confluent", "single_object"])
@pytest.mark.parametrize("seed", range(10))
def test_random_writer_sets(seed, single_object):
    rng = random.Random(seed * 37 + 1 + single_object)
    rj, writers = VC.writer_chain(rng, unmapped_ok=seed % 4 == 3)
    k = [1, 3, 8][seed % 3]
    n = rng.choice([40, 255, 256, 257, 600])
    case = VP.Case(rng, writers, rj, n, single_object)
    for at in rng.sample(range(n), max(1, n // 8)):
        case.damage(rng, at)
    run(case, k)


def test_forged_varints():
    rng = random.Random(77)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    case = VP.Case(rng, writers, rj, 300)
    from tests import mutation as M
    for at in range(0, 300, 9):
        h, body = case.orig[at][:5], case.orig[at][5:]
        case.recs[at] = h + M.forge_varints(random.Random(at), [body])[0]
    run(case, 3)


def test_unmapped_enum_and_bad_branch():
    ev1 = '{"type":"record","name":"R","fields":[{"name":"e","type":{"type":"enum","name":"E","symbols":["A","B","C"]}},{"name":"u","type":["int","string","null"]}]}'
    ev2 = '{"type":"record","name":"R","fields":[{"name":"e","type":{"type":"enum","name":"E","symbols":["A","B"]}},{"name":"u","type":["int","string","null"]}]}'
    case = VP.Case(random.Random(1), {1: ev1, 2: ev2}, ev2, 0)
    msgs = [VC.frame(2, b"\x02\x04"), VC.frame(1, b"\x04\x04"), VC.frame(1, b"\x00\x09"), VC.frame(2, b"\x00\x00\x02")]
    vals = [(2, {"e": 1, "u": (2, None)}), (1, {"e": 2, "u": (2, None)}), (1, {"e": 0, "u": (2, None)}), (2, {"e": 0, "u": (0, 1)})]
    case.recs, case.orig, case.vals = list(msgs), list(msgs), vals
    assert run(case, 2) == [(1, 6), (2, 5)]


PLACEMENTS = {
    "chunk_edges": lambda n, k: sorted({j * (n // k) for j in range(k)} | {min(n, (j + 1) * (n // k)) - 1 for j in range(k)} | {n - 1}),
    "whole_chunk": lambda n, k: list(range(n // k, 2 * (n // k))) if k > 1 else list(range(n)),
    "all": lambda n, k: list(range(n)),
    "tile_edges": lambda n, k: [255, 256, 257],
}


@pytest.mark.parametrize("k", [1, 3, 8])
@pytest.mark.parametrize("where", list(PLACEMENTS))
def test_placements(where, k):
    rng = random.Random(len(where) * 10 + k)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    case = VP.Case(rng, writers, rj, 600)
    for i, at in enumerate(PLACEMENTS[where](600, k)):
        case.damage(rng, at, VP.DAMAGES[i % len(VP.DAMAGES)])
    assert run(case, k)


def test_columns_and_empty_input():
    rng = random.Random(5)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    case = VP.Case(rng, writers, rj, 300, columns=["status", "name", "emails"])
    for at in range(0, 300, 7):
        case.damage(rng, at)
    run(case, 3)
    got, bad = VPE.decode(writers, rj, np.zeros(0, dtype=np.uint8), [0], 0, 4)
    assert [b.num_rows for b in got] == [0] and bad == []


@pytest.mark.parametrize("damaged", [False, True])
def test_one_key(damaged):
    """Every message of one writer (the device's direct path), with and without damaged datums."""
    rng = random.Random(11)
    case = VP.Case(rng, {3: workloads.KAFKA_SCHEMA}, RS.kafka_v2(), 500)
    for at in ((0, 17, 256, 499) if damaged else ()):
        case.damage(rng, at, "datum")
    assert bool(run(case, 3)) == damaged


def test_registry_abi():
    """rv_versions_permissive refuses a permissive registry; the strict registry it was made from is unchanged."""
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    v = pr.Versions(writers, rj)
    before = v.reader.arrow_schema
    p = v.permissive()
    h = ctypes.c_void_p()
    assert pr.lib.rv_versions_permissive(p.handle, ctypes.byref(h)) == 9
    assert b"already permissive" in pr.lib.rv_last_error()
    assert pr.lib.rv_versions_permissive(None, ctypes.byref(h)) == 9
    assert v.reader.arrow_schema.equals(before) and not p.reader.arrow_schema.equals(before)
    assert p.reader.arrow_schema.equals(pr.Schema(rj).permissive().arrow_schema)
    assert not pr.lib.rv_schema_is_permissive(v.reader.handle) and pr.lib.rv_schema_is_permissive(p.reader.handle)
    so = pr.Versions([workloads.KAFKA_SCHEMA, rj], rj, ["name"], single_object=True).permissive()
    assert so.reader.arrow_schema.names == ["name"]
    with pytest.raises(ValueError, match="errors"):
        pr.deserialize_confluent_versions([], writers, rj, errors="skip")
    with pytest.raises(ValueError, match="errors"):
        pr.deserialize_single_object_versions([], [rj], rj, errors=None)
