"""Permissive multi-version decodes on the device (Versions.permissive, errors="null" of deserialize_confluent_versions
and deserialize_single_object_versions): damaged datums, wrong magic bytes, short messages and unregistered ids or
fingerprints become null rows and are reported, through the host and device-resident entry points with both walkers.
The contract and its oracle are in tests/versions_permissive_cases.py."""
import ctypes
import random

import numpy as np
import pyarrow as pa
import pytest

import pyruhvro_b200 as pr
import workloads
from tests import resolution as RS
from tests import versions_cases as VC
from tests import versions_permissive_cases as VP

pytestmark = pytest.mark.gpu


@pytest.fixture(params=[1, 0], ids=["jit", "interp"])
def walker(request):
    pr.set_jit_enabled(request.param)
    yield request.param
    pr.set_jit_enabled(-1)


def device(v, recs, k):
    """rv_decode_device_versions of `recs` with registry `v`: (batches, report)."""
    import torch
    from oracle import pyoracle as po
    data, off = po.pack_records(recs)
    dev = torch.device("cuda", 0)
    d_data = torch.zeros(max(len(data), 1) + 64, dtype=torch.uint8, device=dev)
    if len(data):
        d_data[:len(data)].copy_(torch.from_numpy(np.ascontiguousarray(data)))
    d_off = torch.from_numpy(np.ascontiguousarray(off, dtype=np.int64)).to(dev)
    h = ctypes.c_void_p()
    pr._check(pr.lib.rv_decode_device_versions(v.handle, d_data.data_ptr(), d_off.data_ptr(), len(recs), k,
                                               torch.cuda.current_stream(dev).cuda_stream, ctypes.byref(h)))
    pr._check(pr.lib.rv_result_to_host(h.value))
    return pr._export_batches(h.value, v.reader, True)


def host(case, k):
    if case.so:
        ws = [case.writers[i] for i in sorted(case.writers)]
        return pr.deserialize_single_object_versions(case.recs, ws, case.rj, k, columns=case.columns, errors="null")
    return pr.deserialize_confluent_versions(case.recs, case.writers, case.rj, k, columns=case.columns, errors="null")


def check(case, k):
    strict = case.registry()
    want_bad = case.verdicts(strict)
    want = case.oracle(want_bad, k)
    perm = strict.permissive()
    for name, run in (("host", lambda: host(case, k)), ("device", lambda: device(perm, case.recs, k))):
        batches, bad = run()
        assert VP.report(bad) == want_bad, (name, VP.report(bad)[:5], want_bad[:5])
        for b in batches:
            b.validate(full=True)
        VP.compare(batches, want, name)
    return want_bad


@pytest.mark.parametrize("single_object", [False, True], ids=["confluent", "single_object"])
@pytest.mark.parametrize("seed", range(8))
def test_random_writer_sets(walker, seed, single_object):
    rng = random.Random(seed * 31 + 7 + single_object)
    rj, writers = VC.writer_chain(rng, unmapped_ok=seed % 4 == 3)
    k = [1, 3, 8][seed % 3]
    n = rng.choice([40, 255, 256, 257, 600])
    case = VP.Case(rng, writers, rj, n, single_object)
    for at in rng.sample(range(n), max(1, n // 10)):
        case.damage(rng, at)
    check(case, k)


PLACEMENTS = {
    "chunk_edges": lambda n, k: sorted({j * (n // k) for j in range(k)} | {min(n, (j + 1) * (n // k)) - 1 for j in range(k)} | {n - 1}),
    "whole_chunk": lambda n, k: list(range(n // k, 2 * (n // k))) if k > 1 else list(range(n)),
    "all": lambda n, k: list(range(n)),
    "tile_edges": lambda n, k: [255, 256, 257],
}


@pytest.mark.parametrize("k", [1, 3, 8])
@pytest.mark.parametrize("where", list(PLACEMENTS))
def test_placements(walker, where, k):
    rng = random.Random(hash((where, k)) & 0xFFFF)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    n = 600
    case = VP.Case(rng, writers, rj, n)
    for i, at in enumerate(PLACEMENTS[where](n, k)):
        case.damage(rng, at, VP.DAMAGES[i % len(VP.DAMAGES)])
    got = check(case, k)
    assert got, "no bad message"


def test_columns_and_empty_input(walker):
    rng = random.Random(5)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    case = VP.Case(rng, writers, rj, 300, columns=["status", "name", "emails"])
    for at in range(0, 300, 7):
        case.damage(rng, at)
    check(case, 3)
    batches, bad = pr.deserialize_confluent_versions([], writers, rj, 4, errors="null")
    assert [b.num_rows for b in batches] == [0] and bad.num_rows == 0


@pytest.mark.parametrize("single_object", [False, True], ids=["confluent", "single_object"])
def test_one_key_direct_path(walker, single_object):
    """Every message of one writer: the direct path, with and without damaged datums, equals the oracle; with a message
    of another writer or in the bad group the partition path runs and gives the same rows and report."""
    rng = random.Random(11)
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    case = VP.Case(rng, {3: writers[3]}, rj, 500, single_object)
    check(case, 3)
    for at in (0, 17, 256, 499):
        case.damage(rng, at, "datum")
    direct = check(case, 3)
    assert direct
    # the same messages and one more in the bad group: the partition path
    extra = VP.Case(rng, {3: writers[3]}, rj, 500, single_object)
    extra.recs, extra.orig, extra.vals = case.recs + [b"\x07"], case.orig + [b"\x07"], case.vals + [case.vals[0]]
    got = check(extra, 3)
    assert got[:-1] == direct and got[-1][0] == 500


def test_clean_permissive_equals_strict_read_as_optional(walker):
    rng = random.Random(3)
    rj, writers = VC.writer_chain(rng)
    recs, _ = VC.messages(rng, writers, VC.mix(rng, writers, 700, "alternate"))
    strict = pr.deserialize_confluent_versions(recs, writers, rj, 3)
    batches, bad = pr.deserialize_confluent_versions(recs, writers, rj, 3, errors="null")
    assert bad.num_rows == 0
    assert batches[0].schema.equals(pr.Schema(rj).permissive().arrow_schema)
    VP.compare([pa.RecordBatch.from_arrays(b.columns, schema=batches[0].schema) for b in strict], batches, "clean")


def test_python_surface():
    rj, writers = RS.kafka_v2(), {3: workloads.KAFKA_SCHEMA, 4: RS.kafka_v2()}
    rng = random.Random(9)
    recs, _ = VC.messages(rng, writers, [3, 4] * 20)
    recs[5] = VC.frame(77, recs[5][5:])
    with pytest.raises(ValueError, match=r"schema id 77 is not registered \(record 5\)"):
        pr.deserialize_confluent_versions(recs, writers, rj, 2)
    batches, bad = pr.deserialize_confluent_versions(recs, writers, rj, 2, errors="null")
    assert VP.report(bad) == [(5, 12, "framed message: schema id 77 is not registered")]
    assert sum(b.num_rows for b in batches) == 40 and batches[0].column("name")[5].as_py() is None
    with pytest.raises(ValueError, match="errors"):
        pr.deserialize_confluent_versions(recs, writers, rj, 2, errors="ignore")
    # the strict registry is unchanged, and a permissive one cannot be made permissive again
    v = pr._get_or_create_versions(writers, rj, None)
    p = v.permissive()
    h = ctypes.c_void_p()
    assert pr.lib.rv_versions_permissive(p.handle, ctypes.byref(h)) == 9
    with pytest.raises(ValueError, match="record 5"):
        pr._export_batches(pr._ext().decode_list_versions(v.handle, recs, 2), v.reader)


def test_bench_scale_kafka():
    """2 M Kafka messages of v1 and v2 alternating, every 1000th bad: half of them an empty datum (RV_ERR_EOF), half an
    unregistered schema id (RV_ERR_FRAME).  Every buffer of the good rows equals the strict decode of the clean input."""
    n, k = 2_000_000, 8
    data, off, _, _, v1, v2 = VC.kafka_versions_input(n, "alternate", k=k)
    writers = {3: v1, 4: v2}
    strict = pa.Table.from_batches(pr.deserialize_confluent_versions(_as_list(data, off), writers, v2, k))
    bad_at = np.arange(0, n, 1000)
    empty, unknown = bad_at[0::2], bad_at[1::2]
    lens = np.diff(off)
    keep = np.ones(int(off[-1]), dtype=bool)
    cut = np.repeat(np.isin(np.arange(n), empty), lens) & (np.arange(int(off[-1])) - np.repeat(off[:-1], lens) >= 5)
    keep[cut] = False
    d2 = data.copy()
    d2[off[unknown] + 4] = 99   # ids 3 and 4 become 99
    new_lens = np.where(np.isin(np.arange(n), empty), 5, lens)
    o2 = np.concatenate([[0], np.cumsum(new_lens)]).astype(np.int64)
    msgs = _as_list(np.ascontiguousarray(d2[keep]), o2)
    batches, bad = pr.deserialize_confluent_versions(msgs, writers, v2, k, errors="null")
    rep = bad.to_pydict()
    assert rep["record"] == bad_at.tolist()
    assert rep["status"] == [1 if i % 2 == 0 else 12 for i in range(len(bad_at))]
    assert all(t == "framed message: schema id 99 is not registered" for t in rep["error"][1::2])
    assert [b.num_rows for b in batches] == [b.num_rows for b in strict.to_batches()]
    got = pa.Table.from_batches(batches)
    good = np.ones(n, dtype=bool)
    good[bad_at] = False
    for name in strict.column_names:
        g, w = got.column(name), strict.column(name)
        if pa.types.is_union(g.type):
            gt = np.concatenate([np.frombuffer(c.buffers()[1], dtype=np.int8)[c.offset:c.offset + len(c)] for c in g.chunks])
            wt = np.concatenate([np.frombuffer(c.buffers()[1], dtype=np.int8)[c.offset:c.offset + len(c)] for c in w.chunks])
            assert np.array_equal(gt[good], wt[good]) and not gt[~good].any(), name
            continue
        assert g.filter(pa.array(good)).equals(w.filter(pa.array(good))), name
        if pa.types.is_map(g.type):
            o = g.filter(pa.array(~good)).combine_chunks().offsets.to_numpy()
            assert o[0] == o[-1], name
        else:
            assert g.filter(pa.array(~good)).null_count == len(bad_at), name


def _as_list(data, off):
    arr = pa.LargeBinaryArray.from_buffers(pa.large_binary(), len(off) - 1, [None, pa.py_buffer(np.ascontiguousarray(off)), pa.py_buffer(data)])
    return arr.to_pylist()
