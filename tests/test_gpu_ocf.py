"""Object container files on the GPU: deserialize_ocf / rv_decode_ocf_host — the container reader on the host, the
record-offsets kernel (one lane per block) and the fused decode — against the restated container reader and the C oracle
(the Python decoder for the wider subset), through both walkers.  The host-emulation twin is tests/test_ocf.py; files
whose counts exceed their bytes are tested there only (they are rejected before any CUDA call)."""
import ctypes
import random
import re

import numpy as np
import pytest

import pyruhvro_b200 as pr
from oracle import pyoracle as po
from tests import ocf_files as O
from tests.parity import assert_matches_oracle, expected_schema
from tests.test_ocf import CASES, LAYOUTS, N, bug2_file, case, layout_counts

pytestmark = pytest.mark.gpu
TILE = 384
BIG_SCHEMA = ('{"type":"record","name":"Big","fields":[{"name":"id","type":"long"},{"name":"s","type":"string"},'
              '{"name":"t","type":["null","string"]}]}')


@pytest.fixture(params=["jit", "interp"])
def walker(request):
    pr.set_jit_enabled(1 if request.param == "jit" else 0)
    yield request.param
    pr.set_jit_enabled(-1)


class GpuOcfError(Exception):
    def __init__(self, status, message):
        super().__init__(message)
        m = re.search(r"\(record (-?\d+)\)", message)
        self.status, self.record = status, int(m.group(1)) if m else -1


def gpu_ocf(f, k):
    """rv_decode_ocf_host: the status from its return code, the record from its message."""
    buf = np.frombuffer(f, dtype=np.uint8)
    sh, h = ctypes.c_void_p(), ctypes.c_void_p()
    rc = pr.lib.rv_decode_ocf_host(buf.ctypes.data if buf.size else None, buf.size, k, ctypes.byref(sh), ctypes.byref(h))
    if rc:
        raise GpuOcfError(rc, pr._last_error())
    return pr._export_batches(h.value, pr.Schema._adopt(sh.value))


def gpu_error(e):
    if not isinstance(e, GpuOcfError):
        return None
    if e.status == 12 and "object container file" in str(e):
        return "container"
    return (po.ERR_NAMES.get(e.status, str(e.status)), e.record)


def check(coracle, f, k, wide=False, schema=None):
    assert O.check(coracle, gpu_ocf, gpu_error, f, k, wide) == "decoded"
    if schema is not None and not wide:
        assert all(b.schema.equals(expected_schema(schema)) for b in pr.deserialize_ocf(f, k))


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("name", CASES)
def test_gpu_layouts_decode_like_the_datums(coracle, walker, name, layout):
    sj, recs, wide = case(name)
    rng = random.Random(f"{name}/{layout}")
    for k in (1, 3, 8, N + 5) if layout == "chunk-edges" else (2,):
        check(coracle, O.ocf_file(sj, recs, counts=layout_counts(layout, N, k, rng), rng=rng), k, wide)
        assert pr.last_walker() == walker


def kafka(n, seed):
    import workloads
    sj, data, off = workloads.generate("kafka", n, seed=seed)
    return sj, [data[off[i]:off[i + 1]].tobytes() for i in range(n)]


def check_datums(coracle, f, k, sj, recs):
    """A large file of known datums: every buffer against the C oracle on them (no restated reader in between)."""
    data, off = po.pack_records(recs)
    assert_matches_oracle(coracle, pr.deserialize_ocf(f, k), sj, data, off, len(recs), k, full_validate=False)


def test_gpu_kafka_blocks_at_384_row_tile_edges(coracle):
    sj, recs = kafka(2000, 11)
    ends = [383, 384, 385, 767, 768, 2000]
    counts = [b - a for a, b in zip([0] + ends, ends)]
    f = O.ocf_file(sj, recs, counts=counts, rng=random.Random(1))
    pr.set_jit_enabled(1)
    try:
        for k in (1, 2, 5):
            check(coracle, f, k, schema=sj)
            assert pr.last_walker() == "jit" and pr.lib.rv_last_tile() == TILE
    finally:
        pr.set_jit_enabled(-1)


def test_gpu_large_records_take_the_global_walk(coracle, walker):
    """Records of 36-70 KB: no tile fits the shared-memory window."""
    sj = BIG_SCHEMA
    rng = random.Random(3)
    recs = []
    for i in range(600):
        s = bytes(rng.randrange(97, 123) for _ in range(64)) * (rng.randrange(36 << 10, 70 << 10) // 64)
        recs.append(O.zz(i) + O.zz(len(s)) + s + (b"\x02\x06abc" if i % 2 else b"\x00"))
    f = O.ocf_file(sj, recs, counts=O.counts_with_edges(600, 2), rng=rng)
    got = gpu_ocf(f, 2)
    assert pr.lib.rv_last_slow_tiles() > 0
    assert O.check(coracle, lambda *_: got, gpu_error, f, 2) == "decoded"


def test_gpu_one_block_of_50000_records_and_5000_one_record_blocks(coracle, walker):
    sj, recs = kafka(50_000, 12)
    check_datums(coracle, O.ocf_file(sj, recs, counts=[50_000], rng=random.Random(2)), 4, sj, recs)
    check_datums(coracle, O.ocf_file(sj, recs[:5000], counts=[1] * 5000, rng=random.Random(3)), 3, sj, recs[:5000])


def test_gpu_projected_files(coracle):
    from tests.test_gpu_tile384 import KAFKA_PROJECTIONS
    from tests.test_projection import _assert_selected, _names, _oracle_batches, _random_projection
    from tests.parity import gen_case
    pr.set_jit_enabled(0)   # random projections with the interpreter (no NVRTC compile of their plans here)
    try:
        for seed in (2, 5, 7, 11):
            sj, recs, data, off = gen_case(seed, n=700)
            rng = random.Random(seed)
            cols = _random_projection(rng, _names(sj))
            f = O.ocf_file(sj, recs, [1, 30, 400], rng)
            _assert_selected(pr.deserialize_ocf(f, 3, columns=cols), _oracle_batches(coracle, sj, data, off, 700, 3), cols, expected_schema(sj))
    finally:
        pr.set_jit_enabled(-1)
    sj, recs = kafka(3000, 13)
    data, off = po.pack_records(recs)
    want = _oracle_batches(coracle, sj, data, off, 3000, 2)
    f = O.ocf_file(sj, recs, counts=O.counts_with_edges(3000, 2), rng=random.Random(4))
    for cols in KAFKA_PROJECTIONS:
        _assert_selected(pr.deserialize_ocf(f, 2, columns=cols), want, cols, expected_schema(sj))


def test_gpu_offsets_walk_counts_every_record_from_zero_after_a_large_decode(coracle):
    """Bug regression: the walk's per-stream counters were never zeroed — on the device they started from whatever the
    lane's local memory held — and accumulated over a block, so a block's total, not a batch's, could overflow i32."""
    sj, recs = kafka(50_000, 14)
    check_datums(coracle, O.ocf_file(sj, recs, [1000, 20_000], random.Random(5)), 2, sj, recs)
    _, f = bug2_file()
    for k in (3, 6):
        check(coracle, f, k)
    with pytest.raises(GpuOcfError) as e:
        gpu_ocf(f, 1)
    assert gpu_error(e.value)[0] == "overflow"


@pytest.mark.timeout(600, method="thread")
def test_gpu_damaged_files(coracle, walker):
    """About 120 damaged files (60 per walker): the device reports what the restated reader decides."""
    from tests.test_gpu_parity import JIT_SEEDS
    seen = {"decoded": 0, "error": 0, "container": 0}
    for seed in range(60) if walker == "jit" else range(300, 360):
        f, k = O.damaged_file(seed, schema_seed=JIT_SEEDS[seed % len(JIT_SEEDS)])
        seen[O.check(coracle, gpu_ocf, gpu_error, f, k)] += 1
    assert seen["error"] > 5, seen


def test_gpu_lowest_failing_record_and_frame_record():
    from tests.test_ocf import _bool_string_blocks
    rng = random.Random(2)
    sj, blocks = _bool_string_blocks([5, 5, 5, 5], rng)
    sync = bytes(range(16, 32))
    blocks[1][2] = b"\x07" + blocks[1][2][1:]
    blocks[3][1] = b"\x02" + blocks[3][1][1:]
    with pytest.raises(GpuOcfError) as e:
        gpu_ocf(O.from_blocks(sj, blocks, sync), 1)
    assert gpu_error(e.value) == ("bool", 7)
    sj, blocks = _bool_string_blocks([3, 4, 5, 2], rng)
    with pytest.raises(GpuOcfError) as e:
        gpu_ocf(O.from_blocks(sj, blocks, sync, bodies={1: b"".join(blocks[1]) + b"\x00"}), 2)
    assert gpu_error(e.value) == ("frame", 6)
