"""Object container files on the CPU: the product's container reader (ocf.cpp) and its per-block record-offsets walk
(ocf_walk.cuh, the body of ocf_offsets_kernel) in the host emulation, against a restated container reader
(oracle/pyoracle.py ocf_read) and the C oracle (the Python decoder for the wider subset) on the writer's datums.  The
device twin is tests/test_gpu_ocf.py."""
import ctypes
import random

import numpy as np
import pytest

import pyruhvro_b200 as pr
from oracle import pyoracle as po
from tests import emu as E
from tests import ocf_files as O
from tests.parity import gen_case, gen_case_wide

# array<null> items take no bytes: a list of 2^23 items is four bytes of block count and a terminator
ZW_SCHEMA = ('{"type":"record","name":"ZW","fields":[{"name":"a","type":{"type":"array","items":"null"}},'
             '{"name":"b","type":"long"}]}')
GEN_SEEDS = [0, 1, 2, 3, 5, 7]
WIDE_SEEDS = [1, 2, 4, 5]
N = 800
RV_ERR_FRAME = 12
BOOL_STR_SCHEMA = '{"type":"record","name":"B","fields":[{"name":"b","type":"boolean"},{"name":"s","type":"string"}]}'


def zw_datum(items: int, b: int) -> bytes:
    return (O.zz(items) if items else b"") + b"\x00" + O.zz(b)


def case(name):
    """(schema, datums, wide) of a named case."""
    kind, _, arg = name.partition(":")
    if kind == "gen":
        sj, recs, _, _ = gen_case(int(arg), n=N)
        return sj, recs, False
    if kind == "wide":
        sj, recs, _, _ = gen_case_wide(int(arg), n=N)
        return sj, recs, True
    if kind == "kafka":
        import workloads
        sj, data, off = workloads.generate("kafka", N, seed=3)
        return sj, [data[off[i]:off[i + 1]].tobytes() for i in range(N)], False
    rng = random.Random(5)
    return ZW_SCHEMA, [zw_datum(rng.choice([0, 1, 3, 1000, 2**20]), rng.randrange(-10**9, 10**9)) for _ in range(N)], False


CASES = [f"gen:{s}" for s in GEN_SEEDS] + [f"wide:{s}" for s in WIDE_SEEDS] + ["kafka", "zero-width"]
LAYOUTS = ["one-record-blocks", "one-block", "chunk-edges", "empty-blocks"]


def layout_counts(layout, n, k, rng):
    if layout == "one-record-blocks":
        return [1] * n
    if layout == "one-block":
        return [n]
    if layout == "chunk-edges":
        return O.counts_with_edges(n, k)
    counts, left = [], n
    while left:
        counts.append(min(left, rng.choice([1, 5, 100, 300])))
        left -= counts[-1]
    return O.with_empty_blocks(counts, rng)


def emu_error(e):
    if isinstance(e, E.EmuContainerError):
        return "container"
    if isinstance(e, E.EmuError):
        return (po.ERR_NAMES.get(e.code, str(e.code)), e.record)
    return None


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("name", CASES)
def test_layouts_decode_like_the_datums(coracle, name, layout):
    sj, recs, wide = case(name)
    rng = random.Random(f"{name}/{layout}")
    for k in (1, 2, 3, 8, N + 5):
        counts = layout_counts(layout, N, k, rng)
        f = O.ocf_file(sj, recs, counts=counts, rng=rng)
        got_sj, datums, blocks = po.ocf_read(f, wide=wide)
        assert got_sj == sj and datums == recs
        assert [c for _, c in blocks] == counts and [b for b, _ in blocks] == list(np.cumsum([0] + counts[:-1]))
        assert O.check(coracle, E.decode_ocf, emu_error, f, k, wide) == "decoded"
    ends = set(np.cumsum(O.counts_with_edges(N, 2)))
    assert {255, 256, 257, 383, 384, 385, 655, 656, 657} <= ends


def test_header_forms(coracle):
    """Metadata over several map blocks in the negative-count form, extra keys, a repeated key (the last value counts), no
    codec key, empty blocks, a sync marker whose bytes occur inside the datums, a file that ends after its header."""
    sj = '{"type":"record","name":"S","fields":[{"name":"s","type":"string"},{"name":"n","type":["null","long"]}]}'
    sync = b"SYNC-MARKER-0123"
    rng = random.Random(4)
    recs = []
    for i in range(600):
        s = rng.choice([b"", b"x", sync, sync * 3, b"pre" + sync + b"post", sync[:9]])
        recs.append(O.zz(len(s)) + s + (b"\x00" if i % 3 == 0 else b"\x02" + O.zz(i * 7919)))
    forms = [
        dict(meta_blocks=2),
        dict(meta_blocks=3, meta_extra=[("user.a", b"1"), ("user.b", b"")]),
        dict(meta_extra=[("avro.schema", b'"not this one"'), ("avro.codec", b"deflate")]),   # the later, standard keys win
        dict(meta_extra={"user.meta": bytes(range(256))}, codec=None),
        dict(codec=None, meta_blocks=2),
    ]
    for form in forms:
        for counts in ([600], [0, 0, 256, 0, 1, 343, 0], [1] * 600):
            f = O.ocf_file(sj, recs, counts=counts, sync=sync, **form)
            assert f.count(sync) > len(counts) + 1
            _, datums, _ = po.ocf_read(f)
            assert datums == recs
            for k in (1, 3):
                assert O.check(coracle, E.decode_ocf, emu_error, f, k) == "decoded"
    header_only = O.ocf_file(sj, [], sync=sync)
    assert header_only == O.ocf_header(sj, sync)
    for f, blocks in ((header_only, []), (O.ocf_file(sj, [], counts=[0, 0], sync=sync, meta_blocks=2), [(0, 0), (0, 0)])):
        assert po.ocf_read(f) == (sj, [], blocks)
        got = E.decode_ocf(f, 4)
        assert len(got) == 1 and got[0].num_rows == 0 and got[0].schema.names == ["s", "n"]
    with pytest.raises(po.ContainerError):
        po.ocf_read(O.ocf_file(sj, recs[:3], counts=[3], sync=sync, codec=b"snappy"))
    with pytest.raises(E.EmuContainerError, match="codec"):
        E.decode_ocf(O.ocf_file(sj, recs[:3], counts=[3], sync=sync, codec=b"snappy"), 1)


@pytest.mark.parametrize("part", range(6))
def test_damaged_files(coracle, part):
    """Damage inside the blocks: the emulated decode reports what the restated reader decides — the same buffers, the same
    category at the same record, or a container error."""
    seen = {"decoded": 0, "error": 0, "container": 0}
    for seed in range(part * 50, part * 50 + 50):
        f, k = O.damaged_file(seed)
        seen[O.check(coracle, E.decode_ocf, emu_error, f, k)] += 1
    assert seen["error"] > 5, seen


def _bool_string_blocks(counts, rng):
    sj = BOOL_STR_SCHEMA
    recs = [bytes([rng.randrange(2)]) + O.zz(3) + b"abc" for _ in range(sum(counts))]
    return sj, O.split(recs, counts)


def test_a_block_whose_records_end_before_its_size_fails_at_its_last_record(coracle):
    rng = random.Random(1)
    sj, blocks = _bool_string_blocks([3, 4, 5, 2], rng)
    sync = bytes(range(16))
    for junk in (b"\x00", b"\x01\x02junk"):
        f = O.from_blocks(sj, blocks, sync, bodies={1: b"".join(blocks[1]) + junk})
        assert O.expected(coracle, f, 1)[0] == ("frame", 6)
        with pytest.raises(E.EmuError) as e:
            E.decode_ocf(f, 1)
        assert (e.value.code, e.value.record) == (RV_ERR_FRAME, 6)
    f = O.from_blocks(sj, blocks, sync, bodies={3: b"".join(blocks[3]) + b"\x01"})     # the file's last block
    assert O.expected(coracle, f, 1)[0] == ("frame", 13)
    with pytest.raises(E.EmuError) as e:
        E.decode_ocf(f, 2)
    assert (e.value.code, e.value.record) == (RV_ERR_FRAME, 13)


def test_the_lowest_failing_record_wins_across_blocks(coracle):
    rng = random.Random(2)
    sj, blocks = _bool_string_blocks([5, 5, 5, 5], rng)
    sync = bytes(range(16, 32))
    blocks[1][2] = b"\x07" + blocks[1][2][1:]        # record 7: not a boolean byte
    blocks[3][1] = b"\x02" + blocks[3][1][1:]        # record 16
    f = O.from_blocks(sj, blocks, sync)
    assert O.expected(coracle, f, 1)[0] == ("bool", 7)
    for k in (1, 4):
        assert O.check(coracle, E.decode_ocf, emu_error, f, k) == "error"
    blocks[2] = blocks[2][:4] + [blocks[2][4][:2]]   # and a block cut short in between: E_FRAME / EOF at 14 loses too
    f = O.from_blocks(sj, blocks, sync)
    assert O.expected(coracle, f, 1)[0] == ("bool", 7)
    assert O.check(coracle, E.decode_ocf, emu_error, f, 2) == "error"


def _forged_files():
    """Block counts beyond the block's bytes: each file must be a container error before anything reaches a device."""
    sj = '{"type":"record","name":"R","fields":[{"name":"x","type":"boolean"}]}'
    sync = bytes(range(100, 116))
    h = O.ocf_header(sj, sync)
    blk = O.ocf_block
    files = {
        "size+1": h + blk(4, b"\x01\x00\x01", sync),
        "2^61-1": h + blk(2**61 - 1, b"\x01", sync) + blk(1, b"\x00", sync),   # offsets of 2^61 records: 8 bytes after the wrap
        "2^63-1": h + blk(2**63 - 1, b"\x01", sync),
        "2^40": h + blk(1, b"\x01", sync) + blk(2**40, b"\x00", sync),
        "5 in 2": h + blk(5, b"\x01\x00", sync),
        "sum": h + blk(1, b"\x01", sync) + b"".join(blk(2**62, b"\x01\x00", sync) for _ in range(4)),   # 1 + 4 * 2^62 wraps i64
        "zero-width": O.ocf_header('{"type":"record","name":"N","fields":[{"name":"z","type":"null"}]}', sync) + blk(3, b"", sync),
    }
    return files


@pytest.mark.parametrize("which", list(_forged_files()))
def test_forged_block_counts_are_container_errors_before_any_cuda_call(which):
    f = _forged_files()[which]
    with pytest.raises(po.ContainerError, match=r"holds \d+ records in \d+ bytes"):
        po.ocf_read(f)
    with pytest.raises(E.EmuContainerError, match=r"holds \d+ records in \d+ bytes"):
        E.decode_ocf(f, 1)
    with pytest.raises(ValueError, match=r"object container file: block \d+ holds \d+ records in \d+ bytes"):
        pr.deserialize_ocf(f, 1)
    buf = np.frombuffer(f, dtype=np.uint8)
    sh, h = ctypes.c_void_p(), ctypes.c_void_p()
    assert pr.lib.rv_decode_ocf_host(buf.ctypes.data, buf.size, 1, ctypes.byref(sh), ctypes.byref(h)) == RV_ERR_FRAME
    assert not sh.value and not h.value


def bug2_file():
    """One block of 600 records of a 2^23-item array<null> and a long (4 KiB): 200 records per batch at k = 3 are 1.68e9
    items per batch, within Arrow's i32 offsets; all 600 in one batch are not."""
    rng = random.Random(9)
    recs = [zw_datum(2**23, rng.randrange(-2**40, 2**40)) for _ in range(600)]
    return recs, O.ocf_file(ZW_SCHEMA, recs, counts=[600], sync=bytes(range(7, 23)))


def test_the_offsets_walk_counts_every_record_of_a_block_from_zero(coracle):
    recs, f = bug2_file()
    assert po.ocf_read(f) == (ZW_SCHEMA, recs, [(0, 600)])
    got = E.decode_ocf(f, 3)
    assert [b.num_rows for b in got] == [200] * 3
    assert O.check(coracle, E.decode_ocf, emu_error, f, 3) == "decoded"
    with pytest.raises(E.EmuError) as e:
        E.decode_ocf(f, 1)
    assert po.ERR_NAMES[e.value.code] == "overflow"
