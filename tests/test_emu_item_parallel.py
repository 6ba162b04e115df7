"""Item-parallel list/map emit of the generated walkers (jit.cpp items_par), run through the host emulation with the
lanes of every FAST warp in lock step (tests/emu/warp_walker.cuh), every buffer against the C oracle.  The records are written
by hand so that the cases the emit must get right are certain to occur: warps with more than 32 items (several
rounds), lanes without the list (null branch, lanes past the last record), items spread over several blocks, lists
nested inside an item (per-lane loop inside the item), and warps that fall back to the per-lane loop because a lane
has more than kItemSlots items or its list spans more than 255 bytes."""
import json
import random

import pytest

from oracle import pyoracle as po
from tests import emu
from tests.emu import warp
from tests.parity import gen_case
from tests.parity import assert_matches_oracle

SCHEMA = json.dumps({"type": "record", "name": "R", "fields": [
    {"name": "id", "type": "int"},
    {"name": "tags", "type": ["null", {"type": "array", "items": "string"}]},
    {"name": "attrs", "type": {"type": "map", "values": {"type": "array", "items": "long"}}},
    {"name": "tail", "type": "string"},
]})

K = 4  # dev_types.h kItemSlots


def varint(v: int) -> bytes:
    z = (v << 1) ^ (v >> 63)
    z &= (1 << 64) - 1
    out = bytearray()
    while z >= 0x80:
        out.append((z & 0x7F) | 0x80)
        z >>= 7
    out.append(z)
    return bytes(out)


def string(rng, lo=0, hi=12) -> bytes:
    s = bytes(rng.randrange(97, 123) for _ in range(rng.randint(lo, hi)))
    return varint(len(s)) + s


def blocks(items, rng, split) -> bytes:
    """Items as one block, or (split) as several blocks, then the terminating 0."""
    out = bytearray()
    i = 0
    while i < len(items):
        n = rng.randint(1, len(items) - i) if split else len(items) - i
        out += varint(n) + b"".join(items[i:i + n])
        i += n
    return bytes(out + varint(0))


def record(rng, max_items, split, first_tag=None) -> bytes:
    tags = [string(rng) for _ in range(rng.randint(0, max_items))]
    if first_tag is not None:
        tags[:1] = [first_tag]
    out = bytearray(varint(rng.randint(-1000, 1000)))
    if first_tag is None and rng.random() < 0.3:
        out += varint(0)  # tags: null
    else:
        out += varint(1) + blocks(tags, rng, split)
    entries = []
    for _ in range(rng.randint(0, max_items)):
        longs = [varint(rng.randint(-2**40, 2**40)) for _ in range(rng.randint(0, 3))]
        entries.append(string(rng, 1, 6) + blocks(longs, rng, split))
    out += blocks(entries, rng, split)
    out += string(rng, 0, 20)
    return bytes(out)


def tagged(rng, tags, split=False, n_attrs=None) -> bytes:
    """A record whose `tags` are exactly `tags` (encoded strings; None: the null branch) and with `n_attrs` map
    entries (default: 0 to kItemSlots)."""
    out = bytearray(varint(rng.randint(-1000, 1000)))
    out += varint(0) if tags is None else varint(1) + blocks(tags, rng, split)
    entries = []
    for _ in range(rng.randint(0, K) if n_attrs is None else n_attrs):
        entries.append(string(rng, 1, 6) + blocks([varint(rng.randint(-99, 99)) for _ in range(rng.randint(0, 3))], rng, split))
    out += blocks(entries, rng, split)
    out += string(rng, 0, 20)
    return bytes(out)


def tags_span(tags) -> int:
    """Bytes of the list from after the union branch to after its terminating block (one block): `e = c.pos - l0`."""
    return len(blocks(tags, None, False))


def boundary_cases():
    """(name, records) at the edges of the item-parallel emit.  In all but `one_lane_five` and `span_256` every lane
    has at most kItemSlots items and its list spans at most 255 bytes."""
    rng = random.Random(77)
    four = [tagged(rng, [string(rng) for _ in range(K)], split=i % 2 == 1, n_attrs=K) for i in range(96)]
    five = [record(rng, K, False) for _ in range(96)]
    five[45] = tagged(rng, [string(rng) for _ in range(K + 1)])            # warp 1 only: kItemSeq
    tag_255 = [varint(251) + bytes(rng.randrange(97, 123) for _ in range(251))]
    tag_256 = [varint(252) + bytes(rng.randrange(97, 123) for _ in range(252))]
    assert tags_span(tag_255) == 255 and tags_span(tag_256) == 256
    span = [record(rng, K, False) for _ in range(96)]
    span[10] = tagged(rng, tag_255)                                        # warp 0 stays item-parallel
    span[70] = tagged(rng, tag_256)                                        # warp 2 falls back
    empty = [record(rng, K, False) for _ in range(128)]
    empty[32:64] = [tagged(rng, None, n_attrs=0) for _ in range(32)]       # warp 1: every lane null, no entries
    empty[64:96] = [tagged(rng, [] if i % 2 else None, n_attrs=0) for i in range(32)]  # warp 2: null or empty
    return [("four_each", four), ("one_lane_five", five), ("span_255_256", span), ("empty_warps", empty),
            ("last_warp_1", [record(rng, K, True) for _ in range(97)]),
            ("last_warp_31", [record(rng, K, True) for _ in range(127)])]


BOUNDARY = [name for name, _ in boundary_cases()]


@pytest.mark.parametrize("name", BOUNDARY)
def test_item_parallel_boundaries(coracle, name):
    """Exactly kItemSlots items in every lane (four full rounds, 128 items per warp), one lane with kItemSlots + 1, a
    list spanning exactly 255 (item-parallel) and 256 bytes (per-lane), warps whose lanes are all null or empty (zero
    rounds), and a last warp of 1 or 31 records."""
    recs = dict(boundary_cases())[name]
    for k in (1, 3):
        check(coracle, recs, k)


def check(coracle, recs, k=1):
    data, off = po.pack_records(recs)
    assert "items_par_" in emu.walker_source(SCHEMA)
    before = warp.collectives(SCHEMA)
    assert_matches_oracle(coracle, warp.decode(SCHEMA, data, off, len(recs), k), SCHEMA, data, off, len(recs), k)
    assert warp.collectives(SCHEMA) > before  # the warps met (at least at the vote on the item counts)


@pytest.mark.parametrize("n", [1, 33, 700])
@pytest.mark.parametrize("split", [False, True])
def test_items_within_table(coracle, n, split):
    """Every lane has at most kItemSlots items: all warps emit item-parallel (up to 4 rounds of 32 items per list)."""
    rng = random.Random(n * 2 + split)
    check(coracle, [record(rng, K, split) for _ in range(n)], k=2 if n > 1 else 1)


def test_items_beyond_table_fall_back_per_warp(coracle):
    """A lane with more than kItemSlots items sends its warp (only) to the per-lane loop; the other warps of the
    tile stay item-parallel."""
    rng = random.Random(5)
    recs = [record(rng, K, True) for _ in range(512)]
    for r in (3, 40, 41, 300):  # warps 0, 1, 9
        recs[r] = record(rng, 9, True)
    check(coracle, recs, k=1)


def test_list_over_255_bytes_falls_back(coracle):
    """Item positions are byte offsets from the list's start: a list spanning more than 255 bytes makes its warp loop per lane."""
    rng = random.Random(6)
    recs = [record(rng, K, False) for _ in range(96)]
    long_tag = bytes(rng.randrange(97, 123) for _ in range(300))
    recs[37] = record(rng, K, False, first_tag=varint(len(long_tag)) + long_tag)
    check(coracle, recs, k=1)


@pytest.mark.parametrize("seed", range(100, 112))
def test_random_schemas_in_lock_step(coracle, seed):
    """The random schemas the per-lane emulation of the generated walkers runs (test_emu_parity), with the item-parallel emit."""
    sj, recs, data, off = gen_case(seed)
    k = random.Random(seed).choice([1, 2, 5])
    assert_matches_oracle(coracle, warp.decode(sj, data, off, len(recs), k), sj, data, off, len(recs), k)


def test_workloads_in_lock_step(coracle):
    """The benchmark's schemas: Kafka (two lists of 0-3 items, several rounds per warp), three maps of 0-8 entries (C4)."""
    import workloads
    for name in ("kafka", "wide", "array_map"):
        sj, data, off = workloads.generate(name, 1500, seed=7)
        before = warp.collectives(sj)
        assert_matches_oracle(coracle, warp.decode(sj, data, off, 1500, 3), sj, data, off, 1500, 3)
        met = warp.collectives(sj) - before
        # Kafka: every warp hands out its items (scans, owner searches, carries): far more than one vote per list
        assert met > (10 * 2 * 1500 // 32 if name == "kafka" else 0)
