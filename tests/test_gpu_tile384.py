"""384-record tiles: plans of more than eight streams decoded by the generated walker with one warp per stream.

The tile is a property of the plan and of the shared memory its windows need (engine.cu, choose_tile): 384 rows when
the walker is the generated one, the plan has more than eight streams and two 384-row CTAs fit an SM; 256 otherwise.
The emulation and the other fast-path tests run at 256, so the layout at 384 (tile_of, the scan of twelve records per
lane, the item table, the prefetch of a tile's offsets) is covered here:
  * on the CPU, which plans may take 384-row tiles and the generated kernel source at each tile;
  * on the GPU (`-m gpu`), every buffer against the C oracle at the tile and chunk edges, through a tile on the global
    walk, item-parallel and per-lane list warps, precise warps, both passes of the capacity plan, a projection back to
    256, and the host, device and framed paths — each asserting that the decode really ran at 384."""
import ctypes
import json
import random
import struct

import pytest

import pyruhvro_b200 as pr
from oracle import pyoracle as po
from tests.parity import assert_matches_oracle
from tests.test_gpu_fast_paths import JIT_PROJECTIONS, JIT_SCHEMAS, enc_str, gpu_device, gpu_host, letters, svar, uvar

TILE = 384

# A hand-built plan of eleven streams: five strings, a nullable string, a list of strings (item rows + bytes), a map of
# longs (entry rows + key bytes) and an enum.  Records stay small, so two 384-row CTAs fit whatever the data.
HB_SCHEMA = json.dumps({"type": "record", "name": "T384", "fields": [
    {"name": "id", "type": "long"},
    *[{"name": c, "type": "string"} for c in "abcde"],
    {"name": "ns", "type": ["null", "string"]},
    {"name": "tags", "type": {"type": "array", "items": "string"}},
    {"name": "kv", "type": {"type": "map", "values": "long"}},
    {"name": "en", "type": {"type": "enum", "name": "En", "symbols": ["X", "YY", "ZZZ"]}},
]})


# column projections of the Kafka plan (twelve streams) down to eight or fewer
KAFKA_PROJECTIONS = [["name", "age", "created_at"], ["emails", "phone_numbers"], ["address", "status", "class"]]


def hb_record(rng, r, n_tags=None, padded=False, big=0) -> bytes:
    """One HB_SCHEMA record.  n_tags: items of `tags` (default 0-4, within the item table); padded: `ns`'s union branch
    written as 82 00 (valid, not plain: the warp emits with the precise walker); big: length of `a`."""
    out = bytearray(svar(r))
    for c in "abcde":
        out += enc_str(letters(rng, big if (c == "a" and big) else rng.randint(0, 10)))
    if rng.random() < 0.3 and not padded:
        out += b"\x00"
    else:
        out += (uvar(2, 2) if padded else b"\x02") + enc_str(letters(rng, rng.randint(0, 8)))
    tags = [enc_str(letters(rng, rng.randint(0, 6))) for _ in range(rng.randint(0, 4) if n_tags is None else n_tags)]
    out += (svar(len(tags)) + b"".join(tags) if tags else b"") + b"\x00"
    kv = rng.randint(0, 2)
    out += (svar(kv) + b"".join(enc_str(letters(rng, rng.randint(1, 4))) + svar(rng.randint(-9999, 9999)) for _ in range(kv)) if kv else b"") + b"\x00"
    out += svar(rng.randrange(3))
    return bytes(out)


def hb_case(n, seed=0, special=None):
    """n records; special: {row: hb_record keyword arguments} for chosen rows."""
    rng = random.Random(seed)
    recs = [hb_record(rng, r, **(special or {}).get(r, {})) for r in range(n)]
    return recs, *po.pack_records(recs)


def kafka_case(n, seed=7):
    import workloads
    sj, data, off = workloads.generate("kafka", n, seed=seed)
    return sj, data, off


def lib_tile():
    return pr.lib.rv_last_tile()


def kernel_source(sj, tile, columns=None):
    s = pr._get_or_parse_schema(sj, columns)
    n = pr.lib.rv_schema_kernel_source(s.handle, tile, None, 0)
    assert n > 0
    buf = ctypes.create_string_buffer(n + 1)
    pr.lib.rv_schema_kernel_source(s.handle, tile, buf, n + 1)
    return buf.value.decode()


def max_tile(sj, columns=None):
    return pr.lib.rv_schema_max_tile(pr._get_or_parse_schema(sj, columns).handle)


# ==== CPU: which plans may take 384-row tiles ======================================================================
def test_plans_of_at_most_eight_streams_keep_256_row_tiles():
    import workloads
    plans = [(workloads.FLAT_SCHEMA, None)] + [(sj, None) for sj in JIT_SCHEMAS] + list(JIT_PROJECTIONS)
    plans += [(workloads.KAFKA_SCHEMA, cols) for cols in KAFKA_PROJECTIONS]
    for sj, cols in plans:
        assert max_tile(sj, cols) == 256, (sj, cols)
        src = kernel_source(sj, 256, cols)
        assert "#define RV_KBLOCK 256\n" in src and "__launch_bounds__(rv::kBlock, 3)" in src
        assert pr.lib.rv_schema_kernel_source(pr._get_or_parse_schema(sj, cols).handle, TILE, None, 0) == -1


def test_plans_of_more_than_eight_streams_may_take_384_row_tiles():
    import workloads
    for sj in (workloads.KAFKA_SCHEMA, workloads.WIDE_SCHEMA, HB_SCHEMA):
        assert max_tile(sj) == TILE
        src = kernel_source(sj, TILE)
        assert "#define RV_KBLOCK 384\n" in src and "__launch_bounds__(rv::kBlock, 2)" in src
        assert "#define RV_KBLOCK 256\n" in kernel_source(sj, 256)   # the fallback when two 384-row CTAs do not fit
    assert "items_par_" in pr.Schema(HB_SCHEMA).walker_source     # `tags` is emitted item-parallel


def test_hand_built_cases_reach_their_edges(coracle):
    """The special records are what the GPU tests claim: a record larger than any input window the plan gets (1.5 times
    the mean tile, engine.cu configure), and a padded union branch the oracle reads like the canonical one."""
    n = 20_000
    recs, data, off = hb_case(n, seed=3, special={9_000: {"big": 60_000}})
    assert len(recs[9_000]) > 1.5 * (len(data) / n) * TILE
    rng = random.Random(0)
    padded = hb_record(rng, 7, padded=True)
    plain = padded.replace(b"\x82\x00", b"\x02", 1)
    assert padded != plain and coracle.decode(HB_SCHEMA, [padded]) == coracle.decode(HB_SCHEMA, [plain])


# ==== GPU ===========================================================================================================
@pytest.fixture
def jit():
    pr.set_jit_enabled(1)
    yield
    pr.set_jit_enabled(-1)


def both_paths(coracle, sj, data, off, n, k, slow_tiles=0):
    """Host path and device path, each after a warm-up call; both must run the generated walker at 384 rows."""
    got, slow = gpu_host(sj, data, off, n, k)
    assert pr.last_walker() == "jit" and lib_tile() == TILE
    assert slow == slow_tiles if slow_tiles == 0 else slow >= slow_tiles
    assert_matches_oracle(coracle, got, sj, data, off, n, k)
    got, slow = gpu_device(sj, data, off, n, k)
    assert pr.last_walker() == "jit" and lib_tile() == TILE
    assert slow == slow_tiles if slow_tiles == 0 else slow >= slow_tiles
    assert_matches_oracle(coracle, got, sj, data, off, n, k)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [383, 384, 385, 767, 768, 769])
def test_gpu_rows_at_tile_edges(coracle, jit, n):
    recs, data, off = hb_case(n, seed=n)
    both_paths(coracle, HB_SCHEMA, data, off, n, 1)
    sj, data, off = kafka_case(n)
    both_paths(coracle, sj, data, off, n, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3, 8])
def test_gpu_chunks_not_multiples_of_the_tile(coracle, jit, k):
    n = 5003     # 5003 / 3 = 1667 and 5003 / 8 = 625 rows per chunk, the last chunk takes the rest
    recs, data, off = hb_case(n, seed=k)
    both_paths(coracle, HB_SCHEMA, data, off, n, k)
    sj, data, off = kafka_case(20_011)
    both_paths(coracle, sj, data, off, 20_011, k)


@pytest.mark.gpu
def test_gpu_oversized_record_takes_the_global_walk(coracle, jit):
    n = 20_000
    recs, data, off = hb_case(n, seed=3, special={9_000: {"big": 60_000}})
    both_paths(coracle, HB_SCHEMA, data, off, n, 3, slow_tiles=1)


@pytest.mark.gpu
def test_gpu_per_lane_lists_and_precise_warps_next_to_item_parallel_warps(coracle, jit):
    n = 3 * TILE + 100
    special = {r: {"n_tags": 5 + r % 4} for r in (5, 40, 41, TILE + 31, 2 * TILE + 64)}     # > kItemSlots items
    special.update({r: {"padded": True} for r in (70, TILE + 32 * 11 + 31, 2 * TILE + 3)})  # not plain: precise warps
    recs, data, off = hb_case(n, seed=4, special=special)
    for k in (1, 2):
        both_paths(coracle, HB_SCHEMA, data, off, n, k)


@pytest.mark.gpu
def test_gpu_measuring_pass_then_exact_pass(coracle, jit):
    """The first call on the schema measures (two passes), the same data again takes one; data whose strings outgrow the
    plan repeats once with exact sizes — all at 384 rows."""
    schema = pr._get_or_parse_schema(HB_SCHEMA)
    pr.lib.rv_schema_forget_stats(schema.handle)
    recs, data, off = hb_case(4000, seed=5)
    assert_matches_oracle(coracle, pr.decode_packed(data, off, len(recs), HB_SCHEMA, 3), HB_SCHEMA, data, off, len(recs), 3)
    assert pr.lib.rv_last_passes() == 2 and lib_tile() == TILE
    assert_matches_oracle(coracle, pr.decode_packed(data, off, len(recs), HB_SCHEMA, 3), HB_SCHEMA, data, off, len(recs), 3)
    assert pr.lib.rv_last_passes() == 1 and lib_tile() == TILE
    rng = random.Random(6)
    recs = [hb_record(rng, r, n_tags=rng.randint(3, 4)) for r in range(4000)]
    data, off = po.pack_records(recs)
    assert_matches_oracle(coracle, pr.decode_packed(data, off, len(recs), HB_SCHEMA, 3), HB_SCHEMA, data, off, len(recs), 3)
    assert pr.lib.rv_last_passes() == 2 and lib_tile() == TILE


@pytest.mark.gpu
def test_gpu_projection_to_eight_streams_or_fewer_goes_back_to_256(coracle, jit):
    sj, data, off = kafka_case(10_000)
    full, _ = gpu_host(sj, data, off, 10_000, 3)
    assert lib_tile() == TILE
    assert_matches_oracle(coracle, full, sj, data, off, 10_000, 3)
    for cols in KAFKA_PROJECTIONS:
        got, _ = gpu_host(sj, data, off, 10_000, 3, columns=cols)
        assert pr.last_walker() == "jit" and lib_tile() == 256
        assert [b.schema.names for b in got] == [cols] * 3
        assert all(g.equals(f.select(cols)) for g, f in zip(got, full))


@pytest.mark.gpu
def test_gpu_framed_path(coracle, jit):
    n = 20_011
    sj, data, off = kafka_case(n, seed=9)
    framed = [b"\x00" + struct.pack(">I", 77) + data[off[i]:off[i + 1]].tobytes() for i in range(n)]
    for k in (1, 3, 8):
        pr.deserialize_confluent(framed, sj, k, schema_id=77)
        got = pr.deserialize_confluent(framed, sj, k, schema_id=77)
        assert pr.last_walker() == "jit" and lib_tile() == TILE
        assert_matches_oracle(coracle, got, sj, data, off, n, k, full_validate=False)
    fd, fo = po.pack_records(framed)
    got = pr.decode_packed(fd, fo, n, sj, 2, framing=pr.Framing(5, 1, 77))
    assert lib_tile() == TILE
    assert_matches_oracle(coracle, got, sj, data, off, n, 2, full_validate=False)
