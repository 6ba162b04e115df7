"""GPU tests of the multi-GPU gather (pyruhvro_b200.distributed over the C ABI's rv_gather_* entry points): the size
exchange, the plan, the push kernel (offset rebase + bitmap shift fused into the copy) and the result hand-over.

The push kernel's arithmetic runs on one GPU: every "rank" is a separate rv_decode_device result on cuda:0, and the
ranks push into their group's arena in ordinary device memory (_gather_on_one_device).  So bitmaps land at shifted bit
positions with seam words shared between ranks, offsets are rebased, and RAW copies land at every byte alignment.  The
gathered batches are compared with the C oracle (the wider subset: the Python oracle) on the concatenated records, and
every case recomputes from the exchanged sizes which of those paths its pushes reach (_push_paths).  The stand-alone
fix-ups rv_dev_concat_bits / rv_dev_rebase_i32 are compared with numpy.  The same gather also runs as a world of one
through pyruhvro_b200.distributed; with >= 2 visible GPUs two NCCL ranks are spawned and the non-leader pushes into the
leader's arena through CUDA IPC peer memory over NVLink."""
import ctypes
import os
import random
import sys
import threading

import numpy as np
import pyarrow as pa
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _to_device(data, off, dev):
    """Packed records on the device, padded with 64 zero bytes (rv_decode_device reads up to 16 bytes past the end)."""
    import torch
    d_data = torch.zeros(len(data) + 64, dtype=torch.uint8, device=dev)
    d_data[: len(data)].copy_(torch.from_numpy(np.require(data, np.uint8, "CW")))  # torch wants writable arrays
    return d_data, torch.from_numpy(np.require(off, np.int64, "CW")).to(dev)


def _shard(name, n, seed, world, rank, dev):
    import workloads
    from pyruhvro_b200 import distributed as D
    r0, r1 = D.shard_bounds(n, world, rank)
    sj, data, off = workloads.generate(name, r1 - r0, seed=seed, r0=r0)
    d_data, d_off = _to_device(data, off, dev)
    return sj, d_data, d_off, r1 - r0


def _check_against_oracle(name, n, seed, batches):
    import workloads
    from oracle import pyoracle as po
    from tests.parity import expected_schema
    sj, data, off = workloads.generate(name, n, seed=seed)
    assert len(batches) == 1 and batches[0].num_rows == n
    assert batches[0].schema.equals(expected_schema(sj), check_metadata=True)
    diff = po.canon_diff(po.canon_from_batch(batches[0]), po.COracle().decode_packed(sj, data, off, n))
    assert diff is None, diff


def test_gather_world_of_one():
    import torch
    from pyruhvro_b200 import distributed as D
    dev = torch.device("cuda", 0)
    for name, n in [("kafka", 100_003), ("wide", 20_001), ("flat", 70_000), ("array_map", 33_333)]:
        sj, d_data, d_off, n_local = _shard(name, n, 5, 1, 0, dev)
        out = D.decode_and_gather(sj, d_data, d_off, n_local, to_host=True)
        assert out["n_batches"] == 1 and out["remote_bytes"] == 0
        _check_against_oracle(name, n, 5, out["batches"])


# ---- a multi-rank gather on one GPU ---------------------------------------------------------------------------------
def _gather_on_one_device(sj, shards, batch=0, concurrent=False, metas_out=None):
    """Gathers batch `batch` of every shard in `shards` (per-rank packed (data, offsets)) through the C ABI: each shard
    is decoded device-resident on cuda:0 (num_chunks = 3 when batch > 0), the ranks' metas are planned as one world,
    every group's leader arena is allocated and every rank pushes into it, then the group is finished and exported.
    With `concurrent` the ranks of a group push at once, from one Python thread and CUDA stream each (ctypes releases
    the GIL), so their atomicOr's on shared bitmap words overlap.  Returns [(group, RecordBatch)]; `metas_out` receives
    the [world][meta_len] metas the plan was made from.  Every handle is freed."""
    import torch
    import pyruhvro_b200 as pr
    from pyruhvro_b200 import distributed as D
    L = D._lib()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    handles, g, out = [], ctypes.c_void_p(), []
    try:
        for data, off in shards:
            d_data, d_off = _to_device(data, off, dev)
            s, h = D.decode_sharded(sj, d_data, d_off, len(off) - 1, 3 if batch else 1)
            handles.append(h)
        m = int(L.rv_gather_meta_len(s.handle))
        metas = np.zeros((len(shards), max(m, 1)), dtype=np.int64)
        for r, h in enumerate(handles):
            pr._check(L.rv_result_gather_meta(h, batch, metas[r].ctypes.data, m))
        pr._check(L.rv_gather_plan(s.handle, metas.ctypes.data, len(shards), ctypes.byref(g)))
        for gi in range(L.rv_gather_num_groups(g)):
            info = np.zeros(5, dtype=np.int64)
            pr._check(L.rv_gather_group_info(g, gi, info.ctypes.data))
            ranks = range(int(info[0]), int(info[0] + info[1]))
            base = ctypes.c_void_p()
            pr._check(L.rv_gather_alloc(g, gi, stream, ctypes.byref(base)))
            if concurrent:
                streams = {r: torch.cuda.Stream(dev) for r in ranks}
                start, errors = threading.Barrier(len(ranks)), {}

                def push(r):
                    start.wait()
                    if L.rv_gather_push(g, gi, r, handles[r], batch, base, streams[r].cuda_stream):
                        errors[r] = pr._last_error()

                threads = [threading.Thread(target=push, args=(r,)) for r in ranks]
                for t in threads:
                    t.start()
                for t in threads:
                    t.join()
                assert not errors, errors
            else:
                for r in ranks:
                    pr._check(L.rv_gather_push(g, gi, r, handles[r], batch, base, stream))
            res = ctypes.c_void_p()
            pr._check(L.rv_gather_finish(g, gi, ctypes.byref(res)))
            if L.rv_result_to_host(res):
                msg = pr._last_error()
                L.rv_result_free(res)
                raise ValueError(msg)
            out += [(gi, b) for b in pr._export_batches(res.value, s)]
    finally:
        L.rv_gather_free(g)
        for h in handles:
            L.rv_result_free(h)
    if metas_out is not None:
        metas_out.append(metas)
    return out


def _split(data, off, sizes):
    """Packed records -> consecutive shards of `sizes` records, each packed on its own."""
    shards, r0 = [], 0
    for n in sizes:
        shards.append((data[off[r0]: off[r0 + n]], off[r0: r0 + n + 1] - off[r0]))
        r0 += n
    assert r0 == len(off) - 1
    return shards


def _concat(shards, batch=0):
    """The records of batch `batch` of every shard (num_chunks as _gather_on_one_device decodes them), concatenated."""
    from oracle import pyoracle as po
    parts = []
    for data, off in shards:
        n = len(off) - 1
        r0, r1 = po.chunk_bounds(n, po.clamp_chunks(3 if batch else 1, n))[batch]
        parts.append((data[off[r0]: off[r1]], off[r0: r1 + 1] - off[r0]))
    lens = np.concatenate([np.diff(o) for _, o in parts])
    off = np.zeros(len(lens) + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    return np.ascontiguousarray(np.concatenate([d for d, _ in parts]), dtype=np.uint8), off


def _check_gathered(coracle, sj, got, shards, batch=0):
    """One group holding every rank: the gathered batch equals the oracle's decode of the concatenated records."""
    from oracle import pyoracle as po
    from tests.parity import expected_schema
    data, off = _concat(shards, batch)
    assert [g for g, _ in got] == [0]
    b = got[0][1]
    assert b.num_rows == len(off) - 1
    assert b.schema.equals(expected_schema(sj), check_metadata=True)
    b.validate(full=True)
    diff = po.canon_diff(po.canon_from_batch(b), coracle.decode_packed(sj, data, off, len(off) - 1))
    assert diff is None, diff


def _values_width(t):
    """Bytes per row of the array's RAW-pushed values buffer; 0 when it has none (bitmaps and offsets are not RAW)."""
    if pa.types.is_union(t):
        return 1  # type ids
    if pa.types.is_nested(t) or pa.types.is_boolean(t) or pa.types.is_null(t) or pa.types.is_string(t) or pa.types.is_binary(t):
        return 0
    return t.bit_width // 8


def _push_paths(batch, metas):
    """Which paths of gather_push_kernel the planned pushes of `metas` reach, recomputed from the exchanged sizes: rank
    q's buffers land after the rows (row spaces) and totals (streams) of ranks 0..q-1.  `batch` is the gathered batch of
    one group holding every rank; walking its arrays in plan order names each array's row space (the k-th list / map
    opens row space k) and stream (strings, bytes, lists and maps, in order), and says which bitmaps are exported.
    Returns the set of reached paths."""
    nodes, n_sp, n_st = [], 1, 0

    def walk(a, space):
        nonlocal n_sp, n_st
        t = a.type
        stream = None
        if pa.types.is_string(t) or pa.types.is_binary(t) or pa.types.is_list(t) or pa.types.is_map(t):
            stream, n_st = n_st, n_st + 1
        nodes.append((a, space, stream))
        if pa.types.is_struct(t) or pa.types.is_union(t):
            for i in range(t.num_fields):
                walk(a.field(i), space)
        elif pa.types.is_list(t) or pa.types.is_map(t):
            child, n_sp = n_sp, n_sp + 1
            for c in ((a.keys, a.items) if pa.types.is_map(t) else (a.values,)):
                walk(c, child)

    for col in batch.columns:
        walk(col, 0)
    n_valid = metas.shape[1] - n_sp - n_st  # the rest of a meta row: null counts, one per validity bitmap
    assert n_valid >= 0
    rows, tots = metas[:, :n_sp], metas[:, n_sp: n_sp + n_st]
    for a, sp, st in nodes:  # the mapping agrees with what was gathered
        assert len(a) == rows[:, sp].sum()
        if st is not None:
            assert np.frombuffer(a.buffers()[1], dtype=np.int32)[len(a)] == tots[:, st].sum()
    paths, split = set(), []
    for q in range(len(metas)):
        if rows[q, 0] == 0:
            paths.add("empty rank")
        pre_rows, pre_tots = rows[:q].sum(axis=0), tots[:q].sum(axis=0)
        n_bytes, n_jobs = 0, n_valid  # at most one job per validity bitmap, exported or not
        for a, sp, st in nodes:
            t, my, pre = a.type, int(rows[q, sp]), int(pre_rows[sp])
            if st is not None:  # an OFFSETS job, even for no rows
                n_bytes, n_jobs = n_bytes + 4 * my, n_jobs + 1
                if my and pre_tots[st]:
                    paths.add("OFFSETS rebased")
            if not my:
                continue
            exported_validity = not pa.types.is_union(t) and a.buffers()[0] is not None
            n_bytes += (exported_validity + pa.types.is_boolean(t)) * (my // 8)
            n_jobs += pa.types.is_boolean(t)
            if (exported_validity or pa.types.is_boolean(t)) and pre % 32:
                paths.add("BITS at a shifted bit" if sp == 0 else "BITS at a shifted bit, row space > 0")
            raw = [(pre * _values_width(t), my * _values_width(t))] if _values_width(t) else []
            if pa.types.is_string(t) or pa.types.is_binary(t):
                raw.append((int(pre_tots[st]), int(tots[q, st])))
            for dst, count in raw:
                if count:
                    n_bytes, n_jobs = n_bytes + count, n_jobs + 1
                if dst % 2 and count >= 8:  # 1 or 3 mod 4 (slots start 64-byte aligned), with whole words to shift
                    paths.add("RAW at 1|3 mod 4")
                    if pa.types.is_fixed_size_binary(t):
                        paths.add("ValuesW RAW at 1|3 mod 4")
        split.append(n_jobs > 0 and (n_bytes // n_jobs) >> 16 >= 2)  # a lower bound of rv_gather_push's `parts`
    if all(split):
        paths.add("every push split over parts")
    return paths


SHIFTED = {"BITS at a shifted bit", "RAW at 1|3 mod 4", "OFFSETS rebased"}
SHARDINGS = {  # records per rank, and the paths the pushes of the nested random schemas below reach with them
    "empty first": ([0, 1, 7, 31, 32, 33, 255, 257, 300], SHIFTED | {"BITS at a shifted bit, row space > 0", "empty rank"}),
    "empty in the middle": ([33, 257, 0, 7, 1, 300, 31], SHIFTED | {"BITS at a shifted bit, row space > 0", "empty rank"}),
    "empty last": ([255, 1, 32, 0], SHIFTED | {"BITS at a shifted bit, row space > 0", "empty rank"}),
    "shard_bounds(517, 4)": (None, {"empty rank"}),  # fewer than world * 256 rows: all on the last rank
}
NESTED_SEEDS = [6, 20, 24, 33, 35]  # gen_case schemas with nested lists and maps and nullable records (in JIT_SEEDS)


@pytest.mark.parametrize("concurrent", [False, True], ids=["sequential", "concurrent"])
@pytest.mark.parametrize("sharding", list(SHARDINGS))
@pytest.mark.parametrize("seed", NESTED_SEEDS)
def test_gather_random_schemas_uneven_shards(coracle, seed, sharding, concurrent):
    from pyruhvro_b200 import distributed as D
    from tests.parity import gen_case
    sizes, want = SHARDINGS[sharding]
    if sizes is None:
        sizes = [r1 - r0 for r0, r1 in (D.shard_bounds(517, 4, r) for r in range(4))]
    sj, recs, data, off = gen_case(seed, n=sum(sizes))
    shards = _split(data, off, sizes)
    metas = []
    got = _gather_on_one_device(sj, shards, concurrent=concurrent, metas_out=metas)
    _check_gathered(coracle, sj, got, shards)
    paths = _push_paths(got[0][1], metas[0])
    assert want <= paths, (sizes, sorted(paths))


def test_gather_batch_after_the_first(coracle):
    """Batch 1 of shards decoded into 3 chunks: the pushed buffers sit at non-zero offsets of the shard's arena."""
    from tests.parity import gen_case
    sizes = [100, 35, 771, 8]  # chunk 1: 33, 11, 257, 2 records
    for seed in (6, 33):
        sj, recs, data, off = gen_case(seed, n=sum(sizes))
        shards = _split(data, off, sizes)
        metas = []
        got = _gather_on_one_device(sj, shards, batch=1, metas_out=metas)
        _check_gathered(coracle, sj, got, shards, batch=1)
        assert SHIFTED <= _push_paths(got[0][1], metas[0])


@pytest.mark.parametrize("seed", [20, 22, 35])  # gen_case_wide schemas with fixed(1), fixed(7), fixed(3), decimal, uuid
def test_gather_wide_subset(seed):
    import pyruhvro_b200 as pr
    from tests.parity import assert_matches_pyoracle_wide, gen_case_wide
    sizes = [7, 0, 33, 1, 257, 31]
    sj, recs, data, off = gen_case_wide(seed, n=sum(sizes))
    pr.set_jit_enabled(0)
    try:
        metas = []
        got = _gather_on_one_device(sj, _split(data, off, sizes), metas_out=metas)
    finally:
        pr.set_jit_enabled(-1)
    assert [g for g, _ in got] == [0]
    assert_matches_pyoracle_wide([got[0][1]], sj, recs, 1)
    paths = _push_paths(got[0][1], metas[0])
    assert {"ValuesW RAW at 1|3 mod 4", "OFFSETS rebased", "empty rank"} <= paths, sorted(paths)


def test_gather_kafka_split_pushes(coracle):
    """~300 k Kafka rows over 3 uneven ranks: jobs average more than 128 KiB, so every push is split over blockIdx.y
    parts (only part 0 writes a RAW job's head and tail bytes), and string data lands at every alignment."""
    import workloads
    sizes = [70_001, 150_011, 79_993]
    sj, data, off = workloads.generate("kafka", sum(sizes), seed=9)
    shards = _split(data, off, sizes)
    metas = []
    got = _gather_on_one_device(sj, shards, metas_out=metas)
    _check_gathered(coracle, sj, got, shards)
    paths = _push_paths(got[0][1], metas[0])
    assert SHIFTED | {"every push split over parts"} <= paths, sorted(paths)


def test_gather_two_groups_at_the_i32_ceiling():
    """5 ranks of 64 records holding 2^23 zero-width list items each (2^29 per rank): three ranks fit Arrow's i32
    offsets, a fourth would not, so the plan makes groups {0, 1, 2} and {3, 4}, each with offsets starting at 0."""
    from oracle import pyoracle as po
    from tests.parity import expected_schema
    sj = '{"type":"record","name":"Z","fields":[{"name":"a","type":{"type":"array","items":"null"}},{"name":"b","type":"long"}]}'
    shards = [po.pack_records([po.zigzag_bytes(1 << 23) + b"\x00" + po.zigzag_bytes(64 * r + i) for i in range(64)])
              for r in range(5)]
    got = _gather_on_one_device(sj, shards)
    assert [g for g, _ in got] == [0, 1]
    for (_, b), first, n in zip(got, (0, 192), (192, 128)):
        assert b.num_rows == n
        assert b.schema.equals(expected_schema(sj), check_metadata=True)
        a = b.column("a")
        assert a.null_count == 0 and len(a.values) == n << 23
        assert np.array_equal(a.offsets.to_numpy(), np.arange(n + 1, dtype=np.int64) << 23)
        assert np.array_equal(b.column("b").to_numpy(), np.arange(first, first + n, dtype=np.int64))


# ---- the stand-alone fix-ups ----------------------------------------------------------------------------------------
def _fixups():
    import pyruhvro_b200 as pr
    L = pr.lib
    vp, i64 = ctypes.c_void_p, ctypes.c_int64
    L.rv_dev_rebase_i32.argtypes = [vp, vp, i64, ctypes.c_int32, vp]
    L.rv_dev_concat_bits.argtypes = [vp, i64, vp, i64, vp]
    return L


def _words(bits):
    """0/1 per bit (a multiple of 32 of them) -> LSB-first 32-bit words on the device (as int32)."""
    import torch
    return torch.from_numpy(np.packbits(bits, bitorder="little").view(np.int32)).cuda()


def _bits(d_words):
    return np.unpackbits(d_words.cpu().numpy().view(np.uint8), bitorder="little")


def _source(bits):
    """The source bitmap of `bits`, with every bit past them in its last word set (garbage the fix-up must ignore)."""
    src = np.ones(max(1, -(-len(bits) // 32)) * 32, dtype=np.uint8)
    src[: len(bits)] = bits
    return _words(src)


def test_concat_bits_matches_numpy():
    import torch
    L = _fixups()
    stream = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(3)
    for dst_bit in (0, 1, 7, 31, 32, 33, 63, 1_000_003):
        for nbits in (0, 1, 5, 31, 32, 33, 65, 1_000_007):
            bits = rng.integers(0, 2, nbits, dtype=np.uint8)
            before = rng.integers(0, 2, -(-(dst_bit + nbits) // 32) * 32 + 64, dtype=np.uint8)
            before[dst_bit: dst_bit + nbits] = 0  # the range starts zeroed, everything around it is someone else's
            d_dst, d_src = _words(before), _source(bits)
            assert L.rv_dev_concat_bits(d_dst.data_ptr(), dst_bit, d_src.data_ptr(), nbits, stream) == 0
            want = before.copy()
            want[dst_bit: dst_bit + nbits] = bits
            assert np.array_equal(_bits(d_dst), want), (dst_bit, nbits)
    # shards OR'd in sequence into one zeroed bitmap: their concatenation
    shards = [rng.integers(0, 2, n, dtype=np.uint8) for n in (5, 33, 0, 1, 64, 1000, 31, 7, 100_003, 2)]
    total = sum(len(s) for s in shards)
    d_dst = _words(np.zeros(-(-total // 32) * 32 + 32, dtype=np.uint8))
    pos = 0
    for s in shards:
        d_src = _source(s)
        assert L.rv_dev_concat_bits(d_dst.data_ptr(), pos, d_src.data_ptr(), len(s), stream) == 0
        pos += len(s)
    got = _bits(d_dst)
    assert np.array_equal(got[:total], np.concatenate(shards)) and not got[total:].any()


def test_rebase_i32_matches_numpy():
    import torch
    L = _fixups()
    stream = torch.cuda.current_stream().cuda_stream
    rng = np.random.default_rng(4)
    for n in (0, 1, 255, 257, 3_000_000):
        src = rng.integers(-2**30, 2**30, n, dtype=np.int32)
        d_src = torch.from_numpy(src).cuda()
        for add in (0, 1, 987_654_321, -1_000_000_007):
            d_dst = torch.full((n + 64,), -7, dtype=torch.int32, device="cuda")
            assert L.rv_dev_rebase_i32(d_dst.data_ptr(), d_src.data_ptr(), n, add, stream) == 0
            got = d_dst.cpu().numpy()
            assert np.array_equal(got[:n], src + np.int32(add)), (n, add)
            assert (got[n:] == -7).all()


def test_fixups_reject_bad_arguments():
    import torch
    import pyruhvro_b200 as pr
    L = _fixups()
    d = torch.zeros(64, dtype=torch.int32, device="cuda")
    p = d.data_ptr()
    for rc in (L.rv_dev_rebase_i32(p, p, -1, 0, None), L.rv_dev_rebase_i32(None, p, 5, 0, None), L.rv_dev_rebase_i32(p, None, 5, 0, None),
               L.rv_dev_concat_bits(p, 0, p, -1, None), L.rv_dev_concat_bits(p, -1, p, 5, None),
               L.rv_dev_concat_bits(None, 0, p, 5, None), L.rv_dev_concat_bits(p, 0, None, 5, None)):
        assert rc == 9 and "bad argument" in pr._last_error()  # RV_ERR_INVALID
    assert L.rv_dev_rebase_i32(None, None, 0, 5, None) == 0 and L.rv_dev_concat_bits(None, 3, None, 0, None) == 0
    torch.cuda.synchronize()
    assert not d.any()


def _rank_main(rank, world, port, q):
    try:
        os.environ.update({"MASTER_ADDR": "127.0.0.1", "MASTER_PORT": str(port), "RANK": str(rank), "WORLD_SIZE": str(world), "LOCAL_RANK": str(rank)})
        sys.path.insert(0, ROOT)
        import torch
        import torch.distributed as dist
        torch.cuda.set_device(rank)
        dev = torch.device("cuda", rank)
        dist.init_process_group("nccl", device_id=dev)
        from pyruhvro_b200 import distributed as D
        log = []
        for name, n in [("kafka", 100_003), ("wide", 50_001), ("flat", 70_000), ("array_map", 33_333), ("kafka", 517)]:
            sj, d_data, d_off, n_local = _shard(name, n, 5, world, rank, dev)
            out = D.decode_and_gather(sj, d_data, d_off, n_local, to_host=True)
            if rank == 0:
                _check_against_oracle(name, n, 5, out["batches"])
                log.append(f"{name} n={n} world={world}: OK ({out['remote_bytes']} bytes pushed over NVLink)")
            else:
                assert out["batches"] == []
        # timing at a larger size (C5 shape, scaled): device-resident gather
        n = 4_000_000 * world
        sj, d_data, d_off, n_local = _shard("kafka", n, 42, world, rank, dev)
        best = None
        for _ in range(4):
            out = D.decode_and_gather(sj, d_data, d_off, n_local)
            best = out if best is None or out["gather_ms"] < best["gather_ms"] else best
        if rank == 0:
            log.append(f"kafka {n} rows over {world} GPUs: shard decode {best['decode_ms']:.2f} ms, gather {best['gather_ms']:.2f} ms, "
                       f"{best['remote_bytes'] / 1e9:.2f} GB over NVLink = {best['remote_bytes'] / best['gather_ms'] / 1e6:.0f} GB/s")
        dist.barrier(device_ids=[rank])
        dist.destroy_process_group()
        q.put((rank, "ok", log))
    except Exception as e:  # pragma: no cover
        import traceback
        q.put((rank, "FAIL " + traceback.format_exc()[-1500:], []))


def test_gather_two_gpus_nccl_ipc():
    import torch
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two visible GPUs")
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29700 + random.randint(0, 200)
    procs = [ctx.Process(target=_rank_main, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert all(r[1] == "ok" for r in results), results
    lines = [l for r in results for l in r[2]]
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    with open(os.path.join(ROOT, "gpurun_out", "gather_2gpu.log"), "w") as f:
        f.write("\n".join(lines) + "\n")
    print("\n".join(lines))
