"""world_size-2 gloo tests of the multi-GPU gather's host side: shard partition, the ONE exchange of sizes
(pyruhvro_b200.distributed._all_gather_i64 over the process group), the product's gather plan (csrc/gather.cpp: groups,
prefix offsets, rebase amounts, bit positions) and the semantics of every push job.  The shards are decoded by the host
emulation (tests/emu) and each rank applies its jobs to a zeroed copy of the gathered arena; a bitwise-OR reduce to the
leader stands in for the NVLink stores (the ranks' pushes touch disjoint bytes except for OR-merged bitmap seams).
These byte-wise restatements check the plan, not gather_push_kernel's word-level code: that kernel is tested in
tests/test_gpu_gather.py on one GPU (every rank a separate result on cuda:0) against the oracle, and the NCCL + CUDA
IPC path there with two GPUs."""
import os
import random

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import pyoracle as po
from pyruhvro_b200 import distributed as D
from tests.parity import gen_case


def test_shard_bounds_cover_and_align():
    for n, w in [(10_000_000, 8), (1000, 2), (257, 2), (5, 4), (0, 2), (100_000_003, 8)]:
        b = [D.shard_bounds(n, w, r) for r in range(w)]
        assert b[0][0] == 0 and b[-1][1] == n
        for (a0, a1), (b0, b1) in zip(b, b[1:]):
            assert a1 == b0 and a0 <= a1
        assert all(x[0] % 256 == 0 for x in b if x[0] < n or n == 0)


def test_plan_splits_at_the_i32_ceiling():
    """100 M rows of the Kafka schema hold ~3.3 GB of e-mail bytes: more than one Arrow batch can address.  The plan
    groups consecutive ranks into as few batches as fit (SURVEY.md 8(d) C5)."""
    import workloads
    from tests import emu
    sj, data, off = workloads.generate("kafka", 2000, seed=1)
    sh = emu.Shard(sj, data, off, 2000)
    m = sh.meta()
    per_rank = m * 6250                                   # what a 12.5 M-row shard of the same data would report
    metas = np.stack([per_rank] * 8)
    groups = sh.groups(metas)
    assert len(groups) >= 2 and sum(g[1] for g in groups) == 8 and [g[0] for g in groups] == sorted(g[0] for g in groups)
    assert all(g[3] == 12_500_000 * g[1] for g in groups)
    assert len(sh.groups(np.stack([m] * 8))) == 1          # small shards: one batch


def _worker(rank, world, port, seeds, q):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from tests import emu
    co = po.COracle()
    try:
        for seed in seeds:
            sj, recs, data, off = gen_case(seed, n=random.Random(seed).choice([600, 1000, 1301]))
            n = len(recs)
            r0, r1 = D.shard_bounds(n, world, rank)
            d, o = po.pack_records(recs[r0:r1])
            shard = emu.Shard(sj, d, o, r1 - r0)
            metas = D._all_gather_i64(shard.meta(), None, torch.device("cpu"))       # the product's size exchange
            groups = shard.groups(metas)
            assert len(groups) == 1 and groups[0][0] == 0 and groups[0][1] == world and groups[0][3] == n
            arena = np.zeros(max(groups[0][2], 64), dtype=np.uint8)
            shard.apply(metas, rank, arena)
            t = torch.from_numpy(arena)
            dist.reduce(t, dst=0, op=dist.ReduceOp.BOR)
            if rank == 0:
                batch = shard.export(metas, 0, arena)
                batch.validate(full=True)
                diff = po.canon_diff(po.canon_from_batch(batch), co.decode(sj, recs))
                if diff is not None:
                    raise AssertionError(f"seed {seed}: {diff}")
        q.put((rank, "ok"))
    except Exception as e:  # pragma: no cover
        q.put((rank, f"FAIL {type(e).__name__}: {e}"))
    finally:
        dist.destroy_process_group()


def test_gather_two_ranks_gloo():
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29600 + random.randint(0, 300)
    procs = [ctx.Process(target=_worker, args=(r, world, port, list(range(12)), q)) for r in range(world)]
    for p in procs:
        p.start()
    results = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=60)
    assert all(r[1] == "ok" for r in results), results


def test_plan_grouping_invariants_through_the_c_abi():
    """rv_gather_plan on synthetic per-rank counts (host-only: no CUDA behind it): ranks map to consecutive groups, no
    group exceeds Arrow's i32 ceiling in any row space / stream, the grouping is greedy-minimal (the next rank would not
    have fitted), and a rank that is beyond the ceiling on its own is RV_ERR_OVERFLOW."""
    import ctypes
    import pyruhvro_b200 as pr
    from tests import emu
    L = pr.lib
    L.rv_gather_meta_len.restype = ctypes.c_int64
    L.rv_gather_meta_len.argtypes = [ctypes.c_void_p]
    L.rv_gather_plan.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]
    L.rv_gather_num_groups.argtypes = [ctypes.c_void_p]
    L.rv_gather_group_of_rank.argtypes = [ctypes.c_void_p, ctypes.c_int]
    L.rv_gather_free.argtypes = [ctypes.c_void_p]
    lim, multi, rejected = 2**31 - 1, 0, 0
    for seed in range(400):
        rng = random.Random(seed)
        sj, recs, data, off = gen_case(seed % 40, n=200)
        s = pr._get_or_parse_schema(sj)
        m = emu.Shard(sj, data, off, len(recs)).meta().astype(np.int64)
        assert len(m) == L.rv_gather_meta_len(s.handle)
        world = rng.choice([1, 2, 3, 4, 8, 16])
        metas = np.ascontiguousarray(np.stack([m * rng.choice([0, 1, 1000, 20000, 50000, 100000, 200000, 400000, 800000]) for _ in range(world)]))
        g = ctypes.c_void_p()
        rc = L.rv_gather_plan(s.handle, metas.ctypes.data, world, ctypes.byref(g))
        oversized = any((metas[r] > lim).any() for r in range(world))
        assert (rc != 0) == oversized, (seed, rc, pr._last_error())
        if rc:
            assert rc == 8 and "i32" in pr._last_error()      # RV_ERR_OVERFLOW
            rejected += 1
            continue
        try:
            ng = L.rv_gather_num_groups(g)
            gor = [L.rv_gather_group_of_rank(g, r) for r in range(world)]
            assert gor[0] == 0 and gor[-1] == ng - 1 and all(b - a in (0, 1) for a, b in zip(gor, gor[1:])), gor
            sums = [metas[[r for r in range(world) if gor[r] == k]].sum(axis=0) for k in range(ng)]
            assert not any((t > lim).any() for t in sums)
            for k in range(ng - 1):
                assert ((sums[k] + metas[gor.index(k + 1)]) > lim).any(), (seed, gor)
            multi += ng > 1
        finally:
            L.rv_gather_free(g)
    assert multi > 20 and rejected > 20
