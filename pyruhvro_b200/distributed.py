"""Multi-GPU decode: one process per GPU (torch.distributed), records sharded by message.

The reference's own contract needs no collective: `per_datum_deserialize_threaded` returns one RecordBatch per
contiguous chunk (ruhvro/src/deserialize.rs:57-68,115-119), and rank g decoding rows `shard_bounds(n, world, g)` yields
exactly those batches.  `decode_sharded` is that path.

When single RecordBatches over all ranks' rows are wanted (BASELINE.json configs[4]) the shards are gathered through
the C ABI's gather entry points (include/ruhvro_b200.h, csrc/gather.hpp):

  1. one small collective: every rank's `rv_gather_meta_len()` int64 counts (rows per row space, stream totals, null
     counts) are all-gathered — the only exchange of sizes, no per-buffer round trips;
  2. every rank computes the same plan (`rv_gather_plan`): consecutive ranks are grouped into as few batches as Arrow's
     i32 offsets allow (100 M rows of the Kafka schema need two), each group led by its first rank;
  3. the leader allocates the gathered arena on its GPU and shares it with its group through a CUDA IPC handle;
  4. every member pushes its buffers into that arena with ONE kernel (`rv_gather_push`): stores straight into the
     leader's memory over NVLink/NVSwitch at the exchanged prefix offsets, Arrow offsets rebased and bitmaps
     bit-shifted inside the same kernel (seam words merged with atomic OR);
  5. after a barrier the leader owns an ordinary device-resident result (`rv_gather_finish`): it can stay in HBM or go
     to pinned host memory once — not once per rank.

torch is used for what it is here for: the process group, device tensors and streams.
"""
from __future__ import annotations

import ctypes
import time
from typing import List, Optional

import numpy as np
import pyarrow as pa

INT32_MAX = 2**31 - 1


def shard_bounds(n: int, world: int, rank: int, align: int = 256):
    """Contiguous row range of `rank`: build_slices semantics (floor division, remainder to the last
    rank) with shard starts aligned to `align` rows so top-level bitmaps concatenate on word boundaries."""
    base = (n // world) // align * align if world > 1 else n
    if base == 0:  # tiny inputs: everything on the last rank
        return (0, 0) if rank < world - 1 else (0, n)
    r0 = rank * base
    return (r0, n) if rank == world - 1 else (r0, r0 + base)


_bound = False


def _lib():
    from . import lib
    global _bound
    if not _bound:
        vp, i64 = ctypes.c_void_p, ctypes.c_int64
        lib.rv_gather_meta_len.restype = i64
        lib.rv_gather_meta_len.argtypes = [vp]
        lib.rv_result_gather_meta.argtypes = [vp, i64, vp, i64]
        lib.rv_gather_plan.argtypes = [vp, vp, ctypes.c_int, ctypes.POINTER(vp)]
        lib.rv_gather_num_groups.argtypes = [vp]
        lib.rv_gather_group_of_rank.argtypes = [vp, ctypes.c_int]
        lib.rv_gather_group_info.argtypes = [vp, ctypes.c_int, vp]
        lib.rv_gather_alloc.argtypes = [vp, ctypes.c_int, vp, ctypes.POINTER(vp)]
        lib.rv_gather_push.argtypes = [vp, ctypes.c_int, ctypes.c_int, vp, i64, vp, vp]
        lib.rv_gather_finish.argtypes = [vp, ctypes.c_int, ctypes.POINTER(vp)]
        lib.rv_gather_free.argtypes = [vp]
        lib.rv_gather_free.restype = None
        lib.rv_ipc_export.argtypes = [vp, vp]
        lib.rv_ipc_open.argtypes = [vp, ctypes.POINTER(vp)]
        lib.rv_ipc_close.argtypes = [vp]
        _bound = True
    return lib


def decode_sharded(schema_json: str, d_data, d_offsets, n_local: int, num_chunks: int = 1, *, columns=None, reader_schema=None):
    """This rank's shard -> device-resident result handle (the reference's per-chunk batches; no collective).
    `columns`: a column projection (top-level field names, pyruhvro_b200.Schema.project).  `reader_schema`: the schema to
    read the data as (pyruhvro_b200.Schema.read_as); `schema_json` is the one it was written with."""
    import torch
    from . import _check, _get_or_parse_schema, lib
    s = _get_or_parse_schema(schema_json, columns, reader_schema)
    h = ctypes.c_void_p()
    _check(lib.rv_decode_device(s.handle, d_data.data_ptr(), d_offsets.data_ptr(), n_local, num_chunks,
                                torch.cuda.current_stream().cuda_stream, ctypes.byref(h)))
    return s, h


def _all_gather_i64(local: np.ndarray, group, device) -> np.ndarray:
    """[world][len(local)] int64 — the one exchange of sizes."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        return local.reshape(1, -1).copy()
    t = torch.from_numpy(local.copy()).to(device)
    out = torch.empty(world * local.size, dtype=torch.int64, device=device)
    dist.all_gather_into_tensor(out, t, group=group)
    return out.cpu().numpy().reshape(world, -1)


def _all_gather_u8(local: np.ndarray, group, device) -> np.ndarray:
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if world == 1:
        return local.reshape(1, -1).copy()
    t = torch.from_numpy(local.copy()).to(device)
    out = torch.empty(world * local.size, dtype=torch.uint8, device=device)
    dist.all_gather_into_tensor(out, t, group=group)
    return out.cpu().numpy().reshape(world, -1)


def gather_result(schema, h, group=None, batch: int = 0):
    """Gathers batch `batch` of every rank's device-resident result `h` into single batches.  Returns
    (result handles this rank leads [(group index, rv_result*)], info dict).  Collective: every rank must call it."""
    import torch
    import torch.distributed as dist
    from . import _check
    L = _lib()
    dev = torch.device("cuda", torch.cuda.current_device())
    stream = torch.cuda.current_stream().cuda_stream
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    comm_dev = dev if (world > 1 and dist.get_backend(group) == "nccl") else torch.device("cpu")

    m = int(L.rv_gather_meta_len(schema.handle))
    meta = np.zeros(max(m, 1), dtype=np.int64)
    _check(L.rv_result_gather_meta(h, batch, meta.ctypes.data, m))
    metas = np.ascontiguousarray(_all_gather_i64(meta, group, comm_dev))                      # (1) sizes, once
    g = ctypes.c_void_p()
    _check(L.rv_gather_plan(schema.handle, metas.ctypes.data, world, ctypes.byref(g)))        # (2) same plan everywhere
    try:
        gi = L.rv_gather_group_of_rank(g, rank)
        info = np.zeros(5, dtype=np.int64)
        _check(L.rv_gather_group_info(g, gi, info.ctypes.data))
        leader, n_members = int(info[0]), int(info[1])
        handle = np.zeros(64, dtype=np.uint8)
        base = ctypes.c_void_p()
        if rank == leader:                                                                    # (3) arena on the leader
            _check(L.rv_gather_alloc(g, gi, stream, ctypes.byref(base)))
            if n_members > 1:
                _check(L.rv_ipc_export(base, handle.ctypes.data))
        remote = None
        if world > 1:
            handles = _all_gather_u8(handle, group, comm_dev)
            if rank != leader:
                remote = ctypes.c_void_p()
                hl = np.ascontiguousarray(handles[leader])
                _check(L.rv_ipc_open(hl.ctypes.data, ctypes.byref(remote)))
                base = remote
        _check(L.rv_gather_push(g, gi, rank, h, batch, base, stream))                         # (4) one kernel per rank
        if world > 1:
            dist.barrier(group=group) if comm_dev.type == "cpu" else dist.barrier(group=group, device_ids=[dev.index])
        if remote is not None:
            L.rv_ipc_close(remote)
        led = []
        if rank == leader:                                                                    # (5) an ordinary result
            out = ctypes.c_void_p()
            _check(L.rv_gather_finish(g, gi, ctypes.byref(out)))
            led.append((gi, out))
        n_groups = L.rv_gather_num_groups(g)
        total = {"n_batches": n_groups, "gathered_bytes": 0, "remote_bytes": 0}
        for i in range(n_groups):
            gin = np.zeros(5, dtype=np.int64)
            _check(L.rv_gather_group_info(g, i, gin.ctypes.data))
            total["gathered_bytes"] += int(gin[2])
            total["remote_bytes"] += int(gin[4])
        return led, total
    finally:
        L.rv_gather_free(g)


def decode_and_gather(schema_json: str, d_data, d_offsets, n_local: int, group=None, timing: bool = False, to_host: bool = False, *,
                      columns=None, reader_schema=None):
    """Decode this rank's shard on its GPU, then gather into single RecordBatches on the group leaders.
    Returns a dict: `batches` (pyarrow RecordBatches when to_host, else live rv_result handles freed here), timings."""
    import torch
    from . import _check, _export_batches, lib
    t0 = time.perf_counter()
    s, h = decode_sharded(schema_json, d_data, d_offsets, n_local, 1, columns=columns, reader_schema=reader_schema)
    torch.cuda.synchronize()
    t1 = time.perf_counter()
    try:
        led, info = gather_result(s, h, group=group)
    finally:
        lib.rv_result_free(h)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    batches = []
    for _, res in led:
        if to_host:
            _check(lib.rv_result_to_host(res))
            batches += _export_batches(res.value, s)
        else:
            lib.rv_result_free(res)
    out = dict(info)
    out.update({"decode_ms": 1e3 * (t1 - t0), "gather_ms": 1e3 * (t2 - t1), "batches": batches, "launches": 2,
                "how": "sizes all-gathered once; per-rank push kernel into the leader's arena over NVLink (CUDA IPC peer memory), "
                       "offset rebase + bitmap shift fused; gathered batches stay device-resident on the leaders"})
    return out


def decode_sharded_gather(schema_json: str, d_data, d_offsets, n_local: int, group=None, *, columns=None,
                          reader_schema=None) -> List[pa.RecordBatch]:
    """Decode + gather; the group leaders (rank 0 when everything fits one batch) get the gathered RecordBatches in
    pinned host memory, the other ranks an empty list."""
    return decode_and_gather(schema_json, d_data, d_offsets, n_local, group=group, to_host=True, columns=columns,
                             reader_schema=reader_schema)["batches"]
