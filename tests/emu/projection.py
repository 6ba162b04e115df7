"""Host emulation of column-projected decodes (projection.cpp around emu.cpp): the product's plan with skip nodes, run
by the interpreter, the generated walker (per lane) or the generated walker with each FAST emit warp in lock step
(warp_walker.cuh).  Test infrastructure, like the rest of tests/emu."""
import ctypes
import hashlib
import os
import subprocess

import numpy as np
import pyarrow as pa

from tests import emu

SRC = os.path.join(emu.HERE, "projection.cpp")
SRCS = [SRC] + emu.SRCS[1:]   # projection.cpp includes emu.cpp
DEPS = emu.DEPS + [SRC, os.path.join(emu.HERE, "warp_walker.cuh")]
ARGTYPES = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64,
            ctypes.c_void_p, ctypes.c_int64, ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int64),
            ctypes.POINTER(ctypes.c_int64), ctypes.c_char_p, ctypes.c_size_t]
_libs = {}


def walker_source(schema_json: str, columns) -> str:
    import pyruhvro_b200 as pr
    return pr.Schema(schema_json).project(columns).walker_source


def build(walker: str, schema_json: str, columns) -> str:
    """walker: "interp", "gen" (per lane) or "warp" (lock-step FAST emit warps)."""
    gdir = os.path.join(emu.HERE, "_gen")
    os.makedirs(gdir, exist_ok=True)
    if walker == "interp":
        so, extra = os.path.join(gdir, "libemu_proj.so"), []
    else:
        src = walker_source(schema_json, columns)
        h = hashlib.sha1(src.encode()).hexdigest()[:16]
        hdr = os.path.join(gdir, f"walker_{h}.cuh")
        if not os.path.exists(hdr):
            with open(hdr, "w") as f:
                f.write(src)
        so = os.path.join(gdir, f"libemu_proj_{walker}_{h}.so")
        if walker == "gen":
            extra = ["-I", emu.CSRC, f'-DEMU_GEN_WALKER="{hdr}"']
        else:
            extra = ["-I", emu.CSRC, f'-DEMU_GEN_WALKER="{os.path.join(emu.HERE, "warp_walker.cuh")}"', f'-DEMU_LANE_WALKER="{hdr}"']
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in DEPS):
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-Wall", "-x", "c++"] + extra + ["-o", tmp] + SRCS)
        os.replace(tmp, so)
    return so


def _lib(walker, schema_json, columns):
    so = build(walker, schema_json, columns)
    lib = _libs.get(so)
    if lib is None:
        lib = _libs[so] = ctypes.CDLL(so)
        lib.emu_decode_projected.argtypes = ARGTYPES
        if walker == "warp":
            lib.emu_warp_collectives.restype = ctypes.c_longlong
    return lib


def collectives(schema_json: str, columns) -> int:
    """Warp collectives the lock-step emulation of this projection's walker has run so far in this process."""
    return _lib("warp", schema_json, columns).emu_warp_collectives()


def decode(schema_json: str, data, offsets, n: int, num_chunks: int, columns, walker: str = "interp"):
    """emu.decode of the projection `columns` (top-level field names, planned by the product's select_columns)."""
    from pyruhvro_b200 import _ArrowArray, _ArrowSchema
    lib = _lib(walker, schema_json, columns)
    raw_cols = [c.encode() for c in columns]
    cols = (ctypes.c_char_p * max(len(raw_cols), 1))(*raw_cols)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    arrs = (_ArrowArray * min(max(num_chunks, 1), max(n, 1)))()
    sch = _ArrowSchema()
    k, rec = ctypes.c_int64(0), ctypes.c_int64(-1)
    msg = ctypes.create_string_buffer(512)
    raw = schema_json.encode()
    rc = lib.emu_decode_projected(raw, len(raw), data.ctypes.data if data.size else None, offsets.ctypes.data, n, num_chunks,
                                  ctypes.addressof(cols), len(raw_cols), ctypes.addressof(arrs), ctypes.addressof(sch),
                                  ctypes.byref(k), ctypes.byref(rec), msg, 512)
    if rc != 0:
        raise emu.EmuError(rc, rec.value, msg.value.decode())
    schema = pa.Schema._import_from_c(ctypes.addressof(sch))
    return [pa.RecordBatch._import_from_c(ctypes.addressof(arrs[i]), schema) for i in range(k.value)]
