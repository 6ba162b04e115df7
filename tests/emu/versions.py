"""Host emulation of the multi-version Confluent decode (versions.cpp around resolve.cpp): the product's header check,
output layout, take job tables and per-row take steps, with one emulated resolved decode per (output chunk, writer)
group.  Test infrastructure, like the rest of tests/emu."""
import ctypes
import os
import subprocess

import numpy as np
import pyarrow as pa

from tests import emu
from tests.emu import resolve

SRC = os.path.join(emu.HERE, "versions.cpp")
SRCS = [SRC] + emu.SRCS[1:] + [os.path.join(emu.CSRC, "versions.cpp")]
DEPS = resolve.DEPS + [SRC] + [os.path.join(emu.CSRC, f) for f in ("versions.cpp", "versions.hpp", "take.cuh")]
_lib = None


def _load():
    global _lib
    if _lib is None:
        gdir = os.path.join(emu.HERE, "_gen")
        os.makedirs(gdir, exist_ok=True)
        so = os.path.join(gdir, "libemu_versions.so")
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in DEPS):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-w", "-x", "c++", "-o", tmp] + SRCS)
            os.replace(tmp, so)
        vp, i64 = ctypes.c_void_p, ctypes.c_int64
        lib = ctypes.CDLL(so)
        lib.emu_decode_versions.argtypes = [ctypes.c_char_p, ctypes.c_size_t, vp, vp, i64, vp, vp, i64, i64, vp, i64, vp, vp,
                                            ctypes.POINTER(i64), ctypes.POINTER(i64), ctypes.c_char_p, ctypes.c_size_t]
        _lib = lib
    return _lib


def decode(writer_schemas: dict, reader_json: str, data, offsets, n: int, num_chunks: int = 1, columns=None):
    """The batches of Confluent messages `data` / `offsets` whose ids `writer_schemas` maps to writer schemas, read as
    `reader_json`.  Raises emu.EmuError(status, record) like the library's status and "(record N)"."""
    from pyruhvro_b200 import _ArrowArray, _ArrowSchema
    lib = _load()
    items = sorted(writer_schemas.items())
    raw_w = [sj.encode() for _, sj in items]
    wj = (ctypes.c_char_p * len(raw_w))(*raw_w)
    ids = (ctypes.c_int64 * len(items))(*[i for i, _ in items])
    raw_cols = [c.encode() for c in columns] if columns is not None else []
    cols = (ctypes.c_char_p * max(len(raw_cols), 1))(*raw_cols)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    arrs = (_ArrowArray * min(max(num_chunks, 1), max(n, 1)))()
    sch = _ArrowSchema()
    k, rec = ctypes.c_int64(0), ctypes.c_int64(-1)
    msg = ctypes.create_string_buffer(512)
    r = reader_json.encode()
    rc = lib.emu_decode_versions(r, len(r), ctypes.addressof(wj), ctypes.addressof(ids), len(items), data.ctypes.data if data.size else None,
                                 offsets.ctypes.data, n, num_chunks, ctypes.addressof(cols) if columns is not None else None, len(raw_cols),
                                 ctypes.addressof(arrs), ctypes.addressof(sch), ctypes.byref(k), ctypes.byref(rec), msg, 512)
    if rc != 0:
        raise emu.EmuError(rc, rec.value, msg.value.decode())
    schema = pa.Schema._import_from_c(ctypes.addressof(sch))
    return [pa.RecordBatch._import_from_c(ctypes.addressof(arrs[i]), schema) for i in range(k.value)]
