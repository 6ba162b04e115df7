"""Host emulation of the permissive multi-version decode (versions_permissive.cpp around permissive.cpp): the product's
header classification, permissive resolved plans, layout, take job tables and take steps with the null-row path, with
one emulated permissive resolved decode (interpreter walker) per (output chunk, writer) group.  Test infrastructure, like
the rest of tests/emu."""
import ctypes
import os
import subprocess

import numpy as np
import pyarrow as pa

from tests import emu
from tests.emu import permissive

SRC = os.path.join(emu.HERE, "versions_permissive.cpp")
DEPS = permissive.DEPS + [SRC] + [os.path.join(emu.CSRC, f) for f in ("versions.cpp", "versions.hpp", "take.cuh")]
_lib = None


def _load():
    global _lib
    if _lib is None:
        gdir = os.path.join(emu.HERE, "_gen")
        os.makedirs(gdir, exist_ok=True)
        so = os.path.join(gdir, "libemu_versions_permissive.so")
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in DEPS):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-w", "-x", "c++", "-o", tmp, SRC]
                                  + emu.SRCS[1:] + [os.path.join(emu.CSRC, "versions.cpp")])
            os.replace(tmp, so)
        vp, i64 = ctypes.c_void_p, ctypes.c_int64
        lib = ctypes.CDLL(so)
        lib.emu_decode_versions_permissive.argtypes = [ctypes.c_char_p, ctypes.c_size_t, vp, vp, vp, i64, vp, vp, i64, i64, vp, i64, vp, vp,
                                                       ctypes.POINTER(i64), vp, ctypes.POINTER(i64), ctypes.POINTER(i64), ctypes.c_char_p,
                                                       ctypes.c_size_t]
        _lib = lib
    return _lib


def decode(writer_schemas, reader_json: str, data, offsets, n: int, num_chunks: int = 1, columns=None, fingerprints=None):
    """The permissive registry's (batches, [(message, status), ...]) for Confluent messages whose ids `writer_schemas`
    (dict) maps to writer schemas, or with `fingerprints` (dict fingerprint -> writer schema) single-object messages.
    Raises emu.EmuError(status, record) for a fatal error."""
    from pyruhvro_b200 import _ArrowArray, _ArrowSchema
    lib = _load()
    items = sorted((fingerprints or writer_schemas).items())
    raw_w = [sj.encode() for _, sj in items]
    wj = (ctypes.c_char_p * len(raw_w))(*raw_w)
    keys = (ctypes.c_int64 * len(items))(*[i for i, _ in items]) if fingerprints is None else None
    fps = (ctypes.c_uint64 * len(items))(*[i for i, _ in items]) if fingerprints is not None else None
    raw_cols = [c.encode() for c in columns] if columns is not None else []
    cols = (ctypes.c_char_p * max(len(raw_cols), 1))(*raw_cols)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    arrs = (_ArrowArray * min(max(num_chunks, 1), max(n, 1)))()
    sch = _ArrowSchema()
    k, rec, nbad = ctypes.c_int64(0), ctypes.c_int64(-1), ctypes.c_int64(0)
    bad = np.zeros(max(n, 1), dtype=np.uint64)
    msg = ctypes.create_string_buffer(512)
    r = reader_json.encode()
    rc = lib.emu_decode_versions_permissive(r, len(r), ctypes.addressof(wj), ctypes.addressof(keys) if keys is not None else None,
                                            ctypes.addressof(fps) if fps is not None else None, len(items),
                                            data.ctypes.data if data.size else None, offsets.ctypes.data, n, num_chunks,
                                            ctypes.addressof(cols) if columns is not None else None, len(raw_cols), ctypes.addressof(arrs),
                                            ctypes.addressof(sch), ctypes.byref(k), bad.ctypes.data, ctypes.byref(nbad), ctypes.byref(rec), msg, 512)
    if rc != 0:
        raise emu.EmuError(rc, rec.value, msg.value.decode())
    schema = pa.Schema._import_from_c(ctypes.addressof(sch))
    batches = [pa.RecordBatch._import_from_c(ctypes.addressof(arrs[i]), schema) for i in range(k.value)]
    return batches, [(int(b >> 8), int(b & 0xFF)) for b in bad[:nbad.value]]
