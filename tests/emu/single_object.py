"""Host emulation of the single-object partition (single_object.cpp): the product's 64-bit header check and fingerprint
look-up over a whole input, tile by tile.  Test infrastructure, like the rest of tests/emu."""
import ctypes
import os
import subprocess

import numpy as np

from tests import emu

SRC = os.path.join(emu.HERE, "single_object.cpp")
DEPS = [SRC] + [os.path.join(emu.CSRC, f) for f in ("take.cuh", "dev_types.h")]
_lib = None


def _load():
    global _lib
    if _lib is None:
        gdir = os.path.join(emu.HERE, "_gen")
        os.makedirs(gdir, exist_ok=True)
        so = os.path.join(gdir, "libemu_single_object.so")
        if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in DEPS):
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-Wall", "-x", "c++", "-o", tmp, SRC])
            os.replace(tmp, so)
        vp, i64 = ctypes.c_void_p, ctypes.c_int64
        lib = ctypes.CDLL(so)
        lib.emu_partition_single_object.argtypes = [vp, vp, i64, i64, vp, ctypes.c_int, vp, ctypes.POINTER(i64)]
        _lib = lib
    return _lib


def partition(data, offsets, n: int, k: int, fingerprints):
    """The writer index (into sorted(fingerprints)) of every message.  Raises emu.EmuError(code, record) for the lowest
    failing message: code 12 (short message, not C3 01) or 14 (unregistered fingerprint)."""
    lib = _load()
    fps = np.ascontiguousarray(sorted(fingerprints), dtype=np.uint64)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    writer = np.full(max(n, 1), -2, dtype=np.int32)
    rec = ctypes.c_int64(-1)
    rc = lib.emu_partition_single_object(data.ctypes.data if data.size else None, offsets.ctypes.data, n, k, fps.ctypes.data, len(fps),
                                         writer.ctypes.data, ctypes.byref(rec))
    if rc != 0:
        raise emu.EmuError(rc, rec.value)
    return writer[:n]
