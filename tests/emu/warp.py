"""Host emulation of the generated walkers with each FAST emit warp run in lock step (warp_walker.cuh around emu.cpp),
so that the item-parallel list/map emit — warp shuffles, votes, scans and the item-position table — runs as on the
device.  Test infrastructure, like the rest of tests/emu."""
import ctypes
import hashlib
import os
import subprocess

import numpy as np
import pyarrow as pa

from tests import emu

DEPS = emu.DEPS + [os.path.join(emu.HERE, "warp_walker.cuh")]
_libs = {}


def build(gen_source: str) -> str:
    h = hashlib.sha1(gen_source.encode()).hexdigest()[:16]
    gdir = os.path.join(emu.HERE, "_gen")
    os.makedirs(gdir, exist_ok=True)
    hdr = os.path.join(gdir, f"walker_{h}.cuh")
    if not os.path.exists(hdr):
        with open(hdr, "w") as f:
            f.write(gen_source)
    so = os.path.join(gdir, f"libemu_warp_{h}.so")
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in DEPS):
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-Wall", "-x", "c++", "-I", emu.CSRC,
                               f'-DEMU_GEN_WALKER="{os.path.join(emu.HERE, "warp_walker.cuh")}"', f'-DEMU_LANE_WALKER="{hdr}"',
                               "-o", tmp] + emu.SRCS)
        os.replace(tmp, so)
    return so


def collectives(schema_json: str) -> int:
    """Warp collectives the emulation of this schema's walker has run so far in this process."""
    return _lib(schema_json).emu_warp_collectives()


def _lib(schema_json: str):
    so = build(emu.walker_source(schema_json))
    lib = _libs.get(so)
    if lib is None:
        lib = _libs[so] = ctypes.CDLL(so)
        lib.emu_warp_collectives.restype = ctypes.c_longlong
        lib.emu_decode.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64,
                                   ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int64),
                                   ctypes.c_char_p, ctypes.c_size_t]
    return lib


def decode(schema_json: str, data, offsets, n: int, num_chunks: int = 1):
    """emu.decode(..., walker="gen") with the item-parallel emit in use."""
    from pyruhvro_b200 import _ArrowArray, _ArrowSchema
    lib = _lib(schema_json)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    arrs = (_ArrowArray * min(max(num_chunks, 1), max(n, 1)))()
    sch = _ArrowSchema()
    k, rec = ctypes.c_int64(0), ctypes.c_int64(-1)
    msg = ctypes.create_string_buffer(512)
    raw = schema_json.encode()
    rc = lib.emu_decode(raw, len(raw), data.ctypes.data if data.size else None, offsets.ctypes.data, n, num_chunks,
                        ctypes.addressof(arrs), ctypes.addressof(sch), ctypes.byref(k), ctypes.byref(rec), msg, 512)
    if rc != 0:
        raise emu.EmuError(rc, rec.value, msg.value.decode())
    schema = pa.Schema._import_from_c(ctypes.addressof(sch))
    return [pa.RecordBatch._import_from_c(ctypes.addressof(arrs[i]), schema) for i in range(k.value)]
