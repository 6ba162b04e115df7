"""Host emulation of permissive decodes (permissive.cpp around projection.cpp and emu.cpp): the product's permissive
plan, run by the interpreter, the generated walker (per lane) or the generated walker with each FAST emit warp in lock
step (warp_walker.cuh), with the kernel's per-lane protocol for bad records.  Test infrastructure, like the rest of
tests/emu."""
import ctypes
import hashlib
import os
import subprocess

import numpy as np
import pyarrow as pa

from tests import emu
from tests.emu import projection

SRC = os.path.join(emu.HERE, "permissive.cpp")
SRCS = [SRC] + emu.SRCS[1:]   # permissive.cpp includes projection.cpp, which includes emu.cpp
DEPS = projection.DEPS + [SRC]
_libs = {}

SINGLE_OBJECT = 3   # dev_types.h kFrameSingleObject


def schema(writer_json: str, reader_json=None, columns=None):
    """The product's permissive handle of the same decode."""
    import pyruhvro_b200 as pr
    s = pr.Schema(writer_json)
    if reader_json is not None:
        s = s.read_as(reader_json)
    if columns is not None:
        s = s.project(columns)
    return s.permissive()


def build(walker: str, writer_json: str, reader_json=None, columns=None) -> str:
    """walker: "interp", "gen" (per lane) or "warp" (lock-step FAST emit warps)."""
    gdir = os.path.join(emu.HERE, "_gen")
    os.makedirs(gdir, exist_ok=True)
    if walker == "interp":
        so, extra = os.path.join(gdir, "libemu_permissive.so"), []
    else:
        src = schema(writer_json, reader_json, columns).walker_source
        h = hashlib.sha1(src.encode()).hexdigest()[:16]
        hdr = os.path.join(gdir, f"walker_{h}.cuh")
        if not os.path.exists(hdr):
            with open(hdr, "w") as f:
                f.write(src)
        so = os.path.join(gdir, f"libemu_permissive_{walker}_{h}.so")
        if walker == "gen":
            extra = ["-I", emu.CSRC, f'-DEMU_GEN_WALKER="{hdr}"']
        else:
            extra = ["-I", emu.CSRC, f'-DEMU_GEN_WALKER="{os.path.join(emu.HERE, "warp_walker.cuh")}"', f'-DEMU_LANE_WALKER="{hdr}"']
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in DEPS):
        tmp = f"{so}.{os.getpid()}.tmp"
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-w", "-x", "c++"] + extra + ["-o", tmp] + SRCS)
        os.replace(tmp, so)
    return so


def decode(writer_json: str, data, offsets, n: int, num_chunks: int = 1, reader_json=None, columns=None, walker: str = "interp",
           frame=(0, 0, 0), fingerprint: int = 0):
    """(batches, [(record, code), ...]) of the permissive decode; emu.EmuError for a fatal error.  frame: (header bytes,
    check: 0 none / 1 magic / 2 magic and id / SINGLE_OBJECT, schema id); fingerprint: the single-object check's."""
    from pyruhvro_b200 import _ArrowArray, _ArrowSchema
    so = build(walker, writer_json, reader_json, columns)
    lib = _libs.get(so)
    if lib is None:
        lib = _libs[so] = ctypes.CDLL(so)
        vp, i64 = ctypes.c_void_p, ctypes.c_int64
        lib.emu_decode_permissive.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_char_p, ctypes.c_size_t, vp, vp, i64, i64, vp, i64, vp,
                                              ctypes.c_ulonglong, vp, vp, ctypes.POINTER(i64), vp, ctypes.POINTER(i64), ctypes.POINTER(i64),
                                              ctypes.c_char_p, ctypes.c_size_t]
    raw_cols = [c.encode() for c in columns] if columns is not None else []
    cols = (ctypes.c_char_p * max(len(raw_cols), 1))(*raw_cols)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    fr = np.array(frame, dtype=np.int64)
    arrs = (_ArrowArray * min(max(num_chunks, 1), max(n, 1)))()
    sch = _ArrowSchema()
    k, rec, nbad = ctypes.c_int64(0), ctypes.c_int64(-1), ctypes.c_int64(0)
    bad = np.zeros(max(n, 1), dtype=np.uint64)
    msg = ctypes.create_string_buffer(512)
    w = writer_json.encode()
    r = reader_json.encode() if reader_json is not None else None
    rc = lib.emu_decode_permissive(w, len(w), r, len(r) if r else 0, data.ctypes.data if data.size else None, offsets.ctypes.data, n,
                                   num_chunks, ctypes.addressof(cols) if columns is not None else None, len(raw_cols), fr.ctypes.data,
                                   fingerprint, ctypes.addressof(arrs), ctypes.addressof(sch), ctypes.byref(k), bad.ctypes.data,
                                   ctypes.byref(nbad), ctypes.byref(rec), msg, 512)
    if rc != 0:
        raise emu.EmuError(rc, rec.value, msg.value.decode())
    schema_ = pa.Schema._import_from_c(ctypes.addressof(sch))
    batches = [pa.RecordBatch._import_from_c(ctypes.addressof(arrs[i]), schema_) for i in range(k.value)]
    return batches, [(int(b >> 8), int(b & 0xFF)) for b in bad[:nbad.value]]
