"""Host emulation of the GPU pipeline (test infrastructure; see emu.cpp)."""
import ctypes
import os
import subprocess

import numpy as np
import pyarrow as pa

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "..", "..", "pyruhvro_b200", "csrc")
SO = os.path.join(HERE, "libemu.so")
SRCS = [os.path.join(HERE, "emu.cpp")] + [os.path.join(CSRC, f) for f in ("schema.cpp", "plan.cpp", "result.cpp", "gather.cpp", "ocf.cpp")]
DEPS = SRCS + [os.path.join(CSRC, f) for f in ("dev_core.cuh", "dev_types.h", "interp.cuh", "ocf_walk.cuh", "plan.hpp", "result.hpp", "gather.hpp",
                                               "ocf.hpp", "schema.hpp", "json.hpp")]


class EmuError(ValueError):
    def __init__(self, code, record, msg=""):
        super().__init__(f"emu error {code} at record {record} {msg}")
        self.code, self.record = code, record


class EmuContainerError(ValueError):
    """The product's container reader (ocf.cpp) rejected an object container file."""


def build(gen_source: str = None):
    """gen_source=None: the interpreter walker.  Otherwise the generated, schema-specialised walker
    (what NVRTC compiles for the GPU) is compiled for the host and driven by the same emulation."""
    if gen_source is None:
        so, extra = SO, []
    else:
        import hashlib
        h = hashlib.sha1(gen_source.encode()).hexdigest()[:16]
        gdir = os.path.join(HERE, "_gen")
        os.makedirs(gdir, exist_ok=True)
        hdr = os.path.join(gdir, f"walker_{h}.cuh")
        if not os.path.exists(hdr):
            with open(hdr, "w") as f:
                f.write(gen_source)
        so = os.path.join(gdir, f"libemu_{h}.so")
        extra = ["-I", CSRC, f'-DEMU_GEN_WALKER="{hdr}"']
    if not os.path.exists(so) or any(os.path.getmtime(d) > os.path.getmtime(so) for d in DEPS):
        subprocess.check_call(["g++", "-std=c++17", "-O1", "-g", "-fPIC", "-shared", "-Wall", "-x", "c++"] + extra + ["-o", so] + SRCS)
    return so


_libs = {}


def walker_source(schema_json: str) -> str:
    import pyruhvro_b200 as pr
    return pr.Schema(schema_json).walker_source


def decode(schema_json: str, data, offsets, n: int, num_chunks: int = 1, walker: str = "interp"):
    from pyruhvro_b200 import _ArrowArray, _ArrowSchema
    so = build(walker_source(schema_json) if walker == "gen" else None)
    _lib = _libs.get(so)
    if _lib is None:
        _lib = _libs[so] = ctypes.CDLL(so)
        _lib.emu_decode.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64,
                                    ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int64),
                                    ctypes.c_char_p, ctypes.c_size_t]
    data = np.ascontiguousarray(data, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    k_max = min(max(num_chunks, 1), max(n, 1))
    arrs = (_ArrowArray * k_max)()
    sch = _ArrowSchema()
    k = ctypes.c_int64(0)
    rec = ctypes.c_int64(-1)
    msg = ctypes.create_string_buffer(512)
    raw = schema_json.encode()
    rc = _lib.emu_decode(raw, len(raw), data.ctypes.data if data.size else None, offsets.ctypes.data, n, num_chunks,
                         ctypes.addressof(arrs), ctypes.addressof(sch), ctypes.byref(k), ctypes.byref(rec), msg, 512)
    if rc != 0:
        raise EmuError(rc, rec.value, msg.value.decode())
    schema = pa.Schema._import_from_c(ctypes.addressof(sch))
    return [pa.RecordBatch._import_from_c(ctypes.addressof(arrs[i]), schema) for i in range(k.value)]


def decode_ocf(file: bytes, num_chunks: int = 1):
    """An object container file through the product's container reader, the per-block offsets walk of the device
    (ocf_walk.cuh, every block in turn) and the emulated decode (interpreter walker).  Raises EmuContainerError for a
    malformed container, EmuError(code, record) for a record that fails."""
    from pyruhvro_b200 import _ArrowArray, _ArrowSchema
    lib = _lib_interp()
    if not hasattr(lib, "_ocf_bound"):
        vp, i64 = ctypes.c_void_p, ctypes.c_int64
        lib.emu_decode_ocf.argtypes = [vp, i64, i64, vp, vp, ctypes.POINTER(i64), ctypes.POINTER(i64), ctypes.c_char_p, ctypes.c_size_t]
        lib._ocf_bound = True
    buf = np.frombuffer(bytes(file), dtype=np.uint8)
    arrs = (_ArrowArray * max(num_chunks, 1))()
    sch = _ArrowSchema()
    k, rec = ctypes.c_int64(0), ctypes.c_int64(-1)
    msg = ctypes.create_string_buffer(512)
    rc = lib.emu_decode_ocf(buf.ctypes.data if buf.size else None, buf.size, num_chunks, ctypes.addressof(arrs), ctypes.addressof(sch),
                            ctypes.byref(k), ctypes.byref(rec), msg, 512)
    if rc == -2:
        raise EmuContainerError(msg.value.decode())
    if rc != 0:
        raise EmuError(rc, rec.value, msg.value.decode())
    schema = pa.Schema._import_from_c(ctypes.addressof(sch))
    return [pa.RecordBatch._import_from_c(ctypes.addressof(arrs[i]), schema) for i in range(k.value)]


def _lib_interp():
    so = build(None)
    lib = _libs.get(so)
    if lib is None:
        lib = _libs[so] = ctypes.CDLL(so)
        lib.emu_decode.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int64, ctypes.c_int64,
                                   ctypes.c_void_p, ctypes.c_void_p, ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int64),
                                   ctypes.c_char_p, ctypes.c_size_t]
    if not hasattr(lib, "_gather_bound"):
        vp, i64 = ctypes.c_void_p, ctypes.c_int64
        lib.emu_shard_decode.restype = vp
        lib.emu_shard_decode.argtypes = [ctypes.c_char_p, ctypes.c_size_t, vp, vp, i64, ctypes.c_char_p, ctypes.c_size_t]
        lib.emu_shard_free.argtypes = [vp]
        lib.emu_shard_free.restype = None
        lib.emu_meta_len.restype = i64
        lib.emu_meta_len.argtypes = [vp]
        lib.emu_shard_meta.argtypes = [vp, vp]
        lib.emu_shard_meta.restype = None
        lib.emu_gather_groups.argtypes = [vp, vp, ctypes.c_int, vp, ctypes.c_int]
        lib.emu_gather_apply.argtypes = [vp, vp, ctypes.c_int, ctypes.c_int, vp]
        lib.emu_gather_export.argtypes = [vp, vp, ctypes.c_int, ctypes.c_int, vp, vp, vp]
        lib._gather_bound = True
    return lib


class Shard:
    """One rank's emulated shard decode, for the host emulation of the multi-GPU gather (the product's planning code
    from csrc/gather.cpp + a host restatement of what gather_push_kernel does per job)."""

    def __init__(self, schema_json: str, data, offsets, n: int):
        self.lib = _lib_interp()
        data = np.ascontiguousarray(data, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.int64)
        msg = ctypes.create_string_buffer(512)
        raw = schema_json.encode()
        self.h = self.lib.emu_shard_decode(raw, len(raw), data.ctypes.data if data.size else None, offsets.ctypes.data, n, msg, 512)
        if not self.h:
            raise ValueError(msg.value.decode())

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.emu_shard_free(self.h)
            self.h = None

    def meta(self) -> np.ndarray:
        m = np.zeros(max(self.lib.emu_meta_len(self.h), 1), dtype=np.int64)
        self.lib.emu_shard_meta(self.h, m.ctypes.data)
        return m

    def groups(self, metas: np.ndarray):
        out = np.zeros(1 + 4 * len(metas), dtype=np.int64)
        self.lib.emu_gather_groups(self.h, np.ascontiguousarray(metas).ctypes.data, len(metas), out.ctypes.data, out.size)
        return [tuple(int(x) for x in out[1 + 4 * i: 5 + 4 * i]) for i in range(int(out[0]))]  # (first rank, ranks, arena bytes, rows)

    def apply(self, metas: np.ndarray, rank: int, arena: np.ndarray):
        self.lib.emu_gather_apply(self.h, np.ascontiguousarray(metas).ctypes.data, len(metas), rank, arena.ctypes.data)

    def export(self, metas: np.ndarray, group: int, arena: np.ndarray) -> pa.RecordBatch:
        from pyruhvro_b200 import _ArrowArray, _ArrowSchema
        arr, sch = _ArrowArray(), _ArrowSchema()
        self.lib.emu_gather_export(self.h, np.ascontiguousarray(metas).ctypes.data, len(metas), group, arena.ctypes.data,
                                   ctypes.addressof(arr), ctypes.addressof(sch))
        schema = pa.Schema._import_from_c(ctypes.addressof(sch))
        return pa.RecordBatch._import_from_c(ctypes.addressof(arr), schema)
