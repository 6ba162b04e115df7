"""pyruhvro_b200 — H100-native drop-in for pyruhvro's direct Avro→Arrow decode path.

Python surface mirrored from the reference's PyO3 module (``/root/reference/src/lib.rs``):

    deserialize_array(list, schema)                          -> pyarrow.RecordBatch        (:56-71)
    deserialize_array_threaded(list, schema, num_chunks)     -> list[pyarrow.RecordBatch]  (:73-89)
    deserialize_array_threaded_spawn(list, schema, chunks)   -> list[pyarrow.RecordBatch]  (:108-128)
    serialize_record_batch(batch, schema, num_chunks)        -> list[pyarrow.Array]        (:91-106)
    serialize_record_batch_spawn(batch, schema, num_chunks)  -> list[pyarrow.Array]        (:130-147)

Same argument meaning and error behaviour: elements of ``list`` must be ``bytes`` or ``bytearray`` (PyBackedBytes); every failure is
a ``ValueError`` carrying the native message (:25-27); the GIL is released around the native work
(:64-69); parsed schemas are cached by their source string for the life of the process (:39-54);
batches cross into pyarrow through the Arrow C Data Interface, zero-copy (:70,88).

Deliberate divergences (documented in DESIGN.md): decode runs on the GPU with NO CPU fallback —
schemas outside the direct-decode subset raise instead of dropping to the Value-tree path, and a
missing CUDA device / native library is an error, never a silent Python path.
"""
from __future__ import annotations

import ctypes
import os
import threading
from typing import List

import pyarrow as pa

from . import _build

__all__ = [
    "deserialize_array", "deserialize_array_threaded", "deserialize_array_threaded_spawn",
    "serialize_record_batch", "serialize_record_batch_spawn", "lib", "Schema", "decode_packed", "deserialize_arrow_array",
    "deserialize_confluent", "deserialize_confluent_versions", "deserialize_ocf", "serialize_confluent", "serialize_ocf",
    "deserialize_single_object", "deserialize_single_object_versions", "serialize_single_object",
]

_HERE = os.path.dirname(os.path.abspath(__file__))


class _ArrowSchema(ctypes.Structure):
    _fields_ = [("format", ctypes.c_char_p), ("name", ctypes.c_char_p), ("metadata", ctypes.c_char_p),
                ("flags", ctypes.c_int64), ("n_children", ctypes.c_int64), ("children", ctypes.c_void_p),
                ("dictionary", ctypes.c_void_p), ("release", ctypes.c_void_p), ("private_data", ctypes.c_void_p)]


class _ArrowArray(ctypes.Structure):
    _fields_ = [("length", ctypes.c_int64), ("null_count", ctypes.c_int64), ("offset", ctypes.c_int64),
                ("n_buffers", ctypes.c_int64), ("n_children", ctypes.c_int64), ("buffers", ctypes.c_void_p),
                ("children", ctypes.c_void_p), ("dictionary", ctypes.c_void_p), ("release", ctypes.c_void_p),
                ("private_data", ctypes.c_void_p)]


def _load():
    """Loads the C-ABI library.  Fails loudly: there is no pure-Python or CPU decode path."""
    path = os.path.join(_HERE, "libruhvro_b200.so")
    if os.environ.get("RV_LIB_PATH"):  # development: a library built with other knobs (tools/tile_sweep.sh)
        return _bind(ctypes.CDLL(os.environ["RV_LIB_PATH"]))
    # missing or older than its sources: (re)build in-tree, under a file lock, written to a temporary and renamed.
    # Sources absent (a binary-only install) or no compiler: use what is there, fail loudly if nothing is.
    try:
        _build.build_all()
    except Exception:
        if not os.path.exists(path):
            raise
    return _bind(ctypes.CDLL(path))


def _bind(L):
    vp, i64, cp = ctypes.c_void_p, ctypes.c_int64, ctypes.c_char_p
    L.rv_schema_parse.argtypes = [cp, ctypes.c_size_t, ctypes.POINTER(vp)]
    L.rv_schema_retain.restype = vp
    L.rv_schema_retain.argtypes = [vp]
    L.rv_schema_release.argtypes = [vp]
    L.rv_schema_release.restype = None
    L.rv_schema_is_supported.argtypes = [vp]
    L.rv_schema_export_arrow.argtypes = [vp, vp]
    L.rv_decode_host.argtypes = [vp, vp, vp, i64, i64, ctypes.POINTER(vp)]
    L.rv_decode_device.argtypes = [vp, vp, vp, i64, i64, vp, ctypes.POINTER(vp)]
    L.rv_decode_host_framed.argtypes = [vp, vp, vp, i64, i64, vp, ctypes.POINTER(vp)]
    L.rv_decode_device_framed.argtypes = [vp, vp, vp, i64, i64, vp, vp, ctypes.POINTER(vp)]
    L.rv_decode_host_single_object.argtypes = [vp, vp, vp, i64, i64, ctypes.POINTER(vp)]
    L.rv_decode_device_single_object.argtypes = [vp, vp, vp, i64, i64, vp, ctypes.POINTER(vp)]
    L.rv_schema_canonical_form.restype = i64
    L.rv_schema_canonical_form.argtypes = [vp, cp, ctypes.c_size_t]
    L.rv_schema_fingerprint.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64)]
    L.rv_decode_ocf_host.argtypes = [vp, i64, i64, ctypes.POINTER(vp), ctypes.POINTER(vp)]
    L.rv_decode_ocf_host_projected.argtypes = [vp, i64, i64, vp, i64, ctypes.POINTER(vp), ctypes.POINTER(vp)]
    L.rv_schema_project.argtypes = [vp, vp, i64, ctypes.POINTER(vp)]
    L.rv_schema_resolve.argtypes = [vp, vp, ctypes.POINTER(vp)]
    L.rv_decode_ocf_host_resolved.argtypes = [vp, i64, i64, vp, vp, i64, ctypes.POINTER(vp), ctypes.POINTER(vp)]
    L.rv_versions_create.argtypes = [vp, vp, vp, i64, vp, i64, ctypes.POINTER(vp)]
    L.rv_versions_create_single_object.argtypes = [vp, vp, i64, vp, i64, ctypes.POINTER(vp)]
    L.rv_versions_permissive.argtypes = [vp, ctypes.POINTER(vp)]
    L.rv_versions_release.argtypes = [vp]
    L.rv_versions_release.restype = None
    L.rv_decode_host_versions.argtypes = [vp, vp, vp, i64, i64, ctypes.POINTER(vp)]
    L.rv_decode_device_versions.argtypes = [vp, vp, vp, i64, i64, vp, ctypes.POINTER(vp)]
    L.rv_last_versions_timings.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.c_int]
    L.rv_result_to_host.argtypes = [vp]
    L.rv_result_num_batches.restype = i64
    L.rv_result_num_batches.argtypes = [vp]
    L.rv_result_num_rows.restype = i64
    L.rv_result_num_rows.argtypes = [vp, i64]
    L.rv_result_arrow_bytes.restype = i64
    L.rv_result_arrow_bytes.argtypes = [vp]
    L.rv_schema_permissive.argtypes = [vp, ctypes.POINTER(vp)]
    L.rv_result_num_bad.restype = i64
    L.rv_result_num_bad.argtypes = [vp]
    L.rv_result_bad.restype = i64
    L.rv_result_bad.argtypes = [vp, vp, vp, i64]
    L.rv_result_bad_message.restype = ctypes.c_char_p
    L.rv_result_bad_message.argtypes = [vp, i64]
    L.rv_result_buffer_bytes.restype = i64
    L.rv_result_buffer_bytes.argtypes = [vp]
    L.rv_result_export.argtypes = [vp, i64, vp, vp]
    L.rv_result_export_device.argtypes = [vp, i64, vp, vp]
    L.rv_result_free.argtypes = [vp]
    L.rv_result_free.restype = None
    L.rv_encode_host.argtypes = [vp, vp, vp, i64, ctypes.POINTER(vp)]
    L.rv_encode_host_confluent.argtypes = [vp, vp, vp, i64, i64, ctypes.POINTER(vp)]
    L.rv_encode_host_single_object.argtypes = [vp, vp, vp, i64, ctypes.POINTER(vp)]
    L.rv_encode_ocf_host.argtypes = [vp, vp, vp, i64, vp, vp, vp, vp, i64, ctypes.POINTER(vp)]
    L.rv_encoded_file.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(i64)]
    L.rv_encoded_num_chunks.restype = i64
    L.rv_encoded_num_chunks.argtypes = [vp]
    L.rv_encoded_export.argtypes = [vp, i64, vp, vp]
    L.rv_encoded_free.argtypes = [vp]
    L.rv_encoded_free.restype = None
    L.rv_host_alloc.restype = vp
    L.rv_host_alloc.argtypes = [ctypes.c_size_t]
    L.rv_host_free.argtypes = [vp]
    L.rv_host_free.restype = None
    L.rv_last_timings.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.c_int]
    L.rv_last_launch_count.restype = ctypes.c_int
    L.rv_last_slow_tiles.restype = ctypes.c_longlong
    L.rv_last_passes.restype = ctypes.c_int
    L.rv_schema_forget_stats.argtypes = [vp]
    L.rv_schema_forget_stats.restype = None
    L.rv_last_walker.restype = cp
    L.rv_last_tile.restype = ctypes.c_int
    L.rv_schema_max_tile.restype = ctypes.c_int
    L.rv_schema_max_tile.argtypes = [vp]
    L.rv_schema_kernel_source.restype = i64
    L.rv_schema_kernel_source.argtypes = [vp, ctypes.c_int, cp, ctypes.c_size_t]
    L.rv_set_jit_enabled.argtypes = [ctypes.c_int]
    L.rv_set_jit_enabled.restype = None
    L.rv_schema_walker_source.restype = i64
    L.rv_schema_walker_source.argtypes = [vp, cp, ctypes.c_size_t]
    L.rv_schema_precompile.argtypes = [vp, cp]
    L.rv_last_error.restype = cp
    L.rv_version.restype = cp
    return L


lib = _load()


def last_walker() -> str:
    """"jit" or "interp": which GPU walker the last decode on this thread used."""
    return (lib.rv_last_walker() or b"").decode()


def set_jit_enabled(enabled: int) -> None:
    lib.rv_set_jit_enabled(int(enabled))


def _last_error() -> str:
    return (lib.rv_last_error() or b"").decode("utf-8", "replace")


def _check(status: int):
    if status != 0:
        raise ValueError(_last_error())  # to_py_err (src/lib.rs:25-27)


class Schema:
    """A parsed Avro schema + decode plan (the Arc<Schema> the reference shares across tasks)."""

    def __init__(self, schema_json: str):
        raw = schema_json.encode("utf-8")
        h = ctypes.c_void_p()
        _check(lib.rv_schema_parse(raw, len(raw), ctypes.byref(h)))
        self.handle = h.value
        self._arrow = None

    def __del__(self):
        h, self.handle = getattr(self, "handle", None), None
        if h:
            lib.rv_schema_release(h)

    @classmethod
    def _adopt(cls, handle: int) -> "Schema":
        s = cls.__new__(cls)
        s.handle, s._arrow = handle, None
        return s

    def project(self, columns) -> "Schema":
        """A schema whose batches hold only the top-level fields `columns`, in that order (rv_schema_project).  The other
        fields are still read and validated; a selected record / list / map / union column comes out whole."""
        names, keep = _column_names(columns)
        h = ctypes.c_void_p()
        _check(lib.rv_schema_project(self.handle, names, len(keep), ctypes.byref(h)))
        return Schema._adopt(h.value)

    def read_as(self, reader_json: str) -> "Schema":
        """A schema that reads data written with this schema (the writer's) as `reader_json` (rv_schema_resolve): batches
        in the reader's Arrow form, fields matched by name or reader alias, reader-only fields filled from their defaults,
        promotions and enum symbols resolved per the Avro specification."""
        reader = reader_json if isinstance(reader_json, Schema) else _get_or_parse_schema(reader_json)
        h = ctypes.c_void_p()
        _check(lib.rv_schema_resolve(self.handle, reader.handle, ctypes.byref(h)))
        return Schema._adopt(h.value)

    def permissive(self) -> "Schema":
        """A schema whose decodes turn a damaged record into a null row instead of failing (rv_schema_permissive).  Its
        batches are this schema's with every top-level field that is not a union, null or a map made nullable; the bad
        records are reported with the batches (errors="null" of the decode functions)."""
        h = ctypes.c_void_p()
        _check(lib.rv_schema_permissive(self.handle, ctypes.byref(h)))
        return Schema._adopt(h.value)

    @property
    def canonical_form(self) -> str:
        """The Avro specification's Parsing Canonical Form of the writer's full schema (also for a projected or resolved
        handle: the schema the data was written with)."""
        n = lib.rv_schema_canonical_form(self.handle, None, 0)
        if n < 0:
            raise ValueError(_last_error())
        buf = ctypes.create_string_buffer(n + 1)
        lib.rv_schema_canonical_form(self.handle, buf, n + 1)
        return buf.value.decode()

    @property
    def fingerprint(self) -> int:
        """The CRC-64-AVRO fingerprint of canonical_form, as an unsigned int: the key single-object messages carry."""
        fp = ctypes.c_uint64()
        _check(lib.rv_schema_fingerprint(self.handle, ctypes.byref(fp)))
        return fp.value

    @property
    def is_supported(self) -> bool:
        return bool(lib.rv_schema_is_supported(self.handle))

    def precompile(self, arch: str = "sm_90a") -> None:
        """Compile the schema-specialised kernels into the on-disk cubin cache (no GPU needed)."""
        _check(lib.rv_schema_precompile(self.handle, arch.encode()))

    @property
    def walker_source(self) -> str:
        n = lib.rv_schema_walker_source(self.handle, None, 0)
        if n < 0:
            raise ValueError("schema has no decode plan")
        buf = ctypes.create_string_buffer(n + 1)
        lib.rv_schema_walker_source(self.handle, buf, n + 1)
        return buf.value.decode()

    @property
    def arrow_schema(self) -> pa.Schema:
        if self._arrow is None:
            cs = _ArrowSchema()
            _check(lib.rv_schema_export_arrow(self.handle, ctypes.addressof(cs)))
            self._arrow = pa.Schema._import_from_c(ctypes.addressof(cs))
        return self._arrow


def _column_names(columns):
    """(char** array, keep-alive list) of a column projection; a bare str is refused rather than split into letters."""
    if isinstance(columns, (str, bytes)):
        raise TypeError("argument 'columns': expected a list of field names, not a single string")
    keep = []
    for c in columns:
        if not isinstance(c, str):
            raise TypeError("argument 'columns': field names must be str")
        keep.append(c.encode("utf-8"))
    arr = (ctypes.c_char_p * max(len(keep), 1))(*keep)
    return arr, keep


# schema_cache / get_or_parse_schema (src/lib.rs:39-54): unbounded, keyed by the exact strings of the (writer) schema and
# the reader schema, and the column projection
_schema_cache = {}
_schema_lock = threading.Lock()


def _get_or_parse_schema(schema: str, columns=None, reader_schema=None, permissive=False) -> Schema:
    if not isinstance(schema, str):
        raise TypeError("argument 'schema': expected str")
    if reader_schema is not None and not isinstance(reader_schema, str):
        raise TypeError("argument 'reader_schema': expected str")
    if columns is not None:
        if isinstance(columns, (str, bytes)):
            raise TypeError("argument 'columns': expected a list of field names, not a single string")
        columns = tuple(columns)
    key = (schema, reader_schema, columns, permissive)
    with _schema_lock:
        s = _schema_cache.get(key)
    if s is not None:
        return s
    if permissive:
        parsed = _get_or_parse_schema(schema, columns, reader_schema).permissive()
    elif columns is not None:
        parsed = _get_or_parse_schema(schema, None, reader_schema).project(columns)
    elif reader_schema is not None:
        parsed = _get_or_parse_schema(schema).read_as(reader_schema)
    else:
        parsed = Schema(schema)
    with _schema_lock:
        return _schema_cache.setdefault(key, parsed)


def _export_batches(result_handle: int, schema: Schema, with_bad: bool = False):
    """rv_result -> pyarrow batches through the Arrow C Data Interface; frees the result handle
    (the exported arrays keep the underlying memory alive).  with_bad: (batches, the bad-record report)."""
    try:
        arrow_schema = schema.arrow_schema
        out = []
        for i in range(lib.rv_result_num_batches(result_handle)):
            arr = _ArrowArray()
            _check(lib.rv_result_export(result_handle, i, ctypes.addressof(arr), None))
            out.append(pa.RecordBatch._import_from_c(ctypes.addressof(arr), arrow_schema))
        return (out, _bad_report(result_handle)) if with_bad else out
    finally:
        lib.rv_result_free(result_handle)


# errors="raise" (the default): a record that does not decode fails the call.  errors="null": it becomes a row that is
# null in every top-level column (Schema.permissive), and the call returns (batches, bad); `bad` lists the bad records
# in record order: `record` (index in the call), `status` (rv_status) and `error` (the strict call's message).
_BAD_SCHEMA = pa.schema([("record", pa.int64()), ("status", pa.int32()), ("error", pa.string())])


def _permissive(errors) -> bool:
    if errors == "raise":
        return False
    if errors == "null":
        return True
    raise ValueError(f"argument 'errors': expected \"raise\" or \"null\", got {errors!r}")


def _bad_report(result_handle: int) -> pa.RecordBatch:
    import numpy as np
    n = lib.rv_result_num_bad(result_handle)
    records = np.zeros(n, dtype=np.int64)
    status = np.zeros(n, dtype=np.int32)
    if n:
        lib.rv_result_bad(result_handle, records.ctypes.data, status.ctypes.data, n)
    text = [lib.rv_result_bad_message(result_handle, i).decode() for i in range(n)]
    return pa.RecordBatch.from_arrays([pa.array(records), pa.array(status), pa.array(text, pa.string())], schema=_BAD_SCHEMA)


_native_mod = None


def _ext():
    global _native_mod
    if _native_mod is None:
        import importlib
        _native_mod = importlib.import_module(__name__ + "._native")  # built by _build.build_ext(); ImportError is the loud failure
    return _native_mod


class Framing(ctypes.Structure):
    """rv_framing (include/ruhvro_b200.h): per-message header to skip, optionally validated as a Confluent header."""
    _fields_ = [("header_bytes", ctypes.c_int32), ("check_magic", ctypes.c_int32), ("schema_id", ctypes.c_int64)]


def _decode_list(records, schema: str, num_chunks: int, framing=None, columns=None, reader_schema=None, errors="raise"):
    permissive = _permissive(errors)
    if not isinstance(records, list):
        raise TypeError("argument 'list': expected a list of bytes")
    s = _get_or_parse_schema(schema, columns, reader_schema, permissive)
    if framing is None:
        handle = _ext().decode_list(s.handle, records, int(num_chunks))
    else:
        handle = _ext().decode_list(s.handle, records, int(num_chunks), *framing)
    return _export_batches(handle, s, permissive)


# Every decode entry point takes a keyword-only `columns`: a list of top-level field names.  The batches then hold only
# those columns, in that order, each identical to that column of the full decode (Schema.project).
# And a keyword-only `reader_schema`: the schema to read the data as (Schema.read_as); `schema` stays the schema the data
# was written with.  With both, `columns` names the reader's fields.
# The decodes of message lists and packed inputs also take a keyword-only `errors` ("raise" or "null", see _permissive).


def deserialize_ocf(data, num_chunks=1, *, columns=None, reader_schema=None) -> List[pa.RecordBatch]:
    """The bytes of an Avro Object Container File (uncompressed blocks) -> `num_chunks` RecordBatches; the schema is the
    file's own (with `reader_schema`: the file's schema is the writer's, the batches are the reader's).  Record boundaries
    are found on the GPU (one lane per block), see include/ruhvro_b200.h."""
    import numpy as np
    if num_chunks < 0:
        raise OverflowError("can't convert negative int to unsigned")
    buf = np.frombuffer(data, dtype=np.uint8)
    sh, h = ctypes.c_void_p(), ctypes.c_void_p()
    if reader_schema is not None:
        reader = _get_or_parse_schema(reader_schema)
        names, keep = _column_names(columns) if columns is not None else (None, [])
        _check(lib.rv_decode_ocf_host_resolved(buf.ctypes.data if buf.size else None, buf.size, int(num_chunks), reader.handle,
                                               names, len(keep), ctypes.byref(sh), ctypes.byref(h)))
    elif columns is None:
        _check(lib.rv_decode_ocf_host(buf.ctypes.data if buf.size else None, buf.size, int(num_chunks), ctypes.byref(sh), ctypes.byref(h)))
    else:
        names, keep = _column_names(columns)
        _check(lib.rv_decode_ocf_host_projected(buf.ctypes.data if buf.size else None, buf.size, int(num_chunks), names, len(keep),
                                                ctypes.byref(sh), ctypes.byref(h)))
    return _export_batches(h.value, Schema._adopt(sh.value))


def deserialize_confluent(list, schema, num_chunks=1, schema_id=None, *, columns=None, reader_schema=None, errors="raise"):  # noqa: A002
    """list[bytes] of Confluent-framed Kafka messages (magic 0x00 + big-endian u32 schema id + Avro datum) ->
    `num_chunks` RecordBatches.  The 5-byte header is validated (the id too when `schema_id` is given) and skipped inside
    the decode kernel — no per-message slicing in Python (the reference expects callers to strip it, README.md:93-94)."""
    if num_chunks < 0:
        raise OverflowError("can't convert negative int to unsigned")
    return _decode_list(list, schema, num_chunks, framing=(5, 1, -1 if schema_id is None else int(schema_id)), columns=columns,
                        reader_schema=reader_schema, errors=errors)


def deserialize_single_object(list, schema, num_chunks=1, *, columns=None, reader_schema=None, errors="raise"):  # noqa: A002
    """list[bytes] of Avro single-object messages (C3 01 + the little-endian CRC-64-AVRO fingerprint of the writer schema
    + Avro datum) -> `num_chunks` RecordBatches.  Every header must name `schema`'s fingerprint (Schema.fingerprint); it is
    checked and skipped inside the decode kernel (rv_decode_host_single_object)."""
    permissive = _permissive(errors)
    if num_chunks < 0:
        raise OverflowError("can't convert negative int to unsigned")
    if not isinstance(list, type([])):
        raise TypeError("argument 'list': expected a list of bytes")
    s = _get_or_parse_schema(schema, columns, reader_schema, permissive)
    return _export_batches(_ext().decode_list_single_object(s.handle, list, int(num_chunks)), s, permissive)


class Versions:
    """A registry of writer schemas read as one reader schema: the handle deserialize_confluent_versions and
    deserialize_single_object_versions decode with.  `writer_schemas` is a dict[int, str] by Confluent schema id
    (rv_versions_create), or with single_object=True a list[str] keyed by the schemas' fingerprints
    (rv_versions_create_single_object); `columns` optionally names the reader's top-level fields the batches hold."""

    def __init__(self, writer_schemas, reader_schema: str, columns=None, *, single_object=False):
        if single_object:
            if not isinstance(writer_schemas, (list, tuple)) or not all(isinstance(sj, str) for sj in writer_schemas):
                raise TypeError("argument 'writer_schemas': expected a list[str]")
            self.reader = _get_or_parse_schema(reader_schema, columns)
            full = _get_or_parse_schema(reader_schema)
            self._writers = [_get_or_parse_schema(sj) for sj in writer_schemas]
            n = len(self._writers)
            hs = (ctypes.c_void_p * max(n, 1))(*[w.handle for w in self._writers])
            names, keep = _column_names(columns) if columns is not None else (None, [])
            h = ctypes.c_void_p()
            _check(lib.rv_versions_create_single_object(full.handle, hs, n, names, len(keep), ctypes.byref(h)))
            self.handle = h.value
            return
        if not isinstance(writer_schemas, dict):
            raise TypeError("argument 'writer_schemas': expected a dict[int, str]")
        items = sorted(writer_schemas.items())
        for sid, sj in items:
            if not isinstance(sid, int) or not isinstance(sj, str):
                raise TypeError("argument 'writer_schemas': expected a dict[int, str]")
        self.reader = _get_or_parse_schema(reader_schema, columns)   # the batches' schema
        full = _get_or_parse_schema(reader_schema)
        self._writers = [_get_or_parse_schema(sj) for _, sj in items]   # kept alive with the registry
        n = len(items)
        ids = (ctypes.c_int64 * max(n, 1))(*[max(min(sid, 2 ** 63 - 1), -(2 ** 63)) for sid, _ in items])
        hs = (ctypes.c_void_p * max(n, 1))(*[w.handle for w in self._writers])
        names, keep = _column_names(columns) if columns is not None else (None, [])
        h = ctypes.c_void_p()
        _check(lib.rv_versions_create(full.handle, ids, hs, n, names, len(keep), ctypes.byref(h)))
        self.handle = h.value

    def permissive(self) -> "Versions":
        """A registry whose decodes turn a bad message into a null row and report it (rv_versions_permissive): a damaged
        datum, a short message, a wrong magic byte, or a schema id or fingerprint this registry does not know.  Its
        batches are the reader's with the top-level fields made nullable, as Schema.permissive makes them."""
        h = ctypes.c_void_p()
        _check(lib.rv_versions_permissive(self.handle, ctypes.byref(h)))
        p = Versions.__new__(Versions)
        p.handle = h.value
        p.reader = self.reader.permissive()
        p._writers = self._writers
        return p

    def __del__(self):
        h, self.handle = getattr(self, "handle", None), None
        if h:
            lib.rv_versions_release(h)


_versions_cache = {}


def _cached_versions(key, make, permissive: bool) -> Versions:
    """The registry of `key` (made by make() once), or its permissive form, cached under the mode too."""
    with _schema_lock:
        v = _versions_cache.get(key + (permissive,))
    if v is not None:
        return v
    v = _cached_versions(key, make, False).permissive() if permissive else make()
    with _schema_lock:
        return _versions_cache.setdefault(key + (permissive,), v)


def _get_or_create_versions(writer_schemas, reader_schema, columns, permissive=False) -> Versions:
    if not isinstance(writer_schemas, dict):
        raise TypeError("argument 'writer_schemas': expected a dict[int, str]")
    if not isinstance(reader_schema, str):
        raise TypeError("argument 'reader_schema': expected str")
    if columns is not None:
        if isinstance(columns, (str, bytes)):
            raise TypeError("argument 'columns': expected a list of field names, not a single string")
        columns = tuple(columns)
    key = (tuple(sorted(writer_schemas.items())), reader_schema, columns)
    return _cached_versions(key, lambda: Versions(writer_schemas, reader_schema, columns), permissive)


def deserialize_confluent_versions(list, writer_schemas, reader_schema, num_chunks=1, *, columns=None, errors="raise"):  # noqa: A002
    """list[bytes] of Confluent-framed Kafka messages written with several schema versions -> `num_chunks` RecordBatches
    in `reader_schema`'s Arrow form, rows in message order.  `writer_schemas` maps every schema id that may occur to the
    writer schema it names (dict[int, str]); each message is decoded with its own writer's schema and resolved to the
    reader (rv_decode_host_versions).  An id outside the map is an error, like a short message or a wrong magic byte.
    errors="null": such a message, and one whose datum does not decode, becomes a null row instead (Versions.permissive),
    and the call returns (batches, bad) as the other decodes do; an unregistered id is reported with its id."""
    permissive = _permissive(errors)
    if num_chunks < 0:
        raise OverflowError("can't convert negative int to unsigned")
    if not isinstance(list, type([])):
        raise TypeError("argument 'list': expected a list of bytes")
    v = _get_or_create_versions(writer_schemas, reader_schema, columns, permissive)
    return _export_batches(_ext().decode_list_versions(v.handle, list, int(num_chunks)), v.reader, permissive)


def deserialize_single_object_versions(list, writer_schemas, reader_schema, num_chunks=1, *, columns=None, errors="raise"):  # noqa: A002
    """list[bytes] of Avro single-object messages written with several schemas -> `num_chunks` RecordBatches in
    `reader_schema`'s Arrow form, rows in message order.  `writer_schemas` (list[str]) holds every writer schema that may
    occur; each message is decoded with the writer whose fingerprint its header names and resolved to the reader
    (rv_decode_host_versions).  An unregistered fingerprint is an error, like a short message or a wrong C3 01 marker.
    Two writers with the same canonical form cannot be told apart on the wire and are refused.  errors="null": as in
    deserialize_confluent_versions, an unregistered fingerprint is reported with its fingerprint."""
    permissive = _permissive(errors)
    if num_chunks < 0:
        raise OverflowError("can't convert negative int to unsigned")
    if not isinstance(list, type([])):
        raise TypeError("argument 'list': expected a list of bytes")
    if not isinstance(writer_schemas, (type([]), tuple)):
        raise TypeError("argument 'writer_schemas': expected a list[str]")
    if not isinstance(reader_schema, str):
        raise TypeError("argument 'reader_schema': expected str")
    if columns is not None:
        if isinstance(columns, (str, bytes)):
            raise TypeError("argument 'columns': expected a list of field names, not a single string")
        columns = tuple(columns)
    key = ("single_object", tuple(writer_schemas), reader_schema, columns)
    v = _cached_versions(key, lambda: Versions(writer_schemas, reader_schema, columns, single_object=True), permissive)
    return _export_batches(_ext().decode_list_versions(v.handle, list, int(num_chunks)), v.reader, permissive)


def last_versions_timings() -> dict:
    """CUDA-event times (ms) of the calling thread's last deserialize_confluent_versions / rv_decode_*_versions call."""
    buf = (ctypes.c_float * 4)()
    lib.rv_last_versions_timings(buf, 4)
    return dict(zip(("partition", "decodes", "take", "device"), buf))


def deserialize_array(list, schema, *, columns=None, reader_schema=None, errors="raise"):  # noqa: A002 - the reference names the parameter `list`
    """list[bytes] of schemaless Avro datums -> one RecordBatch (src/lib.rs:56-71); errors="null": (batch, bad)."""
    if _permissive(errors):
        batches, bad = _decode_list(list, schema, 1, columns=columns, reader_schema=reader_schema, errors=errors)
        return batches[0], bad
    return _decode_list(list, schema, 1, columns=columns, reader_schema=reader_schema)[0]


def deserialize_array_threaded(list, schema, num_chunks, *, columns=None, reader_schema=None, errors="raise"):  # noqa: A002
    """list[bytes] -> `num_chunks` RecordBatches over contiguous row ranges (src/lib.rs:73-89;
    chunking per ruhvro/src/deserialize.rs:53-68)."""
    if num_chunks < 0:
        raise OverflowError("can't convert negative int to unsigned")  # usize extraction in PyO3
    return _decode_list(list, schema, num_chunks, columns=columns, reader_schema=reader_schema, errors=errors)


def deserialize_array_threaded_spawn(list, schema, num_chunks, *, columns=None, reader_schema=None, errors="raise"):  # noqa: A002
    """Same results as deserialize_array_threaded (the reference only changes the tokio primitive,
    ruhvro/src/deserialize.rs:123-170)."""
    return deserialize_array_threaded(list, schema, num_chunks, columns=columns, reader_schema=reader_schema, errors=errors)


def decode_packed(data, offsets, n: int, schema: str, num_chunks: int = 1, framing: "Framing | None" = None, *,
                  columns=None, reader_schema=None, errors="raise"):
    """Packed host buffers (numpy uint8 data + int64 offsets[n+1]) -> batches, through rv_decode_host (or
    rv_decode_host_framed when `framing` is given).  This is the C-ABI call a Rust/FFI caller makes; no Python list walk."""
    import numpy as np
    permissive = _permissive(errors)
    s = _get_or_parse_schema(schema, columns, reader_schema, permissive)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.int64)
    h = ctypes.c_void_p()
    _check(lib.rv_decode_host_framed(s.handle, data.ctypes.data if data.size else None, offsets.ctypes.data, n, num_chunks,
                                     ctypes.byref(framing) if framing is not None else None, ctypes.byref(h)))
    return _export_batches(h.value, s, permissive)


def _packed_view(arr):
    """(data uint8[], offsets int64[n+1], n) of a Binary / LargeBinary / String array without copying the
    payload: the offsets are rebased so that offsets[0] indexes into `data` (sliced arrays are fine)."""
    import numpy as np
    if isinstance(arr, pa.ChunkedArray):
        arr = arr.combine_chunks() if arr.num_chunks != 1 else arr.chunk(0)
    t = arr.type
    if pa.types.is_large_binary(t) or pa.types.is_large_string(t):
        odt = np.int64
    elif pa.types.is_binary(t) or pa.types.is_string(t):
        odt = np.int32
    else:
        raise TypeError(f"expected a (Large)Binary / (Large)String array of Avro datums, got {t}")
    if arr.null_count:
        raise ValueError("the datum array contains nulls")
    n = len(arr)
    bufs = arr.buffers()
    if n == 0 or bufs[1] is None:
        return np.zeros(0, dtype=np.uint8), np.zeros(1, dtype=np.int64), 0
    off = np.frombuffer(bufs[1], dtype=odt)[arr.offset: arr.offset + n + 1]
    data = np.frombuffer(bufs[2], dtype=np.uint8) if bufs[2] is not None else np.zeros(0, dtype=np.uint8)
    return data, off.astype(np.int64, copy=False), n


def deserialize_arrow_array(array, schema, num_chunks=1, *, columns=None, reader_schema=None, errors="raise"):
    """An Arrow Binary/LargeBinary array (or ChunkedArray) of schemaless datums -> `num_chunks` RecordBatches.

    The ingest shortcut of SURVEY §8(f) rank 2: what `per_datum_deserialize_threaded` builds internally at
    ruhvro/src/deserialize.rs:90 (a packed values buffer + offsets) is accepted as-is, so there is no Python
    list walk and no gather copy; results are identical to deserialize_array_threaded on `array.to_pylist()`."""
    if num_chunks < 0:
        raise OverflowError("can't convert negative int to unsigned")
    _permissive(errors)
    data, off, n = _packed_view(array)
    return decode_packed(data, off, n, schema, int(num_chunks), columns=columns, reader_schema=reader_schema, errors=errors)


def _encode(encode_fn, data, schema, *args) -> int:
    """Exports the RecordBatch through the Arrow C Data Interface (ownership moves to the library) and runs one of the
    rv_encode_* calls; returns the rv_encoded handle."""
    s = _get_or_parse_schema(schema)
    c_arr, c_sch = _ArrowArray(), _ArrowSchema()
    data._export_to_c(ctypes.addressof(c_arr), ctypes.addressof(c_sch))
    h = ctypes.c_void_p()
    _check(encode_fn(s.handle, ctypes.addressof(c_arr), ctypes.addressof(c_sch), *args, ctypes.byref(h)))
    return h.value


def _export_chunks(h) -> list:
    try:
        out = []
        for i in range(lib.rv_encoded_num_chunks(h)):
            a, sc = _ArrowArray(), _ArrowSchema()
            _check(lib.rv_encoded_export(h, i, ctypes.addressof(a), ctypes.addressof(sc)))
            out.append(pa.Array._import_from_c(ctypes.addressof(a), ctypes.addressof(sc)))
        return out
    finally:
        lib.rv_encoded_free(h)


def _check_batch(data, num_chunks):
    if not isinstance(data, pa.RecordBatch):
        raise TypeError("argument 'data': expected a pyarrow.RecordBatch")
    if num_chunks < 0:
        raise OverflowError("can't convert negative int to unsigned")


def serialize_record_batch(data, schema, num_chunks):
    """pyarrow.RecordBatch -> `num_chunks` pyarrow Binary arrays of schemaless Avro datums
    (src/lib.rs:91-106; ruhvro/src/serialize.rs:38-67), encoded on the GPU (rv_encode_host)."""
    _check_batch(data, num_chunks)
    return _export_chunks(_encode(lib.rv_encode_host, data, schema, int(num_chunks)))


def serialize_confluent(data, schema, schema_id, num_chunks=1):
    """pyarrow.RecordBatch -> `num_chunks` pyarrow Binary arrays of Confluent-framed Kafka messages: element i is 0x00,
    the big-endian u32 `schema_id`, then row i's datum (rv_encode_host_confluent).  The header is written by the encode
    kernels, so there is no per-message slicing or concatenation in Python.  Chunking is serialize_record_batch's; the
    messages read back with deserialize_confluent."""
    _check_batch(data, num_chunks)
    return _export_chunks(_encode(lib.rv_encode_host_confluent, data, schema, int(num_chunks), int(schema_id)))


def serialize_single_object(data, schema, num_chunks=1):
    """pyarrow.RecordBatch -> `num_chunks` pyarrow Binary arrays of Avro single-object messages: element i is C3 01, the
    little-endian CRC-64-AVRO fingerprint of `schema` (Schema.fingerprint), then row i's datum
    (rv_encode_host_single_object).  Chunking is serialize_record_batch's; the messages read back with
    deserialize_single_object."""
    _check_batch(data, num_chunks)
    return _export_chunks(_encode(lib.rv_encode_host_single_object, data, schema, int(num_chunks)))


class _EncodedFile:
    """Keeps an rv_encoded alive for as long as a pa.Buffer over its file exists."""

    def __init__(self, handle):
        self.handle = handle

    def __del__(self):
        h, self.handle = getattr(self, "handle", None), None
        if h:
            lib.rv_encoded_free(h)


def serialize_ocf(data, schema, block_records=1024, *, sync_marker=None, metadata=None) -> pa.Buffer:
    """pyarrow.RecordBatch -> one Avro Object Container File (codec "null") as a pa.Buffer over the library's pinned
    file, without a copy (rv_encode_ocf_host).  The header holds `schema` as avro.schema, avro.codec "null" and the
    `metadata` pairs (dict[str, bytes]; keys must not be empty or start with "avro."); every block holds `block_records`
    rows, the last one the rest, and ends with `sync_marker` (16 bytes; default: os.urandom(16)).  deserialize_ocf reads
    the buffer directly.

    Blocks are the encoder's chunks and its 256-row tiles never span two blocks, so a `block_records` that is not a
    multiple of 256 leaves lanes idle.  The default 1024 is four full tiles per block, about 120 KB per block of Kafka
    rows."""
    _check_batch(data, 0)
    sync = os.urandom(16) if sync_marker is None else bytes(sync_marker)
    if len(sync) != 16:
        raise ValueError(f"sync_marker must be 16 bytes, got {len(sync)}")
    items = list((metadata or {}).items())
    keys = [k.encode("utf-8") if isinstance(k, str) else k for k, _ in items]
    vals = [bytes(v) for _, v in items]
    n = len(items)
    c_keys = (ctypes.c_char_p * max(n, 1))(*keys)
    c_vals = (ctypes.c_char_p * max(n, 1))(*vals)
    c_lens = (ctypes.c_int64 * max(n, 1))(*[len(v) for v in vals])
    h = _encode(lib.rv_encode_ocf_host, data, schema, int(block_records), sync, c_keys, c_vals, c_lens, n)
    owner = _EncodedFile(h)
    ptr, length = ctypes.c_void_p(), ctypes.c_int64()
    _check(lib.rv_encoded_file(h, ctypes.byref(ptr), ctypes.byref(length)))
    return pa.foreign_buffer(ptr.value, length.value, base=owner)


def serialize_record_batch_spawn(data, schema, num_chunks):
    """Same results as serialize_record_batch (the reference only changes the tokio primitive, serialize.rs:70-99)."""
    return serialize_record_batch(data, schema, num_chunks)
