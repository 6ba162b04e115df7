"""Argument errors of the framed encodes (serialize_confluent, serialize_ocf and their C calls).  Every one of them is
raised on the host before any CUDA call, so these tests pass without a GPU."""
import ctypes

import pyarrow as pa
import pytest

import pyruhvro_b200 as pr

SJ = '{"type":"record","name":"R","fields":[{"name":"x","type":"int"},{"name":"s","type":"string"}]}'
EMPTY = ('{"type":"record","name":"Z","fields":[{"name":"a","type":"null"},{"name":"r","type":{"type":"record",'
         '"name":"Q","fields":[{"name":"x","type":"null"}]}}]}')
RV_ERR_SCHEMA, RV_ERR_INVALID = 7, 9
SYNC = bytes(range(16))


def _handle(sj):
    """A full schema handle that lives as long as the test (the schema cache keeps its Schema)."""
    return pr._get_or_parse_schema(sj).handle


def _batch(n=3):
    return pa.record_batch({"x": pa.array(range(n), pa.int32()), "s": [f"v{i}" for i in range(n)]})


def _c_call(fn, handle, batch, *args):
    """(status, message) of a C encode call; the exported batch's ownership moves to the library."""
    c_arr, c_sch = pr._ArrowArray(), pr._ArrowSchema()
    batch._export_to_c(ctypes.addressof(c_arr), ctypes.addressof(c_sch))
    h = ctypes.c_void_p()
    st = fn(handle, ctypes.addressof(c_arr), ctypes.addressof(c_sch), *args, ctypes.byref(h))
    assert c_arr.release is None and c_sch.release is None        # released by the callee, error or not
    if h.value:
        pr.lib.rv_encoded_free(h.value)
    return st, pr._last_error()


def _ocf_c(handle, batch, block_records=4, sync=SYNC, meta=()):
    n = len(meta)
    keys = (ctypes.c_char_p * max(n, 1))(*[k for k, _ in meta])
    vals = (ctypes.c_char_p * max(n, 1))(*[v for _, v in meta])
    lens = (ctypes.c_int64 * max(n, 1))(*[len(v) if v is not None else -1 for _, v in meta])
    return _c_call(pr.lib.rv_encode_ocf_host, handle, batch, block_records, sync, keys, vals, lens, n)


@pytest.mark.parametrize("r", [0, -1, -(1 << 40)])
def test_block_records_below_one(r):
    with pytest.raises(ValueError, match="block_records"):
        pr.serialize_ocf(_batch(), SJ, r, sync_marker=SYNC)
    assert _ocf_c(_handle(SJ), _batch(), r)[0] == RV_ERR_INVALID


@pytest.mark.parametrize("sync", [b"", bytes(15), bytes(17)])
def test_sync_marker_of_another_length(sync):
    with pytest.raises(ValueError, match="16 bytes"):
        pr.serialize_ocf(_batch(), SJ, sync_marker=sync)


def test_null_sync_and_negative_counts_in_the_c_call():
    h = _handle(SJ)
    st, msg = _ocf_c(h, _batch(), 4, None)
    assert st == RV_ERR_INVALID and "sync" in msg
    st, msg = _c_call(pr.lib.rv_encode_ocf_host, h, _batch(), 4, SYNC, None, None, None, -1)
    assert st == RV_ERR_INVALID and "n_meta" in msg
    st, msg = _ocf_c(h, _batch(), meta=[(b"k", None)])
    assert st == RV_ERR_INVALID and "negative value length" in msg


@pytest.mark.parametrize("key,what", [("avro.schema", "reserved"), ("avro.codec", "reserved"), ("avro.x", "reserved"),
                                      ("", "empty")])
def test_reserved_and_empty_metadata_keys(key, what):
    with pytest.raises(ValueError, match=what):
        pr.serialize_ocf(_batch(), SJ, sync_marker=SYNC, metadata={"ok": b"1", key: b"v"})


def test_repeated_metadata_key():
    h = _handle(SJ)
    st, msg = _ocf_c(h, _batch(), meta=[(b"a", b"1"), (b"b", b""), (b"a", b"2")])
    assert st == RV_ERR_INVALID and "'a' repeats" in msg


@pytest.mark.parametrize("sid", [-1, 1 << 32, -(1 << 40)])
def test_confluent_schema_id_out_of_range(sid):
    with pytest.raises(ValueError, match="schema id"):
        pr.serialize_confluent(_batch(), SJ, sid, 2)
    assert _c_call(pr.lib.rv_encode_host_confluent, _handle(SJ), _batch(), 1, sid)[0] == RV_ERR_INVALID


def test_projected_and_resolved_handles():
    full = pr.Schema(SJ)
    reader = pr.Schema(SJ.replace('"type":"int"', '"type":"long"'))
    for h in (full.project(["x"]), full.read_as(reader)):
        assert _ocf_c(h.handle, _batch())[0] == RV_ERR_INVALID
        assert _c_call(pr.lib.rv_encode_host_confluent, h.handle, _batch(), 1, 7)[0] == RV_ERR_INVALID


def test_always_empty_schema_is_refused_for_container_files():
    b = pa.record_batch({"a": pa.nulls(4), "r": pa.StructArray.from_arrays([pa.nulls(4)], ["x"])})
    with pytest.raises(ValueError, match="always empty|every datum"):
        pr.serialize_ocf(b, EMPTY, sync_marker=SYNC)
    assert _ocf_c(_handle(EMPTY), b)[0] == RV_ERR_SCHEMA


def test_missing_column():
    b = _batch().drop_columns(["s"])
    for call in (lambda: pr.serialize_ocf(b, SJ, sync_marker=SYNC), lambda: pr.serialize_confluent(b, SJ, 3)):
        with pytest.raises(ValueError, match="Arrow struct missing column 's' required by Avro schema"):
            call()


def test_python_type_errors_follow_serialize_record_batch():
    for call in (lambda d: pr.serialize_confluent(d, SJ, 1), lambda d: pr.serialize_ocf(d, SJ)):
        with pytest.raises(TypeError):
            call(_batch().to_pydict())
    with pytest.raises(OverflowError):
        pr.serialize_confluent(_batch(), SJ, 1, -1)


def test_file_of_a_chunked_result_and_exported_names():
    assert pr.lib.rv_encoded_file(None, ctypes.byref(ctypes.c_void_p()), ctypes.byref(ctypes.c_int64())) == RV_ERR_INVALID
    assert {"serialize_confluent", "serialize_ocf"} <= set(pr.__all__)
    import pyruhvro
    assert not hasattr(pyruhvro, "serialize_ocf") and not hasattr(pyruhvro, "serialize_confluent")
