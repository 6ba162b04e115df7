"""Column projection (rv_schema_project / Schema.project / `columns=`): the batches hold only the requested top-level
fields, in the requested order, each buffer for buffer the column of the full decode; the other fields are still walked
and validated, so a projected decode fails where the full one does, with the same category (RV_ERR_OVERFLOW excepted:
only produced columns can overflow Arrow's offsets).  CPU tests run the product's plan and walkers through the host
emulation (tests/emu); the GPU tests run every entry point on the device."""
import ctypes
import random
import re

import numpy as np
import pyarrow as pa
import pytest

import pyruhvro_b200 as pr
from oracle import pyoracle as po
from tests import emu, mutation as M
from tests.emu import projection as P
from tests.parity import expected_schema, expected_schema_wide, gen_case, gen_case_wide

C3_PROJECTIONS = [["created_at"], ["name", "age", "created_at"], ["emails", "phone_numbers"], ["status", "class"]]


@pytest.fixture(scope="module")
def kafka():
    import workloads
    return workloads.KAFKA_SCHEMA


def _names(sj, wide=False):
    return [f.name for f in (expected_schema_wide(sj) if wide else expected_schema(sj))]


def _random_projection(rng, names):
    cols = rng.sample(names, rng.randint(1, len(names)))
    return cols


def _assert_selected(batches, want, cols, exp_schema, full_validate=True):
    """`want`: canonical batches of the full decode (oracle); every batch equals them with `cols` selected."""
    names = [f.name for f in exp_schema]
    idx = [names.index(c) for c in cols]
    sel_schema = pa.schema([exp_schema.field(i) for i in idx])
    assert len(batches) == len(want)
    for i, (b, w) in enumerate(zip(batches, want)):
        assert b.schema.equals(sel_schema, check_metadata=True), f"batch {i}\n{b.schema}\n!=\n{sel_schema}"
        if full_validate:
            b.validate(full=True)
        d = po.canon_diff(po.canon_from_batch(b), [w[j] for j in idx], f"batch[{i}]")
        assert d is None, d


def _oracle_batches(coracle, sj, data, off, n, k):
    return coracle.decode_threaded_packed(sj, np.ascontiguousarray(data, dtype=np.uint8), np.ascontiguousarray(off, dtype=np.int64), n, k, threads=4)


def _py_batches(sj, recs, k):
    s = po.parse_schema(sj, wide=True)
    return [po.py_decode(s, recs[r0:r1]) for r0, r1 in po.chunk_bounds(len(recs), po.clamp_chunks(k, len(recs)))]


# ---- front end ------------------------------------------------------------------------------------------------------
def test_projected_arrow_schema_is_the_full_one_selected(kafka):
    full = pr.Schema(kafka).arrow_schema
    for cols in C3_PROJECTIONS + [["class", "name"], ["address", "preferences", "age"]]:
        got = pr.Schema(kafka).project(cols).arrow_schema
        assert got.equals(pa.schema([full.field(c) for c in cols]), check_metadata=True)
        assert got.names == cols
    sj = gen_case_wide(3)[0]
    full = pr.Schema(sj).arrow_schema
    cols = list(reversed(full.names))
    assert pr.Schema(sj).project(cols).arrow_schema.equals(pa.schema([full.field(c) for c in cols]), check_metadata=True)
    # a projection of a projection selects among its columns
    assert pr.Schema(kafka).project(["age", "name", "class"]).project(["class", "age"]).arrow_schema.names == ["class", "age"]


def test_projection_errors(kafka):
    s = pr.Schema(kafka)
    with pytest.raises(ValueError, match="empty"):
        s.project([])
    with pytest.raises(ValueError, match="twice"):
        s.project(["age", "name", "age"])
    with pytest.raises(ValueError, match=r"no top-level field 'city'.*Available fields: \[\"name\", \"age\""):
        s.project(["age", "city"])
    with pytest.raises(ValueError, match="address.city"):
        s.project(["address.city"])
    with pytest.raises(TypeError):
        s.project("age")
    with pytest.raises(TypeError):
        pr.deserialize_array([], kafka, columns="age")
    with pytest.raises(ValueError):   # an unsupported schema stays RV_ERR_SCHEMA
        bad = '{"type": "record", "name": "R", "fields": [{"name": "d", "type": {"type": "fixed", "name": "F", "size": 0}}]}'
        pr.Schema(bad).project(["d"])
    h = ctypes.c_void_p()
    names = (ctypes.c_char_p * 1)(b"age")
    assert pr.lib.rv_schema_project(s.handle, names, 0, ctypes.byref(h)) == 9          # RV_ERR_INVALID: empty
    assert pr.lib.rv_schema_project(s.handle, names, 1, ctypes.byref(h)) == 0
    pr.lib.rv_schema_release(h)


def test_encoding_with_a_projection_is_refused(kafka):
    import workloads
    sj, data, off = workloads.generate("kafka", 10, seed=1)
    batch = emu.decode(sj, data, off, 10, 1)[0]
    p = pr.Schema(kafka).project(["age"])
    c_arr, c_sch = pr._ArrowArray(), pr._ArrowSchema()
    batch.select(["age"])._export_to_c(ctypes.addressof(c_arr), ctypes.addressof(c_sch))
    h = ctypes.c_void_p()
    assert pr.lib.rv_encode_host(p.handle, ctypes.addressof(c_arr), ctypes.addressof(c_sch), 1, ctypes.byref(h)) == 9   # RV_ERR_INVALID
    assert "column projection" in pr._last_error()


def test_walker_source_has_only_the_kept_columns_streams(kafka):
    src = pr.Schema(kafka).project(["created_at", "age"]).walker_source
    assert "kStreams = 0;" in src and "kItemBytes = 0;" in src
    assert "skip_end[" in src and "(skipped)" in src
    src = pr.Schema(kafka).project(["emails", "phone_numbers"]).walker_source
    assert "kStreams = 5;" in src and "2 item-parallel lists" in src
    full = pr.Schema(kafka).walker_source
    assert "skip" not in full   # an unprojected plan has no skip nodes


# ---- emulated parity -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(40))
def test_random_schemas_random_projections(coracle, seed):
    sj, recs, data, off = gen_case(seed)
    rng = random.Random(seed + 7)
    k = rng.choice([1, 2, 5])
    want = _oracle_batches(coracle, sj, data, off, len(recs), k)
    cols = _random_projection(rng, _names(sj))
    walkers = ("interp", "gen") if seed % 4 == 0 else ("interp",)
    for w in walkers:
        _assert_selected(P.decode(sj, data, off, len(recs), k, cols, walker=w), want, cols, expected_schema(sj))


@pytest.mark.parametrize("seed", range(20))
def test_random_wide_schemas_random_projections(seed):
    sj, recs, data, off = gen_case_wide(seed)
    rng = random.Random(seed + 11)
    k = rng.choice([1, 2, 5])
    cols = _random_projection(rng, _names(sj, wide=True))
    _assert_selected(P.decode(sj, data, off, len(recs), k, cols), _py_batches(sj, recs, k), cols, expected_schema_wide(sj))


@pytest.mark.parametrize("cols", C3_PROJECTIONS + [["phone_numbers", "name"]])
def test_kafka_projections_every_walker(coracle, cols):
    """Both walkers and the warp lock-step emulation (the EMIT jump over skipped runs, then item-parallel lists)."""
    import workloads
    sj, data, off = workloads.generate("kafka", 1500, seed=7)
    want = _oracle_batches(coracle, sj, data, off, 1500, 3)
    for w in ("interp", "gen"):
        _assert_selected(P.decode(sj, data, off, 1500, 3, cols, walker=w), want, cols, expected_schema(sj))
    before = P.collectives(sj, cols)
    _assert_selected(P.decode(sj, data, off, 1500, 3, cols, walker="warp"), want, cols, expected_schema(sj))
    if "emails" in cols or "phone_numbers" in cols:
        assert P.collectives(sj, cols) > before


# ---- emulated damaged inputs -----------------------------------------------------------------------------------------
def _check_damaged(coracle, sj, recs, k, cols, walker, wide=False):
    data, off = po.pack_records(recs)
    want = M.expected_wide(sj, recs) if wide else M.expected(coracle, sj, recs)
    try:
        got = P.decode(sj, data, off, len(recs), k, cols, walker=walker)
    except emu.EmuError as e:
        g = (po.ERR_NAMES.get(e.code, str(e.code)), e.record)
        assert g == want, f"projection reports {g}, the full decode {want}"
        return
    if want is not None:   # only a column that is produced can overflow Arrow's offsets
        assert want[0] == "overflow", f"projection accepted a batch the full decode rejects with {want}"
        return
    full = _py_batches(sj, recs, k) if wide else _oracle_batches(coracle, sj, data, off, len(recs), k)
    _assert_selected(got, full, cols, expected_schema_wide(sj) if wide else expected_schema(sj), full_validate=False)


@pytest.mark.parametrize("seed", range(60))
def test_damaged_inputs_under_projections(coracle, seed):
    rng = random.Random(seed)
    if seed % 3 == 0:
        sj, recs, k = M.damaged_case(910000 + seed)
    elif seed % 3 == 1:
        sj, recs, k = M.forged_case(960000 + seed)
    else:
        sj, recs, k = M.damaged_case_wide(950000 + seed)
        _check_damaged(coracle, sj, recs, k, _random_projection(rng, _names(sj, wide=True)), "interp", wide=True)
        return
    if not pr.Schema(sj).is_supported:
        return
    cols = _random_projection(rng, _names(sj))
    _check_damaged(coracle, sj, recs, k, cols, "interp")
    if seed % 6 == 0:
        _check_damaged(coracle, sj, recs, k, cols, "gen")


# ---- GPU -------------------------------------------------------------------------------------------------------------
class _GpuError(Exception):
    def __init__(self, status, message):
        super().__init__(message)
        m = re.search(r"\(record (-?\d+)\)", message)
        self.category, self.record = po.ERR_NAMES.get(status, str(status)), int(m.group(1)) if m else -1


def _gpu_host(s, data, off, n, k):
    data = np.ascontiguousarray(data, dtype=np.uint8)
    off = np.ascontiguousarray(off, dtype=np.int64)
    h = ctypes.c_void_p()
    rc = pr.lib.rv_decode_host(s.handle, data.ctypes.data if data.size else None, off.ctypes.data, n, k, ctypes.byref(h))
    if rc:
        raise _GpuError(rc, pr._last_error())
    return h.value


@pytest.fixture(params=["jit", "interp"])
def walker(request):
    pr.set_jit_enabled(1 if request.param == "jit" else 0)
    yield request.param
    pr.set_jit_enabled(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 33, 256, 257, 2500])
def test_gpu_random_schemas(coracle, walker, n):
    from tests.test_gpu_parity import JIT_SEEDS
    for seed in JIT_SEEDS[:3] if walker == "jit" else (n, n + 1, n + 2):
        sj, recs, data, off = gen_case(seed, n=n)
        rng = random.Random(seed * 31 + n)
        cols = _random_projection(rng, _names(sj))
        k = rng.choice([1, 2, 5])
        s = pr._get_or_parse_schema(sj, cols)
        got = pr._export_batches(_gpu_host(s, data, off, n, k), s)
        assert pr.last_walker() == walker
        _assert_selected(got, _oracle_batches(coracle, sj, data, off, n, k), cols, expected_schema(sj))


@pytest.mark.gpu
def test_gpu_every_entry_point(coracle):
    import workloads
    from tests.test_gpu_framed import _confluent, _ocf
    sj, data, off = workloads.generate("kafka", 20_000, seed=5)
    n = len(off) - 1
    recs = [data[off[i]:off[i + 1]].tobytes() for i in range(n)]
    want = {k: _oracle_batches(coracle, sj, data, off, n, k) for k in (1, 3)}
    exp = expected_schema(sj)
    for cols in C3_PROJECTIONS:
        _assert_selected([pr.deserialize_array(recs, sj, columns=cols)], want[1], cols, exp)
        _assert_selected(pr.deserialize_array_threaded(recs, sj, 3, columns=cols), want[3], cols, exp)
        _assert_selected(pr.deserialize_array_threaded_spawn(recs, sj, 3, columns=cols), want[3], cols, exp)
        _assert_selected(pr.deserialize_arrow_array(pa.array(recs, pa.binary()), sj, 3, columns=cols), want[3], cols, exp)
        _assert_selected(pr.decode_packed(data, off, n, sj, 3, columns=cols), want[3], cols, exp)
        _assert_selected(pr.deserialize_confluent(_confluent(recs, 9), sj, 3, schema_id=9, columns=cols), want[3], cols, exp)
        _assert_selected(pr.deserialize_ocf(_ocf(sj, recs, [1, 300, 1000], random.Random(1)), 3, columns=cols), want[3], cols, exp)
    with pytest.raises(ValueError, match="framed message.*record 0"):
        pr.deserialize_confluent(_confluent(recs[:10], 9), sj, 1, schema_id=8, columns=["age"])
    with pytest.raises(ValueError, match="no top-level field"):
        pr.deserialize_ocf(_ocf(sj, recs[:10], [10], random.Random(1)), 1, columns=["nope"])


@pytest.mark.gpu
def test_gpu_device_resident_kafka_2m_and_steady_state(coracle):
    import torch
    import workloads
    sj, data, off = workloads.generate("kafka", 2_000_000, seed=11)
    n = len(off) - 1
    dev = torch.device("cuda", 0)
    d_data = torch.zeros(len(data) + 64, dtype=torch.uint8, device=dev)
    d_data[:len(data)] = torch.from_numpy(data).to(dev)
    d_off = torch.from_numpy(np.ascontiguousarray(off, dtype=np.int64)).to(dev)
    stream = torch.cuda.current_stream(dev).cuda_stream

    def device_decode(s):
        h = ctypes.c_void_p()
        pr._check(pr.lib.rv_decode_device(s.handle, d_data.data_ptr(), d_off.data_ptr(), n, 4, stream, ctypes.byref(h)))
        return h.value

    def arrow_bytes_by_column(h, s):
        nbytes = pr.lib.rv_result_arrow_bytes(h)
        pr._check(pr.lib.rv_result_to_host(h))
        return nbytes, pr._export_batches(h, s)

    want = _oracle_batches(coracle, sj, data, off, n, 4)
    full = pr._get_or_parse_schema(sj)
    full_bytes, full_batches = arrow_bytes_by_column(device_decode(full), full)
    col_bytes = {}
    for name in full_batches[0].schema.names:   # the full result's bytes per column (validity counted when exported)
        col_bytes[name] = sum(sum(b.size for b in fb.column(name).buffers() if b is not None) for fb in full_batches)
    for cols in C3_PROJECTIONS:
        s = pr._get_or_parse_schema(sj, cols)
        pr.lib.rv_result_free(device_decode(s))
        h = device_decode(s)                     # the second call on the handle: one pass
        assert pr.lib.rv_last_passes() == 1
        nbytes, got = arrow_bytes_by_column(h, s)
        _assert_selected(got, want, cols, expected_schema(sj), full_validate=False)
        sel = sum(sum(b.size for b in fb.column(c).buffers() if b is not None) for fb in full_batches for c in cols)
        assert nbytes == sel <= full_bytes
    # the full handle is unaffected by the projected calls on the same schema string
    again_bytes, again = arrow_bytes_by_column(device_decode(full), full)
    assert again_bytes == full_bytes
    for b, w in zip(again, want):
        assert po.canon_diff(po.canon_from_batch(b), w) is None


@pytest.mark.gpu
@pytest.mark.timeout(600, method="thread")
def test_gpu_damaged_inputs_under_projections(coracle):
    seen = {"decoded": 0, "error": 0}
    for seed in range(60):
        rng = random.Random(seed)
        sj, recs, k = (M.damaged_case if seed % 2 else M.forged_case)(980000 + seed)
        if not pr.Schema(sj).is_supported:
            continue
        cols = _random_projection(rng, _names(sj))
        s = pr._get_or_parse_schema(sj, cols)
        data, off = po.pack_records(recs)
        want = M.expected(coracle, sj, recs)
        try:
            got = pr._export_batches(_gpu_host(s, data, off, len(recs), k), s)
        except _GpuError as e:
            assert (e.category, e.record) == want
            seen["error"] += 1
            continue
        if want is not None:
            assert want[0] == "overflow", want
            continue
        _assert_selected(got, _oracle_batches(coracle, sj, data, off, len(recs), k), cols, expected_schema(sj), full_validate=False)
        seen["decoded"] += 1
    assert seen["decoded"] > 5 and seen["error"] > 5


@pytest.mark.gpu
def test_gpu_projected_gather_on_one_device(coracle):
    import torch
    import workloads
    from pyruhvro_b200 import distributed as D
    from tests.test_gpu_gather import _split, _to_device
    sj, data, off = workloads.generate("kafka", 30_000, seed=3)
    cols = ["phone_numbers", "name", "created_at"]
    L = D._lib()
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev).cuda_stream
    handles, g = [], ctypes.c_void_p()
    try:
        for d, o in _split(data, off, [9_984, 10_240, 9_776]):
            d_data, d_off = _to_device(d, o, dev)
            s, h = D.decode_sharded(sj, d_data, d_off, len(o) - 1, 1, columns=cols)
            handles.append(h)
        m = int(L.rv_gather_meta_len(s.handle))
        metas = np.zeros((len(handles), max(m, 1)), dtype=np.int64)
        for r, h in enumerate(handles):
            pr._check(L.rv_result_gather_meta(h, 0, metas[r].ctypes.data, m))
        pr._check(L.rv_gather_plan(s.handle, metas.ctypes.data, len(handles), ctypes.byref(g)))
        assert L.rv_gather_num_groups(g) == 1
        base = ctypes.c_void_p()
        pr._check(L.rv_gather_alloc(g, 0, stream, ctypes.byref(base)))
        for r, h in enumerate(handles):
            pr._check(L.rv_gather_push(g, 0, r, h, 0, base, stream))
        res = ctypes.c_void_p()
        pr._check(L.rv_gather_finish(g, 0, ctypes.byref(res)))
        pr._check(L.rv_result_to_host(res))
        got = pr._export_batches(res.value, s)
    finally:
        L.rv_gather_free(g)
        for h in handles:
            L.rv_result_free(h)
    _assert_selected(got, _oracle_batches(coracle, sj, data, off, len(off) - 1, 1), cols, expected_schema(sj))
