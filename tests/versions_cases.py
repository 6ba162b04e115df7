"""Cases of the multi-version Confluent decode (deserialize_confluent_versions): writer schemas drawn from random
evolution chains, message mixes of their ids, and the oracle's batches — each message resolved with its own writer's
schema (tests/resolution.py), re-encoded with the reader's and decoded by the oracle in k chunks."""
import json
import random
import struct

import pyruhvro_b200 as pr
from oracle import pyoracle as po
from tests import resolution as RS


def frame(sid: int, datum: bytes) -> bytes:
    return b"\x00" + struct.pack(">I", sid) + datum


def resolves(wj: str, rj: str) -> bool:
    try:
        pr.Schema(wj).read_as(rj)
        return True
    except ValueError:
        return False


def writer_chain(rng, wide=False, unmapped_ok=False):
    """(reader, {id: writer}): 3 to 6 writers from one evolution chain that resolve to its last schema, the reader itself
    among them."""
    chain = [po.random_schema_json(rng, wide=wide)]
    for _ in range(rng.randint(3, 6)):
        try:
            chain.append(RS.random_evolution(rng, chain[-1], wide=wide, unmapped_ok=unmapped_ok))
        except ValueError:   # an evolution of an evolution may reuse an added field's name: branch from the start instead
            chain.append(RS.random_evolution(rng, chain[0], wide=wide, unmapped_ok=unmapped_ok))
    rj = chain[-1]
    ws = []
    for sj in chain:
        if sj not in ws and resolves(sj, rj):
            ws.append(sj)
    ids = rng.sample(range(1, 1 << 20), len(ws))
    return rj, dict(zip(ids, ws))


def mix(rng, ids, n, kind, k=1):
    """The schema id of every message: "one" (the first id only), "runs" (runs of random length), "alternate" (strict
    per-message alternation), "absent" (the last id only outside chunk 0), "single" (chunk 0 holds one id only)."""
    ids = list(ids)
    if kind == "one":
        return [ids[0]] * n
    if kind == "alternate":
        return [ids[i % len(ids)] for i in range(n)]
    if kind == "runs":
        out = []
        while len(out) < n:
            out += [rng.choice(ids)] * rng.randint(1, 300)
        return out[:n]
    cr = n // max(1, min(k, n))
    if kind == "absent":
        return [ids[-1] if i >= cr and rng.random() < 0.5 else rng.choice(ids[:-1] or ids) for i in range(n)]
    if kind == "single":
        return [ids[0] if i < cr else rng.choice(ids) for i in range(n)]
    raise ValueError(kind)


def messages(rng, writers, id_seq, wide=False):
    """(framed messages, [(id, value)])"""
    parsed = {i: po.parse_schema(sj, wide=wide) for i, sj in writers.items()}
    vals = [(i, po.random_value(parsed[i], rng)) for i in id_seq]
    return [frame(i, po.encode_datum(parsed[i], v)) for i, v in vals], vals


def expected(coracle, writers, rj, vals, k, wide=False):
    """The oracle's batches, or ("error", index) for the first message whose enum symbol the reader cannot map."""
    rs = po.parse_schema(rj, wide=wide)
    parsed = {i: po.parse_schema(sj, wide=wide) for i, sj in writers.items()}
    meta = RS.ReaderMeta(rj)
    rvals = []
    for m, (i, v) in enumerate(vals):
        try:
            rvals.append(RS.resolve_value(parsed[i], rs, v, meta))
        except RS.Unmapped:
            return ("error", m)
    recs = [po.encode_datum(rs, v) for v in rvals]
    n = len(recs)
    if wide:
        return [po.py_decode(rs, recs[a:b]) for a, b in po.chunk_bounds(n, po.clamp_chunks(k, n))]
    data, off = po.pack_records(recs)
    return coracle.decode_threaded_packed(rj, data, off, n, k, threads=4)


def compare(got, want, what=""):
    assert len(got) == len(want), (what, len(got), len(want))
    for i, (b, w) in enumerate(zip(got, want)):
        d = po.canon_diff(po.canon_from_batch(b), w, f"{what} batch[{i}]")
        assert d is None, d


def roles_of(t, depth=0, out=None):
    """Which slot roles (plan.hpp SlotRole) an Arrow type's buffers take, and the deepest list nesting."""
    import pyarrow as pa
    out = out if out is not None else {"roles": set(), "depth": 0, "map": False}
    out["depth"] = max(out["depth"], depth)
    if pa.types.is_boolean(t):
        out["roles"].add("Bits")
    elif pa.types.is_string(t) or pa.types.is_binary(t):
        out["roles"] |= {"Offsets", "Data"}
    elif pa.types.is_fixed_size_binary(t) or pa.types.is_decimal(t):
        out["roles"].add("ValuesW")
    elif pa.types.is_union(t):
        out["roles"].add("TypeIds")
    elif pa.types.is_map(t):
        out["map"] = True
        out["roles"].add("Offsets")
        roles_of(t.key_type, depth + 1, out)
        roles_of(t.item_type, depth + 1, out)
    elif pa.types.is_list(t):
        out["roles"].add("Offsets")
        roles_of(t.value_type, depth + 1, out)
    elif pa.types.is_struct(t):
        for f in t:
            roles_of(f.type, depth, out)
    elif pa.types.is_null(t):
        pass
    elif t.bit_width == 32:
        out["roles"].add("Values32")
    elif t.bit_width == 64:
        out["roles"].add("Values64")
    if pa.types.is_union(t):
        for f in t:
            roles_of(f.type, depth, out)
    return out


def schema_roles(rj, out=None):
    out = out if out is not None else {"roles": set(), "depth": 0, "map": False}
    for f in pr.Schema(rj).arrow_schema:
        if f.nullable:
            out["roles"].add("Validity")
        roles_of(f.type, 0, out)
    return out


# A hand-made pair: a reader-only nullable record (null default: an absent subtree in the writer's plan), a map, three
# list levels, a promotion and a writer non-union read as a nullable field.
ABSENT_W = json.dumps({"type": "record", "name": "R", "fields": [
    {"name": "a", "type": "int"},
    {"name": "m", "type": {"type": "map", "values": "string"}},
    {"name": "l3", "type": {"type": "array", "items": {"type": "array", "items": {"type": "array", "items": "int"}}}}]})
ABSENT_R = json.dumps({"type": "record", "name": "R", "fields": [
    {"name": "a", "type": ["null", "long"], "default": None},
    {"name": "m", "type": {"type": "map", "values": "string"}},
    {"name": "l3", "type": {"type": "array", "items": {"type": "array", "items": {"type": "array", "items": "int"}}}},
    {"name": "rec", "type": ["null", {"type": "record", "name": "In", "fields": [
        {"name": "x", "type": "int"}, {"name": "s", "type": ["null", "string"]}]}], "default": None},
    {"name": "flag", "type": "boolean", "default": True}]})


# ---- bench scale (GPU): Kafka messages of workloads.KAFKA_SCHEMA (v1) and workloads.kafka_v2_schema() (v2) -------------
def kafka_versions_input(n, mix, ids=(3, 4), k=8, seed=42):
    """(data uint8, offsets int64, plain source batches of the oracle's input, v1 json, v2 json): n Confluent messages,
    message i framed with ids[sel(i)] and holding row i of workloads.generate("kafka", n) encoded with that id's schema
    (v1: the generated datum; v2: the row read as v2 and re-encoded by the GPU encoder).  mix: "one", "alternate" or
    ("runs", length).  With four ids, ids[2] and ids[3] name v1 and v2 again."""
    import numpy as np
    import pyarrow as pa
    import pyarrow.compute as pc
    import workloads
    v1, h_data, h_off = workloads.generate("kafka", n, seed=seed)
    v2 = workloads.kafka_v2_schema()
    h_data, h_off = np.ascontiguousarray(h_data), np.ascontiguousarray(h_off, dtype=np.int64)
    as_v2 = pr.decode_packed(h_data, h_off, n, v1, k, reader_schema=v2)
    i = np.arange(n)
    if mix == "one":
        sel = np.zeros(n, dtype=np.int64)
    elif mix == "alternate":
        sel = i % len(ids)
    else:
        sel = (i // mix[1]) % len(ids)
    plain = pr.decode_packed(h_data, h_off, n, v1, k)
    out, row = [], 0
    for part_v1, b2 in zip(plain, as_v2):
        m = b2.num_rows
        cand = [pr.serialize_confluent(part_v1, v1, ids[q], 1)[0] if q % 2 == 0 else pr.serialize_confluent(b2, v2, ids[q], 1)[0]
                for q in range(len(ids))]
        s = sel[row:row + m]
        pick = cand[0].cast(pa.large_binary())
        for q in range(1, len(ids)):
            pick = pc.if_else(pa.array(s == q), cand[q].cast(pa.large_binary()), pick)
        out.append(pick)
        row += m
    arr = pa.concat_arrays(out)
    data, off, _ = pr._packed_view(arr)
    return np.ascontiguousarray(data), np.ascontiguousarray(off, dtype=np.int64), h_data, h_off, v1, v2


def check_kafka_v2(batches, v1, v2, h_data, h_off, n, k):
    """Every buffer of the v2 batches against the C oracle's decode of the v1 source rows, converted as v2 reads them."""
    import os
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from bench_resolve import expected_v2
    want = po.COracle().decode_threaded_packed(v1, h_data, h_off, n, k, threads=os.cpu_count() or 4)
    plain_schema = pr.Schema(v1).arrow_schema
    v2_schema = pr.Schema(v2).arrow_schema
    assert len(batches) == len(want)
    for i, (b, w) in enumerate(zip(batches, want)):
        exp = expected_v2(po.canon_to_batch(w, plain_schema), v2_schema)
        for j, col in enumerate(exp):
            assert b.column(j).equals(col), f"batch {i} column {v2_schema.names[j]} differs from the oracle"
