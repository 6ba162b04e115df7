"""Expected results of permissive decodes (errors="null", Schema.permissive), shared by tests/test_permissive.py (host
emulation) and tests/test_gpu_permissive.py (the device).

The contract: a record's verdict is the strict decode of that record alone.  A good record's row holds its values; a bad
record's row is null in every top-level column.  The batches are, buffer for buffer, the plain decode with R' (every
top-level field that is neither a union nor null made optional) of the input in which each good record is re-encoded
as an R' datum and each bad record is the R' datum with branch null in every optional field.  Two kinds of column have
no validity at a bad row.  A map column (R' cannot make it optional) holds an empty map there.  An N-variant union
column holds type id 0 and absent children, which no datum encodes unless branch 0 is null; for those columns the good
rows are compared and the bad rows checked for type id 0."""
import json
import random

import numpy as np
import pyarrow as pa

from oracle import pyoracle as po

# rv_status of each oracle error category (include/ruhvro_b200.h)
STATUS = {"eof": 1, "varint": 2, "bool": 3, "neg_len": 4, "branch": 5, "enum": 6, "schema": 7, "overflow": 8, "value": 11, "frame": 12}


def _is_optional_kind(t) -> bool:
    """Fields R' leaves as they are: unions, null, and maps (["null", map] has no Arrow form here)."""
    return isinstance(t, list) or t in ("null", "map") or (isinstance(t, dict) and t.get("type") in ("null", "map"))


def _is_map(t) -> bool:
    return t == "map" or (isinstance(t, dict) and t.get("type") == "map")


def optional_json(schema_json: str) -> str:
    """R' of a record schema: T -> ["null", T]; a field with a non-null default -> [T, "null"] (schema.cpp optional_fields)."""
    s = json.loads(schema_json)
    for f in s["fields"]:
        if _is_optional_kind(f["type"]):
            continue
        f["type"] = [f["type"], "null"] if f.get("default", None) is not None else ["null", f["type"]]
    return json.dumps(s)


def split_fields(s: po.AvroSchema, rec: bytes):
    """The bytes of each top-level field of a record that decodes."""
    c = po._Cur(rec)
    spans = []
    for f in s.fields:
        a = c.p
        po._decode(po._make(f[1]), c)
        spans.append(rec[a:c.p])
    return spans


def verdict(coracle, schema_json: str, rec: bytes, wide: bool = False):
    """None for a good record, else the oracle's error category of the record decoded alone."""
    try:
        if wide:
            po.py_decode(po.parse_schema(schema_json, wide=True), [rec])
        else:
            coracle.decode(schema_json, [rec])
        return None
    except po.DecodeError as e:
        return e.code


class Expected:
    """What a permissive decode of `recs` (plain handle of `schema_json`) must give."""

    def __init__(self, coracle, schema_json: str, recs, k: int, wide: bool = False, verdicts=None):
        self.sj, self.wide = schema_json, wide
        self.rj = optional_json(schema_json)
        s = po.parse_schema(schema_json, wide=wide)
        top = json.loads(schema_json)["fields"]
        self.verdicts = verdicts if verdicts is not None else [verdict(coracle, schema_json, r, wide) for r in recs]
        self.bad = [(i, STATUS[v]) for i, v in enumerate(self.verdicts) if v is not None]
        self.union_cols = [j for j, f in enumerate(top) if isinstance(f["type"], list) and not self._nullable_pair(f["type"])]
        rng = random.Random(len(recs))
        out = []
        for r, v in zip(recs, self.verdicts):
            parts = []
            spans = split_fields(s, r) if v is None else None
            for j, (f, fs) in enumerate(zip(top, s.fields)):
                t = f["type"]
                if v is None:
                    if _is_optional_kind(t):
                        parts.append(spans[j])
                    else:
                        parts.append((b"\x00" if f.get("default", None) is not None else b"\x02") + spans[j])
                elif t == "null" or (isinstance(t, dict) and t.get("type") == "null"):
                    pass
                elif _is_map(t):   # an empty map: what the absent path writes
                    parts.append(b"\x00")
                elif not isinstance(t, list):
                    parts.append(b"\x02" if f.get("default", None) is not None else b"\x00")
                elif self._nullable_pair(t):
                    parts.append(b"\x00" if self._is_null(t[0]) else b"\x02")
                else:  # N-variant union: branch 0 (a placeholder value unless it is null; see the module doc)
                    b = bytearray(b"\x00")
                    v0 = fs[1].variants[0]
                    if v0.kind != "null":
                        po.encode_value(v0, po.random_value(v0, rng), b)
                    parts.append(bytes(b))
            out.append(b"".join(parts))
        self.recs = out
        n = len(out)
        self.bounds = po.chunk_bounds(n, po.clamp_chunks(k, n))
        if wide:
            rs = po.parse_schema(self.rj, wide=True)
            self.batches = [po.py_decode(rs, out[a:b]) for a, b in self.bounds]
        else:
            data, off = po.pack_records(out)
            self.batches = coracle.decode_threaded_packed(self.rj, data, off, n, k, threads=4)

    @staticmethod
    def _is_null(t) -> bool:
        return t == "null" or (isinstance(t, dict) and t.get("type") == "null")

    def _nullable_pair(self, t) -> bool:
        return len(t) == 2 and sum(self._is_null(x) for x in t) == 1

    def check(self, batches, bad, columns=None):
        """`batches` of the decoder under test, `bad`: [(record, status)] it reported.  columns: a projection (names)."""
        assert list(bad) == self.bad, f"bad records {list(bad)[:10]} != {self.bad[:10]}"
        top = [f["name"] for f in json.loads(self.sj)["fields"]]
        sel = list(range(len(top))) if columns is None else [top.index(c) for c in columns]
        assert len(batches) == len(self.batches)
        bad_rows = {i for i, _ in self.bad}
        for bi, (b, w, (r0, r1)) in enumerate(zip(batches, self.batches, self.bounds)):
            assert b.num_rows == r1 - r0
            got = po.canon_from_batch(b)
            for out_j, j in enumerate(sel):
                if j in self.union_cols and not self._branch0_null(j):
                    col = b.column(out_j)
                    tids = np.frombuffer(col.buffers()[1], dtype=np.int8)[col.offset:col.offset + len(col)]
                    want = po.canon_to_arrow(w[j], b.schema.field(out_j).type)
                    a = r0
                    while a < r1:   # the runs of good rows compare whole; every bad row has type id 0
                        if a in bad_rows:
                            assert tids[a - r0] == 0, f"batch {bi} row {a - r0}: union type id {tids[a - r0]} at a bad row"
                            a += 1
                            continue
                        e = a
                        while e < r1 and e not in bad_rows:
                            e += 1
                        assert col.slice(a - r0, e - a).equals(want.slice(a - r0, e - a)), f"batch {bi} rows {a - r0}..{e - r0} of {top[j]}"
                        a = e
                    continue
                d = po.canon_diff(got[out_j], w[j], f"batch[{bi}].{top[j]}")
                assert d is None, d

    def _branch0_null(self, j) -> bool:
        t = json.loads(self.sj)["fields"][j]["type"]
        return self._is_null(t[0])


def pack(recs):
    return po.pack_records(recs)
