"""Cases of permissive multi-version decodes (Versions.permissive, errors="null" of deserialize_confluent_versions and
deserialize_single_object_versions).

The contract: a message's verdict is the strict versions decode of that message alone, with the same registry.  A bad
message becomes a null row and is reported with its index, status and the strict message without "(record N)".  The
batches equal the permissive single-schema decode deserialize_confluent(L', R, k, errors="null") of a rebuilt list L':
a good message becomes its value resolved with its own writer and re-encoded as an R datum, Confluent-framed; a bad
message becomes a message with a wrong magic byte."""
import ctypes
import random
import re
import struct

import numpy as np

import pyruhvro_b200 as pr
from oracle import pyoracle as po
from tests import mutation as M
from tests import resolution as RS
from tests import versions_cases as VC

UNKNOWN_ID = 0xFFFFFFFF   # writer_chain draws ids below 2^20
DAMAGES = ["datum", "magic", "short", "unregistered"]


def so_frame(fp: int, datum: bytes) -> bytes:
    return b"\xc3\x01" + struct.pack("<Q", fp) + datum


class Case:
    """Messages of `writers` (dict id -> json) read as `rj`; single_object: framed by fingerprint instead of id."""

    def __init__(self, rng, writers, rj, n, single_object=False, columns=None):
        self.writers, self.rj, self.so, self.columns = writers, rj, single_object, columns
        self.hdr = 10 if single_object else 5
        ids = VC.mix(rng, writers, n, rng.choice(["runs", "alternate"])) if n else []
        self.recs, self.vals = VC.messages(rng, writers, ids)
        if single_object:
            self.fps = {i: pr.Schema(sj).fingerprint for i, sj in writers.items()}
            self.recs = [so_frame(self.fps[i], r[5:]) for (i, _), r in zip(self.vals, self.recs)]
        self.orig = list(self.recs)

    def damage(self, rng, at, kind=None):
        """Damage message `at`; a damage that leaves it decodable is undone (its value must stay known)."""
        kind = kind or rng.choice(DAMAGES)
        r = self.orig[at]
        h, body = r[:self.hdr], r[self.hdr:]
        if kind == "datum":
            m = h + M.damage(random.Random(rng.random()), [body] * 4)[rng.randrange(4)]
            if m == r:
                m = h + body[:max(len(body) // 2 - 1, 0)]
        elif kind == "magic":
            m = bytes([h[0] ^ 0x41]) + r[1:]
        elif kind == "short":
            m = r[:rng.randrange(self.hdr)]
        else:
            m = so_frame(0x0123456789ABCDEF, body) if self.so else VC.frame(UNKNOWN_ID, body)
        self.recs[at] = m

    def registry(self):
        if self.so:
            return pr.Versions([self.writers[i] for i in sorted(self.writers)], self.rj, self.columns, single_object=True)
        return pr.Versions(self.writers, self.rj, self.columns)

    def verdicts(self, strict: "pr.Versions"):
        """[(index, status, text)] of the messages whose strict decode alone fails; damaged messages that decode are
        restored first."""
        out = []
        for i, m in enumerate(self.recs):
            v = strict_verdict(strict, m)
            if v is None and m != self.orig[i]:
                self.recs[i] = self.orig[i]
                v = strict_verdict(strict, self.orig[i])
            if v is not None:
                out.append((i,) + v)
        return out

    def oracle(self, bad, k):
        """deserialize_confluent(L', R, k, errors="null") with L' as in the module doc."""
        rs = po.parse_schema(self.rj)
        parsed = {i: po.parse_schema(sj) for i, sj in self.writers.items()}
        meta = RS.ReaderMeta(self.rj)
        bad_at = {i for i, _, _ in bad}
        lp = []
        for i, (sid, v) in enumerate(self.vals):
            if i in bad_at:
                lp.append(b"\x01\x00\x00\x00\x00")
            else:
                lp.append(VC.frame(1, po.encode_datum(rs, RS.resolve_value(parsed[sid], rs, v, meta))))
        return pr.deserialize_confluent(lp, self.rj, k, columns=self.columns, errors="null")[0]


def strict_verdict(strict: "pr.Versions", msg: bytes):
    """(status, message without "(record 0)") of the strict decode of `msg` alone, or None."""
    data = np.frombuffer(msg + b"\x00" * 16, dtype=np.uint8)
    off = np.array([0, len(msg)], dtype=np.int64)
    h = ctypes.c_void_p()
    st = pr.lib.rv_decode_host_versions(strict.handle, data.ctypes.data, off.ctypes.data, 1, 1, ctypes.byref(h))
    if st == 0:
        pr.lib.rv_result_free(h.value)
        return None
    text = pr._last_error()
    return st, re.sub(r" \(record 0\)$", "", text)


def report(bad):
    """[(record, status, error)] of a bad-message report RecordBatch."""
    assert bad.schema.names == ["record", "status", "error"]
    return list(zip(bad.column(0).to_pylist(), bad.column(1).to_pylist(), bad.column(2).to_pylist()))


def compare(got, want, what=""):
    assert len(got) == len(want), (what, len(got), len(want))
    for i, (b, w) in enumerate(zip(got, want)):
        assert b.schema.equals(w.schema), (what, i, b.schema, w.schema)
        d = po.canon_diff(po.canon_from_batch(b), po.canon_from_batch(w), f"{what} batch[{i}]")
        assert d is None, d
