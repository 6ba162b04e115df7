"""The fused kernel's device-only fast paths at their edges, every buffer against the C oracle.

Several pieces of the FAST walk exist only on the device (`#if defined(__CUDA_ARCH__)` in dev_core.cuh, and
dev_kernels.cuh): the shared -> shared string copy `copy_smem_words`, the three-word `varint_tail`, the funnel-shift
loads of `ld_le32` / `ld_le64`, `put_bit`'s ballot word, the staging map and write-out of the Utf8 bytes, and the real
shuffles / votes / item table of the item-parallel list emit.  Random schemas reach their edges only by chance, so the
records here are written by hand to reach them, and `reach()` proves from the oracle's output which edges the data
reached.  Each case runs twice:
  * on the GPU (`-m gpu`), both walkers, every buffer against the C oracle;
  * on the CPU through the host emulation of both walkers (and the lock-step warp emulation for the item-parallel
    cases), together with the coverage assertions — so the data and its claims hold before a GPU runs them."""
import ctypes
import json
import random
import struct
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import pyoracle as po
from tests import emu
from tests import test_emu_item_parallel as IP
from tests.emu import projection as P
from tests.emu import warp
from tests.parity import assert_matches_oracle, assert_matches_pyoracle_wide, expected_schema
from tests.test_emu_item_parallel import SCHEMA, record

TILE, WARP = 256, 32  # dev_types.h kBlock, warp size


# ---- wire encoding ----------------------------------------------------------------------------------------------
def uvar(z: int, width: int = 1) -> bytes:
    """Unsigned varint of `z` in at least `width` bytes (more than it needs: a padded, non-canonical encoding)."""
    out = []
    while True:
        out.append(z & 0x7F)
        z >>= 7
        if z == 0 and len(out) >= width:
            break
    return bytes([b | 0x80 for b in out[:-1]] + [out[-1]])


def zz(v: int) -> int:
    return ((v << 1) ^ (v >> 63)) & 0xFFFFFFFFFFFFFFFF


def unzz(z: int) -> int:
    return (z >> 1) ^ -(z & 1)


def svar(v: int) -> bytes:
    return uvar(zz(v))


def enc_str(b: bytes) -> bytes:
    return svar(len(b)) + b


def letters(rng, n: int) -> bytes:
    return bytes(rng.randrange(97, 123) for _ in range(n))


# ---- coverage accounting ----------------------------------------------------------------------------------------
# Layout facts the accounting relies on:
#  * Source.  A byte at packed offset x lands at a shared-memory address = x (mod 16): stage_in copies each tile's window
#    from the 16-byte aligned-down address of its first byte (TileWindow.mis), rv_decode_host uploads the packed bytes to
#    a device address = offsets[0] (mod 16) (engine.cu, decode_host_range: the `b0 & 15` shift), and rv_decode_device
#    requires a 16-byte aligned data pointer.
#  * Destination.  stage_map places chunk-relative Utf8 byte o of a stream at a staging address = (address of the
#    column's data buffer + o) (mod 16), and the arena's buffers are 64-byte aligned (engine.cu compute_layout /
#    arena_to_host round every buffer to 64 bytes), so the staging address = o (mod 16), o being the oracle's offset.
#  * Tiles are kBlock = 256 rows counted from each chunk's first row (tile_of); warps are 32 rows.
def _uvar_at(b: bytes, p: int):
    z, shift = 0, 0
    while True:
        x = b[p]
        p += 1
        z |= (x & 0x7F) << shift
        if not x & 0x80:
            return z & 0xFFFFFFFFFFFFFFFF, p
        shift += 7


def _walk(s, b, p, path, rec, log):
    """Wire positions of every leaf value of one record: log[path] += (record, position, wire bytes, raw value)."""
    k = s.kind
    if k == "union":
        z, p = _uvar_at(b, p)
        inner = s.variants[unzz(z)]
        return p if inner.kind == "null" else _walk(inner, b, p, path, rec, log)
    if k == "record":
        for name, fs, _ in s.fields:
            p = _walk(fs, b, p, path + (name,), rec, log)
        return p
    if k in ("int", "long"):
        z, q = _uvar_at(b, p)
        log.setdefault(path, []).append((rec, p, q - p, z))
        return q
    if k in ("float", "double"):
        n = 4 if k == "float" else 8
        log.setdefault(path, []).append((rec, p, n, int.from_bytes(b[p:p + n], "little")))
        return p + n
    if k in ("string", "bytes"):
        z, q = _uvar_at(b, p)
        n = unzz(z)
        log.setdefault(path, []).append((rec, q, n, None))
        return q + n
    if k == "enum":
        return _uvar_at(b, p)[1]
    if k in ("array", "map"):
        while True:
            z, p = _uvar_at(b, p)
            n = unzz(z)
            if n == 0:
                return p
            if n < 0:
                p = _uvar_at(b, p)[1]
                n = -n
            for _ in range(n):
                if k == "map":
                    p = _walk(po.AvroSchema("string"), b, p, path + ("key",), rec, log)
                    p = _walk(s.values, b, p, path + ("value",), rec, log)
                else:
                    p = _walk(s.items, b, p, path + ("[]",), rec, log)
    raise AssertionError(f"kind {k} is not used here")


def _canon_at(cols, names, path):
    c = cols[names.index(path[0])]
    for step in path[1:]:
        c = c["children"][0] if step == "[]" else c["children"][0]["children"][0 if step == "key" else 1]
    return c


def reach(sj, data, offsets, want, k, path):
    """Which edge cases the values of column `path` (a top-level field name, then "[]" / "key" / "value" steps) reached,
    given the packed input, the oracle's canonical batches `want` and the chunk count `k`.
      copies:  (destination words, source address mod 4, destination address mod 4) of every non-empty string copy
               (copy_smem_words: nwords = (d % 4 + len + 3) / 4);
      lengths: string lengths;  max_share: most records whose strings meet in one destination word;
      warp_edge / tile_edge: a destination word shared by lane 31 and lane 0 of the next warp / by the last row of a
               tile and the first of the next;
      tiles:   (tile's bytes in the column, destination of its first byte mod 16) of every tile (top-level columns);
      reads:   (wire bytes, source address mod 8, raw value) of every varint / float / double."""
    s = po.parse_schema(sj, wide=True)
    names = [f[0] for f in s.fields]
    data = np.asarray(data, dtype=np.uint8)
    n = len(offsets) - 1
    bounds = po.chunk_bounds(n, po.clamp_chunks(k, n))
    assert len(want) == len(bounds)
    log = {}
    for r in range(n):
        _walk(s, data[offsets[r]:offsets[r + 1]].tobytes(), 0, (), r, log)
    vals = log.get(tuple(path), [])
    out = SimpleNamespace(copies=set(), lengths=set(), max_share=0, warp_edge=False, tile_edge=False, tiles=set(),
                          reads={(w, int(offsets[r] + p) & 7, v) for r, p, w, v in vals if v is not None})
    if any(v is not None for *_, v in vals):
        return out
    chunk = np.searchsorted(np.array([b[1] for b in bounds]), np.arange(n), side="right")
    dsts = []
    for j, cols in enumerate(want):
        c = _canon_at(cols, names, path)
        off = np.frombuffer(c["buffers"][0], dtype="<i4")
        ln = np.diff(off)
        dsts += [(j, int(off[i]), int(ln[i])) for i in np.nonzero(ln)[0]]
        if len(path) == 1:
            out.tiles |= {(int(off[min(t + TILE, len(off) - 1)] - off[t]), int(off[t]) & 15) for t in range(0, len(off) - 1, TILE)}
    out.lengths = {ln for _, _, ln, _ in vals}
    srcs = [(r, int(offsets[r]) + p, ln) for r, p, ln, _ in vals if ln > 0]
    assert len(srcs) == len(dsts), (len(srcs), len(dsts))
    words = {}
    for (r, sa, ln), (j, d, ln2) in zip(srcs, dsts):
        assert ln == ln2 and chunk[r] == j
        out.copies.add((((d & 3) + ln + 3) >> 2, sa & 3, d & 3))
        row = r - bounds[j][0]
        for w in {d >> 2, (d + ln - 1) >> 2}:
            words.setdefault((j, w), set()).add(row)
    for rows in words.values():
        out.max_share = max(out.max_share, len(rows))
        for x in rows:
            if x + 1 in rows:
                out.warp_edge |= x % WARP == WARP - 1 and x % TILE != TILE - 1
                out.tile_edge |= x % TILE == TILE - 1
    return out


def assert_copy_matrix(rc, big=True):
    """All 16 (source mod 4, destination mod 4) pairs at every destination word count from 1 to 12 (0, 1, 4 and 5
    interior words, and one to three trips of the interior loop), and (big) a copy of at least 40 words."""
    missing = [(w, a, b) for w in range(1, 13) for a in range(4) for b in range(4) if (w, a, b) not in rc.copies]
    assert not missing, f"{len(missing)} copy cases not reached, e.g. {missing[:8]}"
    if big:
        assert max(w for w, _, _ in rc.copies) >= 40


def assert_tiles_fit(offsets, k, slack=1.3):
    """No full tile spans more than `slack` times the mean tile: the input window is sized for the largest tile up to
    1.5 times the mean (engine.cu configure), so every tile is walked in shared memory."""
    n = len(offsets) - 1
    mean = float(offsets[-1] - offsets[0]) / n * TILE
    for r0, r1 in po.chunk_bounds(n, po.clamp_chunks(k, n)):
        for t in range(r0, r1, TILE):
            assert offsets[min(t + TILE, r1)] - offsets[t] <= slack * mean


# ---- section: strings ---------------------------------------------------------------------------------------------
SYMBOLS = ["a", "bb", "ccc", "ddddd", "eeeeeeee", "fffffffffffff", "g" * 17, "h" * 31]
STR_SCHEMA = json.dumps({"type": "record", "name": "S", "fields": [
    {"name": "lead", "type": "long"},
    {"name": "s", "type": "string"},
    {"name": "ns", "type": ["null", "string"]},
    {"name": "arr", "type": {"type": "array", "items": "string"}},
    {"name": "m", "type": {"type": "map", "values": "string"}},
    {"name": "e", "type": {"type": "enum", "name": "E", "symbols": SYMBOLS}},
]})
BYTES_SCHEMA = json.dumps({"type": "record", "name": "B", "fields": [
    {"name": "lead", "type": "long"}, {"name": "b", "type": "bytes"}, {"name": "nb", "type": ["null", "bytes"]}]})

BIG_S = {17: 100, 60: 255, 101: 256, 150: 1000, 200: 4096, 240: 16384}  # row % 256 -> length of `s` (16384: 3-byte length)
BIG_A = {33: 100, 80: 255, 120: 1000, 170: 4096}                        # row % 256 -> length of `arr`'s first item
TINY_LANES = (29, 30, 31, 0, 1, 2)  # row % 32 -> `s` of 1-3 bytes: destination words shared by up to 4 lanes, across warps and tiles


def lead_value(rng, width: int) -> int:
    """A raw zigzag value whose varint takes `width` bytes: the bytes before `s` shift its source alignment."""
    return rng.randrange(0 if width == 1 else 1 << (7 * (width - 1)), 1 << (7 * width))


def str_values(rng, r):
    t = r % TILE
    ls = BIG_S.get(t, rng.randint(1, 3) if r % WARP in TINY_LANES else rng.randint(0, 64))
    arr = [letters(rng, rng.randint(0, 64) if rng.random() < 0.6 else rng.randint(1, 5)) for _ in range(rng.randint(0, 3))]
    if t in BIG_A:
        arr = [letters(rng, BIG_A[t])] + arr
    return {"lead": lead_value(rng, rng.randint(1, 4)), "s": letters(rng, ls),
            "ns": None if rng.random() < 0.3 else letters(rng, rng.randint(0, 8)), "arr": arr,
            "m": [(letters(rng, rng.randint(0, 6)), letters(rng, rng.randint(0, 10))) for _ in range(rng.randint(0, 2))],
            "e": rng.randrange(len(SYMBOLS))}


def str_record(v, odd=None) -> bytes:
    """One STR_SCHEMA record.  odd: a valid encoding the FAST walk does not take ("not plain"): "branch" writes `ns`'s
    union branch as 82 00, "enum" the enum index padded to two bytes, "negblock" `arr` as a negative block count
    followed by the block's byte size."""
    out = bytearray(uvar(v["lead"]) + enc_str(v["s"]))
    out += b"\x00" if v["ns"] is None else (uvar(2, 2) if odd == "branch" else b"\x02") + enc_str(v["ns"])
    if v["arr"]:
        items = b"".join(enc_str(x) for x in v["arr"])
        out += (svar(-len(v["arr"])) + svar(len(items)) if odd == "negblock" else svar(len(v["arr"]))) + items
    out += b"\x00"
    if v["m"]:
        out += svar(len(v["m"])) + b"".join(enc_str(a) + enc_str(b) for a, b in v["m"])
    out += b"\x00"
    out += uvar(zz(v["e"]), 2 if odd == "enum" else 1)
    return bytes(out)


class CopyPlan:
    """Steers string lengths towards copy cases (destination words 1-12, source mod 4, destination mod 4) not yet
    reached, given where the next string's bytes start and where they go."""

    def __init__(self):
        self.need = {(w, a, b) for w in range(1, 13) for a in range(4) for b in range(4)}

    def length(self, src: int, dst: int, default: int) -> int:
        for w, a, b in sorted(self.need):
            if a == src & 3 and b == dst & 3:
                self.need.discard((w, a, b))
                return max(1, 4 * w - 3 - b)  # the shortest string of w words from destination offset b
        return default


def string_case(n=3072, seed=1):
    """The lengths of `s` and of `arr`'s items are steered towards every copy case within rows 0-1023 (the first
    chunk for both k = 1 and k = 3), where the source is the packed offset and the destination the column's running
    byte count.  `s` also picks its source alignment through the width of the `lead` varint in front of it."""
    rng = random.Random(seed)
    plan_s, plan_a = CopyPlan(), CopyPlan()
    recs, pos, cum_s, cum_a = [], 0, 0, 0
    for r in range(n):
        v = str_values(rng, r)
        here = sorted(x for x in plan_s.need if x[2] == cum_s & 3)
        if r % TILE not in BIG_S and r % WARP not in TINY_LANES and here:
            w, a, b = here[0]
            plan_s.need.discard((w, a, b))
            width = (a - pos - 1) % 4 + 1  # `s`'s bytes start after the lead varint and a one-byte length
            v["lead"] = lead_value(rng, width)
            v["s"] = letters(rng, max(1, 4 * w - 3 - b))
        rec = str_record(v)
        # `arr`'s items: where each starts in the record, then steer its length
        p = len(uvar(v["lead"])) + len(enc_str(v["s"])) + (1 if v["ns"] is None else 1 + len(enc_str(v["ns"])))
        if v["arr"]:
            p += len(svar(len(v["arr"])))
            for i, x in enumerate(v["arr"]):
                if len(x) < 60:
                    v["arr"][i] = x = letters(rng, plan_a.length(pos + p + 1, cum_a, len(x)))
                p += len(enc_str(x))
                cum_a += len(x)
            rec = str_record(v)
        recs.append(rec)
        pos += len(rec)
        cum_s += len(v["s"])
    return recs, *po.pack_records(recs)


def write_out_plan():
    """Per-tile totals of the sparse column: every total in {0, 1..17, 31, 32, 33} at every destination offset mod 16
    of the tile's first byte (stage_write_out's head / 16-byte body / tail split).  Greedy: take a total still needed
    at the current offset, else move the offset to one that still has needs."""
    need = {(t, m) for t in [0, *range(1, 18), 31, 32, 33] for m in range(16)}
    seq, pos = [], 0
    while need:
        m = pos % 16
        here = sorted(t for t, mm in need if mm == m)
        t = here[0] if here else next(t for t in range(1, 17) if any(mm == (m + t) % 16 for _, mm in need))
        need.discard((t, m))
        seq.append(t)
        pos += t
    return seq


def sparse_case():
    """Minimal records whose `ns` is null except for one or two values per tile, which make up the planned totals."""
    rng = random.Random(3)
    recs = []
    for i, total in enumerate(write_out_plan()):
        vals = [None] * TILE
        rows = sorted(rng.sample(range(TILE), 2))
        if total >= 2 and i % 2:
            a = rng.randint(1, total - 1)
            vals[rows[0]], vals[rows[1]] = letters(rng, a), letters(rng, total - a)
        else:
            vals[rows[1]] = letters(rng, total)
        for v in vals:
            recs.append(str_record({"lead": 0, "s": b"", "ns": v, "arr": [], "m": [], "e": 0}))
    return recs, *po.pack_records(recs)


PRECISE_ROWS = [2 * WARP + 7, 3 * WARP + 31] + [TILE + w * WARP + (5 * w) % WARP for w in range(8) if w != 5]
ODD = ("branch", "enum", "negblock")


def precise_case(n=1024):
    """string_case data with valid but not plain records in chosen lanes (warp 2 lane 7, warp 3 lane 31, one lane of
    every warp of tile 1 but warp 5): their warps emit with the precise walker, staging their strings into the same
    words as the fast warps next to them."""
    rng = random.Random(5)
    recs = []
    for r in range(n):
        v = str_values(rng, r)
        odd = None
        if r in PRECISE_ROWS:
            odd = ODD[PRECISE_ROWS.index(r) % 3]
            v["ns"] = v["ns"] if v["ns"] is not None else letters(rng, 3)
            v["arr"] = v["arr"] or [letters(rng, 5), b""]
        recs.append(str_record(v, odd))
    return recs, *po.pack_records(recs)


def bytes_case(n=3072):
    rng = random.Random(9)
    recs = []
    for r in range(n):
        lb = BIG_S.get(r % TILE, rng.randint(1, 3) if r % WARP in TINY_LANES else rng.randint(0, 64))
        nb = None if rng.random() < 0.3 else bytes(rng.randrange(256) for _ in range(rng.randint(0, 12)))
        recs.append(uvar(lead_value(rng, rng.randint(1, 4))) + enc_str(bytes(rng.randrange(256) for _ in range(lb)))
                    + (b"\x00" if nb is None else b"\x02" + enc_str(nb)))
    return recs, *po.pack_records(recs)


def check_string_reach(coracle, data, off, n, k):
    want = coracle.decode_threaded_packed(STR_SCHEMA, data, off, n, k, threads=4)
    s = reach(STR_SCHEMA, data, off, want, k, ["s"])
    assert set(range(65)) | set(BIG_S.values()) <= s.lengths
    assert_copy_matrix(s)
    assert s.max_share >= 3 and s.warp_edge and s.tile_edge
    assert_copy_matrix(reach(STR_SCHEMA, data, off, want, k, ["arr", "[]"]))


# ---- section: fast readers ----------------------------------------------------------------------------------------
NUM_SCHEMA = json.dumps({"type": "record", "name": "N", "fields": [
    {"name": "pad", "type": "string"},
    {"name": "l", "type": "long"},
    {"name": "i", "type": "int"},
    {"name": "f", "type": "float"},
    {"name": "d", "type": "double"},
    {"name": "nl", "type": ["null", "long"]},
    {"name": "xs", "type": {"type": "array", "items": "long"}},
]})


def _ends(widths):
    """Raw zigzag values at both ends of every varint width (even: >= 0, odd: < 0)."""
    out = []
    for w in widths:
        lo, hi = (0 if w == 1 else 1 << (7 * (w - 1))), min((1 << (7 * w)) - 1, (1 << 64) - 1)
        out += [(lo, None), (lo + 1, None), (hi - 1, None), (hi, None)]
    return out


# (raw zigzag value, padded width or None): i64::MIN / i64::MAX are the two ends of width 10
LONGS = _ends(range(1, 11)) + [(0, 2), (0, 3), (1, 5), (2, 7), (300, 6), (zz(-5), 9), (0, 10), (zz(2**40), 10)]
INTS = _ends(range(1, 6)) + [(zz(2**31), None), (zz(-2**31), None), (0, 3), (zz(-7), 6), (zz(2**31 - 1), 10)]
F32 = [0x00000000, 0x80000000, 0x00000001, 0x7F7FFFFF, 0x7F800000, 0xFF800000, 0x7FC12345, 0x7F800001]
F64 = [0, 1 << 63, 1, 0x7FEFFFFFFFFFFFFF, 0x7FF0000000000000, 0xFFF0000000000000, 0x7FF8000000012345, 0x7FF0000000000001]
# validity of `nl` per warp: all null, all valid, alternating, only lane 0 / 31 valid, only lane 0 / 31 null
PATTERNS = [lambda l: False, lambda l: True, lambda l: l % 2 == 1, lambda l: l == 0, lambda l: l == 31,
            lambda l: l != 0, lambda l: l != 31]


def num_case(k, n=620):
    """Every varint / float / double of the lists above at every source alignment (mod 4 for varints, mod 8 for
    floats), placed by the length of the `pad` string in front of them; `nl`'s validity per warp of each chunk follows
    PATTERNS; `xs` lists of 64-200 items (two-byte block counts) now and then."""
    targets = [("l", z, w, a) for z, w in LONGS for a in range(4)] + [("i", z, w, a) for z, w in INTS for a in range(4)]
    targets += [("f", b, None, a) for b in F32 for a in range(8)] + [("d", b, None, a) for b in F64 for a in range(8)]
    rng = random.Random(13)
    bounds = po.chunk_bounds(n, po.clamp_chunks(k, n))
    recs, pos = [], 0
    for r in range(n):
        j = next(j for j, (r0, r1) in enumerate(bounds) if r0 <= r < r1)
        row = r - bounds[j][0]
        col, val, width, align = targets[r % len(targets)]
        fl = {"l": LONGS[r % len(LONGS)], "i": INTS[(r * 7) % len(INTS)], "f": F32[(r * 3) % 8], "d": F64[(r * 5) % 8]}
        fl[col] = (val, width) if col in "li" else val
        body = [uvar(fl["l"][0], fl["l"][1] or 1), uvar(fl["i"][0], fl["i"][1] or 1),
                struct.pack("<I", fl["f"]), struct.pack("<Q", fl["d"])]
        before = sum(len(x) for x in body[:"lifd".index(col)])
        pad = (align - (pos + 1 + before)) % (4 if col in "li" else 8)
        out = enc_str(letters(rng, pad)) + b"".join(body)
        valid = PATTERNS[(j + row // WARP) % len(PATTERNS)](row % WARP)
        out += b"\x02" + svar(rng.randint(-2**40, 2**40)) if valid else b"\x00"
        items = rng.randint(64, 200) if r % 17 == 0 else rng.randint(0, 3)
        out += (svar(items) + b"".join(svar(rng.randint(-300, 300)) for _ in range(items)) if items else b"") + b"\x00"
        recs.append(out)
        pos += len(out)
    return recs, *po.pack_records(recs)


def check_num_reach(coracle, data, off, n, k):
    want = coracle.decode_threaded_packed(NUM_SCHEMA, data, off, n, k, threads=4)
    for col, vals, mod in (("l", LONGS, 4), ("i", INTS, 4), ("f", [(b, None) for b in F32], 8), ("d", [(b, None) for b in F64], 8)):
        got = {(v, a % mod) for _, a, v in reach(NUM_SCHEMA, data, off, want, k, [col]).reads}
        missing = [(v, a) for v, _ in vals for a in range(mod) if (v, a) not in got]
        assert not missing, (col, missing[:8])
    widths = {w for w, _, _ in reach(NUM_SCHEMA, data, off, want, k, ["l"]).reads}
    assert widths >= set(range(1, 11))
    assert any(len(svar(c)) == 2 for c in _block_counts(data, off))  # two-byte block counts
    # every validity pattern, in full and partial warps (the chunk's last warp)
    seen = set()
    for j, cols in enumerate(want):
        c = _canon_at(cols, [f[0] for f in po.parse_schema(NUM_SCHEMA).fields], ["nl"])
        bits = np.unpackbits(np.frombuffer(c["validity"], dtype=np.uint8), bitorder="little")[:c["length"]]
        for w0 in range(0, c["length"], WARP):
            lanes = bits[w0:w0 + WARP]
            seen |= {i for i, p in enumerate(PATTERNS) if all(bool(b) == p(l) for l, b in enumerate(lanes))}
    assert seen == set(range(len(PATTERNS)))


def _block_counts(data, off):
    s = po.parse_schema(NUM_SCHEMA)
    out = []
    for r in range(len(off) - 1):
        b = np.asarray(data)[off[r]:off[r + 1]].tobytes()
        p = 0
        for name, fs, _ in s.fields[:-1]:
            p = _walk(fs, b, p, (name,), r, {})
        out.append(unzz(_uvar_at(b, p)[0]))
    return out


# ---- section: item-parallel emit ----------------------------------------------------------------------------------
PROJECTIONS = [["tags"], ["attrs", "id"], ["tail", "tags"]]


def item_cases():
    """(name, records) of tests/test_emu_item_parallel.py: every lane with at most kItemSlots items, a lane beyond
    the table, a list over 255 bytes, and the boundary cases."""
    out = []
    for n in (1, 33, 700):
        for split in (False, True):
            rng = random.Random(n * 2 + split)
            out.append((f"within_{n}_{'split' if split else 'one'}", [record(rng, IP.K, split) for _ in range(n)]))
    rng = random.Random(5)
    recs = [record(rng, IP.K, True) for _ in range(512)]
    for r in (3, 40, 41, 300):
        recs[r] = record(rng, 9, True)
    out.append(("beyond_table", recs))
    rng = random.Random(6)
    recs = [record(rng, IP.K, False) for _ in range(96)]
    long_tag = letters(rng, 300)
    recs[37] = record(rng, IP.K, False, first_tag=IP.varint(len(long_tag)) + long_tag)
    out.append(("over_255_bytes", recs))
    return out + IP.boundary_cases()


ITEM_CASES = [name for name, _ in item_cases()]


def tags_case(n=2048):
    """Records of 1-4 tags (or one long tag of 160-200 bytes) whose lists stay within 255 bytes, so every warp emits
    item-parallel: the tags' string cursors come from the warp scans."""
    rng = random.Random(21)
    recs = []
    for r in range(n):
        if r % 97 == 0:
            tags = [enc_str(letters(rng, rng.randint(160, 200)))]
        else:
            while True:
                tags = [enc_str(letters(rng, rng.randint(0, 48))) for _ in range(rng.randint(1, IP.K))]
                if IP.tags_span(tags) <= 255:
                    break
        recs.append(IP.tagged(rng, tags))
    return recs, *po.pack_records(recs)


# schemas (and projected plans) whose generated walkers tools/warm_jit_cache.py precompiles
JIT_SCHEMAS = [STR_SCHEMA, BYTES_SCHEMA, NUM_SCHEMA, SCHEMA]
JIT_PROJECTIONS = [(SCHEMA, cols) for cols in PROJECTIONS]


# ==== CPU: the same cases through the host emulation ================================================================
@pytest.mark.parametrize("k", [1, 3])
def test_emu_string_copy_matrix(coracle, k):
    recs, data, off = string_case()
    assert_tiles_fit(off, k)
    check_string_reach(coracle, data, off, len(recs), k)
    for w in ("gen", "interp"):
        assert_matches_oracle(coracle, emu.decode(STR_SCHEMA, data, off, len(recs), k, walker=w), STR_SCHEMA, data, off, len(recs), k)


def test_emu_bytes_copy_matrix():
    recs, data, off = bytes_case()
    s = po.parse_schema(BYTES_SCHEMA, wide=True)
    want = [po.py_decode(s, recs[r0:r1]) for r0, r1 in po.chunk_bounds(len(recs), 1)]
    assert_copy_matrix(reach(BYTES_SCHEMA, data, off, want, 1, ["b"]))
    for w in ("gen", "interp"):
        assert_matches_pyoracle_wide(emu.decode(BYTES_SCHEMA, data, off, len(recs), 1, walker=w), BYTES_SCHEMA, recs, 1)


def test_emu_write_out_matrix(coracle):
    recs, data, off = sparse_case()
    want = coracle.decode_threaded_packed(STR_SCHEMA, data, off, len(recs), 1, threads=4)
    tiles = reach(STR_SCHEMA, data, off, want, 1, ["ns"]).tiles
    missing = [(t, m) for t in [0, *range(1, 18), 31, 32, 33] for m in range(16) if (t, m) not in tiles]
    assert not missing, missing[:8]
    for w in ("gen", "interp"):
        assert_matches_oracle(coracle, emu.decode(STR_SCHEMA, data, off, len(recs), 1, walker=w), STR_SCHEMA, data, off, len(recs), 1)


def test_emu_precise_warps_in_staged_tiles(coracle):
    recs, data, off = precise_case()
    rng = random.Random(0)
    for odd in ODD:   # the oracle accepts each encoding, with the values of the canonical one
        v = str_values(rng, 0)
        v["ns"], v["arr"] = b"xyz", [b"ab", b""]
        assert coracle.decode(STR_SCHEMA, [str_record(v, odd)]) == coracle.decode(STR_SCHEMA, [str_record(v)])
        assert str_record(v, odd) != str_record(v)
    for w in ("gen", "interp"):
        assert_matches_oracle(coracle, emu.decode(STR_SCHEMA, data, off, len(recs), 1, walker=w), STR_SCHEMA, data, off, len(recs), 1)


@pytest.mark.parametrize("k", [1, 3])
def test_emu_fast_readers(coracle, k):
    recs, data, off = num_case(k)
    check_num_reach(coracle, data, off, len(recs), k)
    for w in ("gen", "interp"):
        assert_matches_oracle(coracle, emu.decode(NUM_SCHEMA, data, off, len(recs), k, walker=w), NUM_SCHEMA, data, off, len(recs), k)


def test_emu_tags_copy_matrix_and_projections(coracle):
    recs, data, off = tags_case()
    for k in (1, 3):
        want = coracle.decode_threaded_packed(SCHEMA, data, off, len(recs), k, threads=4)
        assert_copy_matrix(reach(SCHEMA, data, off, want, k, ["tags", "[]"]))
        assert_matches_oracle(coracle, warp.decode(SCHEMA, data, off, len(recs), k), SCHEMA, data, off, len(recs), k)
        for cols in PROJECTIONS:
            for w in ("interp", "gen", "warp"):
                _assert_selected(P.decode(SCHEMA, data, off, len(recs), k, cols, walker=w), want, cols)


def _assert_selected(batches, want, cols):
    exp = expected_schema(SCHEMA)
    idx = [exp.names.index(c) for c in cols]
    assert len(batches) == len(want)
    for i, (b, w) in enumerate(zip(batches, want)):
        assert b.schema.names == cols
        b.validate(full=True)
        d = po.canon_diff(po.canon_from_batch(b), [w[j] for j in idx], f"batch[{i}]")
        assert d is None, d


# ==== GPU ===========================================================================================================
@pytest.fixture(params=["jit", "interp"])
def walker(request):
    import pyruhvro_b200 as pr
    pr.set_jit_enabled(1 if request.param == "jit" else 0)
    yield request.param
    pr.set_jit_enabled(-1)


def gpu_host(sj, data, off, n, k, columns=None):
    """rv_decode_host, after one warm-up call that teaches the schema handle the tiles' sizes; (batches, slow tiles)."""
    import pyruhvro_b200 as pr
    pr.decode_packed(data, off, n, sj, k, columns=columns)
    got = pr.decode_packed(data, off, n, sj, k, columns=columns)
    return got, pr.lib.rv_last_slow_tiles()


def gpu_device(sj, data, off, n, k):
    """rv_decode_device on a 16-byte aligned torch buffer (warm-up call, then the measured one); (batches, slow tiles)."""
    import torch
    import pyruhvro_b200 as pr
    s = pr._get_or_parse_schema(sj)
    total = int(off[n])
    d_data = torch.zeros(total + 64, dtype=torch.uint8, device="cuda")
    assert d_data.data_ptr() % 16 == 0
    d_data[:total].copy_(torch.from_numpy(np.array(data[:total], dtype=np.uint8)))
    d_off = torch.from_numpy(np.ascontiguousarray(off, dtype=np.int64)).cuda()
    for _ in range(2):
        h = ctypes.c_void_p()
        pr._check(pr.lib.rv_decode_device(s.handle, d_data.data_ptr(), d_off.data_ptr(), n, k,
                                          torch.cuda.current_stream().cuda_stream, ctypes.byref(h)))
        slow = pr.lib.rv_last_slow_tiles()
        pr._check(pr.lib.rv_result_to_host(h))
        got = pr._export_batches(h.value, s)
    return got, slow


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3])
def test_gpu_string_copy_matrix(coracle, walker, k):
    recs, data, off = string_case()
    n = len(recs)
    check_string_reach(coracle, data, off, n, k)
    got, slow = gpu_host(STR_SCHEMA, data, off, n, k)
    assert slow == 0
    assert_matches_oracle(coracle, got, STR_SCHEMA, data, off, n, k)
    got, slow = gpu_device(STR_SCHEMA, data, off, n, k)
    assert slow == 0
    assert_matches_oracle(coracle, got, STR_SCHEMA, data, off, n, k)


@pytest.mark.gpu
def test_gpu_bytes_copy_matrix(walker):
    recs, data, off = bytes_case()
    got, slow = gpu_host(BYTES_SCHEMA, data, off, len(recs), 1)
    assert slow == 0
    assert_matches_pyoracle_wide(got, BYTES_SCHEMA, recs, 1)


@pytest.mark.gpu
def test_gpu_write_out_matrix(coracle, walker):
    recs, data, off = sparse_case()
    got, slow = gpu_host(STR_SCHEMA, data, off, len(recs), 1)
    assert slow == 0
    assert_matches_oracle(coracle, got, STR_SCHEMA, data, off, len(recs), 1)


@pytest.mark.gpu
def test_gpu_precise_warps_in_staged_tiles(coracle, walker):
    recs, data, off = precise_case()
    got, slow = gpu_host(STR_SCHEMA, data, off, len(recs), 1)
    assert slow == 0
    assert_matches_oracle(coracle, got, STR_SCHEMA, data, off, len(recs), 1)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3])
def test_gpu_fast_readers(coracle, walker, k):
    recs, data, off = num_case(k)
    got, _ = gpu_host(NUM_SCHEMA, data, off, len(recs), k)
    assert_matches_oracle(coracle, got, NUM_SCHEMA, data, off, len(recs), k)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ITEM_CASES)
def test_gpu_item_parallel(coracle, name):
    """The generated walker's item-parallel emit with the device's shuffles, votes and item table.  That it ran is
    the construction, not a counter: where every lane has at most kItemSlots items and a list of at most 255 bytes,
    no lane's table entry is kItemSeq, so the warp's vote (warp_any) is false and the warp emits item-parallel."""
    import pyruhvro_b200 as pr
    assert "items_par_" in pr.Schema(SCHEMA).walker_source
    recs = dict(item_cases())[name]
    data, off = po.pack_records(recs)
    pr.set_jit_enabled(1)
    try:
        for k in (1, 2, 3):
            got, _ = gpu_host(SCHEMA, data, off, len(recs), k)
            assert pr.last_walker() == "jit"
            assert_matches_oracle(coracle, got, SCHEMA, data, off, len(recs), k)
    finally:
        pr.set_jit_enabled(-1)


@pytest.mark.gpu
def test_gpu_tags_copy_matrix_and_projections(coracle):
    import pyruhvro_b200 as pr
    recs, data, off = tags_case()
    n = len(recs)
    pr.set_jit_enabled(1)
    try:
        for k in (1, 3):
            want = coracle.decode_threaded_packed(SCHEMA, data, off, n, k, threads=4)
            assert_copy_matrix(reach(SCHEMA, data, off, want, k, ["tags", "[]"]))
            full, _ = gpu_host(SCHEMA, data, off, n, k)
            assert_matches_oracle(coracle, full, SCHEMA, data, off, n, k)
            for cols in PROJECTIONS:
                got, _ = gpu_host(SCHEMA, data, off, n, k, columns=cols)
                assert pr.last_walker() == "jit"
                _assert_selected(got, want, cols)
                assert all(g.equals(f.select(cols)) for g, f in zip(got, full))
    finally:
        pr.set_jit_enabled(-1)
