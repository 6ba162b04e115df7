"""Schema resolution's device paths at their edges, against an exact reference (tests/exact_numbers.py).

Resolution adds three pieces to the fused walk (dev_core.cuh): `op_promote` (int / long / float read as a wider
number), `op_default` (a reader-only field's constant: a number, or bytes copied from the symbol table by
`copy_from_symbols`) and `op_enum`'s remap check.  Random values reach their edges only by chance, so the records here
are written by hand:
  * promotions at rounding ties and range ends, every varint width at every source offset mod 4 (the FAST walk's
    three-word `varint_tail`), ints whose varints lie outside the i32 range, floats of every class (NaN payloads and
    signalling NaNs too) at every offset mod 4 (`ld_le32`), in FAST warps and in warps the precise walker emits;
  * numeric defaults that round twice, underflow, overflow, and 64-bit constants whose halves must stay apart;
  * default strings and enum text of many lengths staged into shared words next to other lanes' bytes, at warp and
    tile edges, in 256- and 384-row tiles, and a default too big to stage;
  * a 70-symbol enum read by readers with and without a default, unmapped symbols in FAST and precise lanes.
The promoted and numeric default columns are compared as raw bits with their validity; every other column against the
oracle's decode of the converted values (tests/resolution.py).  Each case runs on the CPU through the host emulation,
with assertions that the packed input reaches the edges it claims, and on the GPU with both walkers."""
import ctypes
import json
import random

import numpy as np
import pytest

import pyruhvro_b200 as pr
from oracle import pyoracle as po
from tests import emu
from tests import exact_numbers as X
from tests import resolution as RS
from tests.emu import resolve as R
from tests.test_gpu_fast_paths import _uvar_at, _walk, enc_str, letters, svar, unzz, uvar, zz

WARP = 32
M64 = X.M64


def varint(spec) -> bytes:
    """(raw zigzag value, width, bits or-ed into a 10th byte) -> wire bytes; padded past the value's own width."""
    z, width, hi = spec
    b = bytearray(uvar(z & M64, width))
    if hi:
        assert len(b) == 10
        b[9] |= hi
    return bytes(b)


def canon(v):
    return (zz(v), 1, 0)


def min_width(z):
    return len(uvar(z))


def rec(*fields, name="R"):
    return dict(type="record", name=name, fields=list(fields))


def fld(name, t, **kw):
    return dict({"name": name, "type": t}, **kw)


def with_raw_defaults(j, raw):
    """JSON text of schema `j` whose defaults "@@i@@" are replaced by the number texts raw[i], verbatim."""
    s = json.dumps(j)
    for i, t in enumerate(raw):
        s = s.replace(f'"@@{i}@@"', t)
    return s


def flavour_rows(off, k, is_odd):
    """Per record: True where its warp (rows of the same chunk, 32 at a time) has a lane the FAST walk cannot take, so
    the whole warp emits with the precise walker."""
    n = len(off) - 1
    out = np.zeros(n, dtype=bool)
    for r0, r1 in po.chunk_bounds(n, po.clamp_chunks(k, n)):
        for w0 in range(r0, r1, WARP):
            out[w0:min(w0 + WARP, r1)] = any(is_odd(r) for r in range(w0, min(w0 + WARP, r1)))
    return out


def warp_plan(n, k, odd_every=4):
    """(precise warps, odd rows): every `odd_every`-th warp of each chunk carries two records the FAST walk cannot take."""
    odd = set()
    for r0, r1 in po.chunk_bounds(n, po.clamp_chunks(k, n)):
        for w, w0 in enumerate(range(r0, r1, WARP)):
            if w % odd_every == 1:
                odd |= {w0 + (7 * w) % WARP, w0 + (7 * w + 13) % WARP}
    return {r for r in odd if r < n}


def assert_tiles_fit(off, k, tile=256, slack=1.3):
    n = len(off) - 1
    mean = float(off[-1] - off[0]) / n * tile
    for r0, r1 in po.chunk_bounds(n, po.clamp_chunks(k, n)):
        for t in range(r0, r1, tile):
            assert off[min(t + tile, r1)] - off[t] <= slack * mean


# ==== a-d, g: promotions and numeric defaults =======================================================================
def _long_values():
    v = [0, 1, -1, 2**31 - 1, -2**31, 2**63 - 1, -2**63]
    v += [2**24 + d for d in range(-2, 4)] + [2**53 + d for d in range(-2, 4)]
    for e in (25, 31, 40, 53, 62):   # float ties: halfway to the next float, on an even and on an odd mantissa
        for h in (2**e + 2**(e - 24), 2**e + 3 * 2**(e - 24)):
            v += [h - 1, h, h + 1]
    for e in (54, 60, 62):           # double ties
        for h in (2**e + 2**(e - 53), 2**e + 3 * 2**(e - 53)):
            v += [h - 1, h, h + 1]
    v += [2**60 + 2**36 + 1, 2**62 + 2**38 + 2**9 + 1]   # float results that a rounding through double would change
    v = sorted(set(v) | {-x for x in v if -x >= -2**63})
    return [x for x in v if -2**63 <= x < 2**63]


def _int_values():
    v = [0, 1, -1, 2**31 - 1, -2**31, 2**31 - 64, 2**31 - 65] + [2**24 + d for d in range(-2, 4)]
    for e in (25, 28, 30):
        for h in (2**e + 2**(e - 24), 2**e + 3 * 2**(e - 24)):
            v += [h - 1, h, h + 1]
    return sorted(set(v) | {-x for x in v if -x >= -2**31})


LONGS = _long_values()
INTS = _int_values()
# int varints outside the i32 range (a writer's int decode keeps the low 32 bits): (raw zigzag, width, 10th-byte bits)
WILD_INTS = [(zz(2**31), 5, 0), (zz(-2**31 - 1), 5, 0), (zz(2**32 + 7), 5, 0), (zz(-2**35 - 3), 6, 0), (zz(2**40 + 2**24 + 1), 7, 0),
             (zz(-2**49), 8, 0), (zz(2**56 + 2**31), 9, 0), (zz(2**63 - 1), 10, 0), (zz(-2**63), 10, 0), (zz(2**62 + 5), 10, 0x7E),
             (zz(-2**33 + 2**24 + 1), 10, 0x40), ((1 << 64) - 1, 10, 0x7E), (1 << 35, 10, 0x02)]
F32S = [0x00000000, 0x80000000, 0x00000001, 0x80000001, 0x007FFFFF, 0x00800000, 0x7F7FFFFF, 0xFF7FFFFF, 0x7F800000, 0xFF800000,
        0x3F800001, 0x7FC12345, 0xFFC00001, 0x7FC00000, 0x7F800001, 0x7FBFFFFF, 0xFF800001, 0x7FFFFFFF]

PROMO_W = json.dumps(rec(fld("pad", "string"), fld("l", "long"), fld("ld", "long"), fld("i", "int"), fld("il", "int"), fld("id", "int"),
                         fld("f", "float"), fld("nl", ["null", "long"]), fld("u", ["null", "string"]),
                         fld("xs", {"type": "array", "items": "long"}), name="P"))
DEF_F = ["-0.0", "1e-45", "1e-46", "3.4028235e38", "3.5e38", "-1e39", "1.00000005960464477540", "0.1", "16777217"]
DEF_D = ["-0.0", "5e-324", "1e-400", "1.7976931348623157e308", "0.1", "-2.5e-310", "9007199254740993"]
DEF_L = [-2**63, 2**63 - 1, -2**32, 2**32 - 1]
DEF_I = [-2**31, 2**31 - 1]
_RAW = DEF_F + DEF_D + [str(x) for x in DEF_L + DEF_I] + ["5e-324"]
_ph = iter(f"@@{i}@@" for i in range(len(_RAW)))
PROMO_DEFAULTS = ([fld(f"df{i}", "float", default=next(_ph)) for i in range(len(DEF_F))]
                  + [fld(f"dd{i}", "double", default=next(_ph)) for i in range(len(DEF_D))]
                  + [fld(f"dl{i}", "long", default=next(_ph)) for i in range(len(DEF_L))]
                  + [fld(f"di{i}", "int", default=next(_ph)) for i in range(len(DEF_I))]
                  + [fld("dn", ["double", "null"], default=next(_ph))])
_OTHER = [fld("pad", "string"), fld("u", ["null", "string"]), fld("xs", {"type": "array", "items": "long"})]
PROMO_R = with_raw_defaults(rec(fld("f", ["null", "double"]), fld("l", "float"), PROMO_DEFAULTS[0], _OTHER[0], fld("ld", "double"),
                                *PROMO_DEFAULTS[1:8], fld("i", "float"), fld("nl", ["null", "double"]), fld("il", "long"), _OTHER[1],
                                *PROMO_DEFAULTS[8:], fld("id", "double"), _OTHER[2], name="P"), _RAW)
PROMO_OTHER_R = json.dumps(rec(*_OTHER, name="P"))   # the columns the oracle checks

# reader column -> (dtype, per-record expectation from the writer's values)
PROMOTED = {"l": (np.uint32, lambda v: X.int_to_f32_bits(unzz(v["l"][0]))),
            "ld": (np.uint64, lambda v: X.int_to_f64_bits(unzz(v["ld"][0]))),
            "i": (np.uint32, lambda v: X.int_to_f32_bits(X.int32_of_varint(v["i"][0]))),
            "il": (np.uint64, lambda v: X.int32_of_varint(v["il"][0]) & M64),
            "id": (np.uint64, lambda v: X.int_to_f64_bits(X.int32_of_varint(v["id"][0]))),
            "f": (np.uint64, lambda v: X.widen_f32_bits(v["f"])),
            "nl": (np.uint64, lambda v: None if v["nl"] is None else X.int_to_f64_bits(unzz(v["nl"][0])))}
DEFAULT_BITS = dict([(f"df{i}", (np.uint32, X.decimal_text_to_f32_bits(t))) for i, t in enumerate(DEF_F)]
                    + [(f"dd{i}", (np.uint64, X.decimal_text_to_f64_bits(t))) for i, t in enumerate(DEF_D)]
                    + [(f"dl{i}", (np.uint64, x & M64)) for i, x in enumerate(DEF_L)]
                    + [(f"di{i}", (np.uint32, x & 0xFFFFFFFF)) for i, x in enumerate(DEF_I)]
                    + [("dn", (np.uint64, X.decimal_text_to_f64_bits("5e-324")))])
VARINT_COLS = ("l", "ld", "i", "il", "id")


def promo_targets():
    """(column, varint spec or float bits, source offset mod 4): every long value at every width from its own to 10 in
    `l` and `ld`; every int value at widths up to 5 and the out-of-range ints in `i`, `il` and `id`; every float
    class in `f`.  All at every offset mod 4."""
    t = []
    for col in ("l", "ld"):
        t += [(col, (zz(x), w, 0)) for x in LONGS for w in range(min_width(zz(x)), 11)]
    for col in ("i", "il", "id"):
        t += [(col, (zz(x), w, 0)) for x in INTS for w in range(min_width(zz(x)), 6)] + [(col, s) for s in WILD_INTS]
    t += [("f", b) for b in F32S]
    return [(c, v, a) for c, v in t for a in range(4)]


def promo_record(v, odd=None) -> bytes:
    """odd: "branch" writes `u`'s union branch as 82 00, "negblock" `xs` as a negative block count and a byte size —
    valid encodings the FAST walk leaves to the precise one."""
    out = bytearray(enc_str(v["pad"]))
    for c in VARINT_COLS:
        out += varint(v[c])
    out += v["f"].to_bytes(4, "little")
    out += b"\x00" if v["nl"] is None else b"\x02" + varint(v["nl"])
    out += b"\x00" if v["u"] is None else (uvar(2, 2) if odd == "branch" else b"\x02") + enc_str(v["u"])
    if v["xs"]:
        items = b"".join(svar(x) for x in v["xs"])
        out += (svar(-len(v["xs"])) + svar(len(items)) if odd == "negblock" else svar(len(v["xs"]))) + items
    return bytes(out + b"\x00")


def _offset_in_record(v, col):
    p = len(enc_str(v["pad"]))
    for c in VARINT_COLS:
        if c == col:
            return p
        p += len(varint(v[c]))
    return p   # "f"


def promo_case(k):
    """Records whose FAST warps take the targets one each, the pad string in front placing each at its offset; every
    fourth warp of a chunk holds two odd records and emits precise, its lanes cycling through every value."""
    rng = random.Random(11)
    targets = promo_targets()
    cyc = {"l": [canon(x) for x in LONGS], "ld": [canon(x) for x in reversed(LONGS)], "f": F32S,
           **{c: [canon(x) for x in INTS] + WILD_INTS for c in ("i", "il", "id")}}
    n = int(len(targets) * 4 / 3) + 256
    odd = warp_plan(n, k)
    recs, vals, pos, ti, pc = [], [], 0, 0, 0
    precise = flavour_rows(np.arange(n + 1), k, lambda x: x in odd)
    for r in range(n):
        v = {c: cyc[c][(r * (3 + j)) % len(cyc[c])] for j, c in enumerate(("l", "ld", "i", "il", "id", "f"))}
        v["pad"] = b""
        v["nl"] = None if r % 3 == 0 else cyc["ld"][(r * 5) % len(LONGS)]
        v["u"] = None if r % 5 == 0 else letters(rng, rng.randint(0, 6))
        v["xs"] = [rng.randint(-300, 300) for _ in range(rng.randint(0, 3))]
        kind = None
        if r in odd:
            kind = ("branch", "negblock")[r % 2]
            v["u"] = v["u"] or b"odd"
            v["xs"] = v["xs"] or [5, -7]
        if precise[r]:
            for j, c in enumerate(("l", "ld", "i", "il", "id", "f")):
                v[c] = cyc[c][(pc + 11 * j) % len(cyc[c])]
            pc += 1
        elif ti < len(targets):
            col, val, align = targets[ti]
            ti += 1
            v[col] = val
            v["pad"] = letters(rng, (align - pos - _offset_in_record(v, col)) % 4)
        recs.append(promo_record(v, kind))
        vals.append(v)
        pos += len(recs[-1])
    assert ti == len(targets)
    data, off = po.pack_records(recs)
    return recs, vals, data, off, odd


def _promo_reads(data, off, col):
    """(record, wire bytes, source offset mod 4, raw value) of every value of writer column `col`, from the packed input."""
    s = po.parse_schema(PROMO_W)
    log = {}
    for r in range(len(off) - 1):
        _walk(s, bytes(data[off[r]:off[r + 1]]), 0, (), r, log)
    return [(r, w, (int(off[r]) + p) & 3, v) for r, p, w, v in log[(col,)]]


def _odd_kind(b: bytes):
    """Which encoding of a PROMO_W record the FAST walk cannot take, read from its bytes."""
    p = _uvar_at(b, 0)[1]
    p += unzz(_uvar_at(b, 0)[0])
    for _ in VARINT_COLS:
        p = _uvar_at(b, p)[1]
    p += 4
    z, p = _uvar_at(b, p)
    if z:
        p = _uvar_at(b, p)[1]
    if b[p] == 0x82:
        return "branch"
    z, p = _uvar_at(b, p)
    if z:
        n, p = _uvar_at(b, p)
        p += unzz(n)
    return "negblock" if unzz(_uvar_at(b, p)[0]) < 0 else None


def check_promo_reach(recs, data, off, k):
    precise = flavour_rows(off, k, lambda r: _odd_kind(recs[r]) is not None)
    assert 0.15 < precise.mean() < 0.5
    for col in VARINT_COLS + ("f",):
        got = _promo_reads(data, off, col)
        fast = {(w, a, v) for r, w, a, v in got if not precise[r]}
        slow = {v for r, w, a, v in got if precise[r]}
        if col == "f":
            assert {(4, a, b) for b in F32S for a in range(4)} <= fast, col
            assert set(F32S) <= slow
            continue
        values = LONGS if col in ("l", "ld") else INTS
        need = {(w, a, zz(x)) for x in values for w in range(min_width(zz(x)), 11 if col in ("l", "ld") else 6) for a in range(4)}
        assert need <= fast, (col, sorted(need - fast)[:5])
        assert {zz(x) for x in values} <= slow, col
        if col not in ("l", "ld"):
            assert {(s[1], a, s[0]) for s in WILD_INTS for a in range(4)} <= fast
            assert {s[0] for s in WILD_INTS} <= slow
    # every shift of the three-word varint_tail: tails ending in the low word (widths 3-6) and the high word (7-10)
    tails = {(w, (a + 2) & 3) for r, w, a, _ in _promo_reads(data, off, "l") if not precise[r] and w >= 3}
    assert tails == {(w, s) for w in range(3, 11) for s in range(4)}
    # 10th bytes whose high bits fall off (the reads above found them at every offset, in both flavours)
    assert sum(1 for b in recs if any(varint(x) in b for x in WILD_INTS if x[2])) >= 8
    assert_tiles_fit(off, k)


def assert_promo_batches(batches, vals, k, coracle):
    n = len(vals)
    bounds = po.chunk_bounds(n, po.clamp_chunks(k, n))
    assert len(batches) == len(bounds)
    want_other = RS.expected_batches(coracle, PROMO_W, PROMO_OTHER_R, [{c: _po_val(v, c) for c in ("pad", "u", "xs")} for v in vals], k)
    names = [f["name"] for f in json.loads(PROMO_OTHER_R)["fields"]]
    for j, (b, (r0, r1)) in enumerate(zip(batches, bounds)):
        assert b.num_rows == r1 - r0
        assert b.schema.names == [f["name"] for f in json.loads(PROMO_R)["fields"]]
        for col, (dt, fn) in list(PROMOTED.items()) + [(c, (dt, (lambda v, x=x: x))) for c, (dt, x) in DEFAULT_BITS.items()]:
            a = b.column(col)
            want = [fn(v) for v in vals[r0:r1]]
            got = np.frombuffer(a.buffers()[1], dtype=dt)[a.offset:a.offset + len(a)]
            exp = np.array([0 if x is None else x for x in want], dtype=dt)
            bad = np.nonzero(got != exp)[0]
            assert not len(bad), f"batch {j} column {col} row {r0 + bad[0]}: got {int(got[bad[0]]):#x} want {int(exp[bad[0]]):#x}"
            valid = np.array([x is not None for x in want])
            if a.buffers()[0] is None:   # (no bitmap: no nulls)
                assert valid.all() and a.null_count == 0, (j, col)
            else:
                bits = np.unpackbits(np.frombuffer(a.buffers()[0], dtype=np.uint8), bitorder="little")[a.offset:a.offset + len(a)]
                assert (bits.astype(bool) == valid).all() and a.null_count == int((~valid).sum()), (j, col)
        d = po.canon_diff(po.canon_from_batch(b.select(names)), want_other[j], f"batch[{j}]")
        assert d is None, d


def _po_val(v, c):
    if c == "u":
        return (0, None) if v["u"] is None else (1, v["u"])
    return v[c]


# ==== e-g: default strings, enum text, enum remapping ===============================================================
def utf8_of_len(n, salt=0) -> str:
    """A string of exactly `n` UTF-8 bytes mixing 1- to 4-byte characters."""
    chars = ["é", "✓", "\U0001D11E", "a", "Ω", "z"]
    out, size, i = [], 0, salt
    while size < n:
        c = chars[i % len(chars)]
        i += 1
        if size + len(c.encode()) > n:
            c = "q"
        out.append(c)
        size += len(c.encode())
    return "".join(out)


W_SYMS = [f"S{i}" + "x" * (i * 5 % 11) for i in range(70)]        # texts of 2-14 bytes
UNMAPPED = {2, 5, 11, 40, 62, 63, 64, 66, 69}                     # writer symbols the reader does not have
R_SYMS = ["NEWA"] + [s for i, s in enumerate(W_SYMS) if i not in UNMAPPED][::-1] + ["Dq"]
ENUM_W = {"type": "enum", "name": "E", "symbols": W_SYMS}
ENUM_R1 = {"type": "enum", "name": "E", "symbols": R_SYMS, "default": "Dq"}
ENUM_R2 = {"type": "enum", "name": "E", "symbols": R_SYMS}
_TAIL = fld("tail", ["null", "string"])
_XS = fld("xs", {"type": "array", "items": "long"})
STR_W = json.dumps(rec(fld("lead", "long"), fld("e", ENUM_W), _TAIL, _XS, name="T"))
SHORT_DEFAULTS = [fld(f"ds{n}", "string", default=utf8_of_len(n, n)) for n in range(14)]
LONG_DEFAULTS = [fld(f"db{n}", "string", default=utf8_of_len(n, n)) for n in (31, 32, 33, 301)]
STR_RA = json.dumps(rec(*SHORT_DEFAULTS[:7], fld("e", ENUM_R1), *SHORT_DEFAULTS[7:], _TAIL, _XS, name="T"))   # > 8 streams
STR_RB = json.dumps(rec(LONG_DEFAULTS[0], fld("e", ENUM_R1), *LONG_DEFAULTS[1:], _TAIL, _XS, name="T"))
STR_RC = json.dumps(rec(fld("e", ENUM_R1), fld("dbig", "string", default=utf8_of_len(1200, 3)), _TAIL, name="T"))  # too big to stage
STR_RD = json.dumps(rec(fld("e", ENUM_R2), _TAIL, _XS, name="T"))   # no default: unmapped symbols fail


def str_record(v, odd=None) -> bytes:
    out = bytearray(svar(v["lead"]) + uvar(zz(v["e"]), 1))
    out += b"\x00" if v["tail"] is None else (uvar(2, 2) if odd == "branch" else b"\x02") + enc_str(v["tail"])
    if v["xs"]:
        items = b"".join(svar(x) for x in v["xs"])
        out += (svar(-len(v["xs"])) + svar(len(items)) if odd == "negblock" else svar(len(v["xs"]))) + items
    return bytes(out + b"\x00")


def str_case(k, n=2600, mapped_only=False):
    """Every fourth warp of a chunk emits precise: it holds two odd records, and only its lanes take enum indices of 64
    and above (two varint bytes: not plain).  The FAST warps take indices 0-63 (63 is the last one-byte index).
    mapped_only: every unmapped index replaced by the next mapped one."""
    rng = random.Random(23)
    odd = warp_plan(n, k)
    precise = flavour_rows(np.arange(n + 1), k, lambda r: r in odd)
    recs, vals, pc = [], [], 0
    for r in range(n):
        if precise[r]:
            e, pc = (pc * 3) % 70, pc + 1
        else:
            e = (r * 37 + r // 7) % 64
        if mapped_only:
            while e in UNMAPPED:
                e = (e + 1) % (70 if precise[r] else 64)
        v = {"lead": rng.randint(-2**20, 2**20), "e": e, "tail": None if r % 4 == 0 else letters(rng, rng.randint(0, 5)),
             "xs": [rng.randint(-99, 99) for _ in range(rng.randint(0, 2))]}
        kind = None
        if r in odd:
            kind = ("branch", "negblock")[r % 2]
            v["tail"] = v["tail"] or b"odd"
            v["xs"] = v["xs"] or [1, 2]
        recs.append(str_record(v, kind))
        vals.append(v)
    data, off = po.pack_records(recs)
    return recs, vals, data, off, odd


def enum_text(e):
    return W_SYMS[e] if e not in UNMAPPED else "Dq"


def check_enum_staging_reach(vals, k, odd):
    """Destinations of the enum text: every offset mod 4 for every length mod 4 in FAST warps, and words shared
    across lanes, warp edges and tile edges of 256- and 384-row tiles."""
    n = len(vals)
    precise = flavour_rows(np.arange(n + 1), k, lambda r: r in odd)
    seen, share = set(), {"warp": False, 256: False, 384: False, "three": False}
    for r0, r1 in po.chunk_bounds(n, po.clamp_chunks(k, n)):
        d, words = 0, {}
        for r in range(r0, r1):
            ln = len(enum_text(vals[r]["e"]).encode())
            if not precise[r]:
                seen.add((d & 3, ln & 3))
            for w in {d >> 2, (d + ln - 1) >> 2}:
                words.setdefault(w, set()).add(r - r0)
            d += ln
        for rows in words.values():
            share["three"] |= len(rows) >= 3
            for x in rows:
                if x + 1 in rows:
                    share["warp"] |= x % WARP == WARP - 1
                    share[256] |= x % 256 == 255
                    share[384] |= x % 384 == 383
    assert seen == {(a, b) for a in range(4) for b in range(4)}
    assert all(share.values()), share
    assert {vals[r]["e"] for r in range(n) if not precise[r]} >= set(range(64))        # every one-byte index FAST
    assert {vals[r]["e"] for r in range(n) if precise[r]} == set(range(70))


def str_expected(coracle, rj, vals, k):
    wv = [{"lead": v["lead"], "e": v["e"], "tail": (0, None) if v["tail"] is None else (1, v["tail"]), "xs": v["xs"]} for v in vals]
    return RS.expected_batches(coracle, STR_W, rj, wv, k)


def assert_str_batches(batches, want, rj):
    from tests.parity import expected_schema
    exp = expected_schema(rj)
    assert len(batches) == len(want)
    for i, (b, w) in enumerate(zip(batches, want)):
        assert b.schema.equals(exp, check_metadata=True), (b.schema, exp)
        b.validate(full=True)
        d = po.canon_diff(po.canon_from_batch(b), w, f"batch[{i}]")
        assert d is None, d


def first_unmapped(vals, rows_fast, rows_precise, which):
    """Records with unmapped symbols at the given rows (FAST: index 2, 5, 11, 40, 62 or 63; precise: 64, 66, 69),
    everything else mapped."""
    out = [dict(v) for v in vals]
    fast_syms, precise_syms = [2, 5, 11, 40, 62, 63], [64, 66, 69]
    for i, r in enumerate(rows_fast):
        out[r]["e"] = fast_syms[(i + which) % len(fast_syms)]
    for i, r in enumerate(rows_precise):
        out[r]["e"] = precise_syms[(i + which) % len(precise_syms)]
    return out


# (FAST rows, precise rows): the lowest failing record is a FAST lane, then a precise lane, of one warp; then in later
# warps, tiles and chunks
ENUM_ERRORS = [([70, 75], [66, 90]), ([40, 33], [39]), ([1700, 1900], [1701]), ([2599], [2598]), ([300, 1030], [2000])]


def enum_error_records(vals, case):
    fast, prec = ENUM_ERRORS[case]
    v = first_unmapped(vals, fast, prec, case)
    return [str_record(x) for x in v], min(fast + prec)


# schemas whose generated walkers tools/warm_jit_cache.py precompiles: (writer, reader)
JIT_RESOLVED = [(PROMO_W, PROMO_R), (STR_W, STR_RA), (STR_W, STR_RB), (STR_W, STR_RC), (STR_W, STR_RD)]


# ==== CPU ===========================================================================================================
def test_exact_reference_by_hand():
    assert X.int_to_f32_bits(2**24 + 1) == 0x4B800000
    assert X.int_to_f32_bits(2**24 + 3) == 0x4B800002
    assert X.int_to_f32_bits(2**60 + 2**36 + 1) == 0x5D800001      # a rounding through double would give 0x5D800000
    assert X.int_to_f32_bits(-2**63) == 0xDF000000 and X.int_to_f32_bits(2**63 - 1) == 0x5F000000
    assert X.int_to_f32_bits(-2**31) == 0xCF000000 and X.int_to_f32_bits(2**31 - 1) == 0x4F000000
    assert X.int_to_f64_bits(2**53 + 1) == 0x4340000000000000 and X.int_to_f64_bits(2**53 + 3) == 0x4340000000000002
    assert X.int_to_f64_bits(2**63 - 1) == 0x43E0000000000000 and X.int_to_f64_bits(-1) == 0xBFF0000000000000
    assert X.int_to_f64_bits(0) == 0 and X.int_to_f32_bits(0) == 0
    assert X.widen_f32_bits(0x00000001) == 0x36A0000000000000      # 2^-149
    assert X.widen_f32_bits(0x007FFFFF) == 0x380FFFFFC0000000
    assert X.widen_f32_bits(0x80000000) == 1 << 63
    assert X.widen_f32_bits(0x3F800000) == 0x3FF0000000000000
    assert X.widen_f32_bits(0xFF800000) == 0xFFF0000000000000
    assert X.widen_f32_bits(0x7F800001) == 0x7FF8000020000000      # signalling: quiet bit set, payload kept
    assert X.widen_f32_bits(0x7FC12345) == 0x7FF82468A0000000
    assert X.widen_f32_bits(0xFFC00001) == 0xFFF8000020000000
    assert X.decimal_text_to_f32_bits("1.00000005960464477540") == 0x3F800000   # one rounding: 0x3F800001
    assert X.decimal_text_to_f32_bits("1e-45") == 0x00000001 and X.decimal_text_to_f32_bits("1e-46") == 0
    assert X.decimal_text_to_f32_bits("3.4028235e38") == 0x7F7FFFFF and X.decimal_text_to_f32_bits("3.5e38") == 0x7F800000
    assert X.decimal_text_to_f32_bits("-1e39") == 0xFF800000 and X.decimal_text_to_f32_bits("-0.0") == 0x80000000
    assert X.decimal_text_to_f32_bits("0.1") == 0x3DCCCCCD
    assert X.decimal_text_to_f64_bits("5e-324") == 1 and X.decimal_text_to_f64_bits("1e-400") == 0
    assert X.decimal_text_to_f64_bits("0.1") == 0x3FB999999999999A
    assert X.decimal_text_to_f64_bits("1.7976931348623157e308") == 0x7FEFFFFFFFFFFFFF
    assert X.decimal_text_to_f64_bits("1e400") == 0x7FF0000000000000
    assert X.int32_of_varint(zz(2**31)) == -2**31 and X.int32_of_varint(zz(-2**31 - 1)) == 2**31 - 1
    assert X.int32_of_varint((1 << 64) - 1) == 0 and X.int32_of_varint(1 << 65) == 0


@pytest.mark.parametrize("k", [1, 3])
def test_emu_promotions_and_defaults(coracle, k):
    recs, vals, data, off, odd = promo_case(k)
    check_promo_reach(recs, data, off, k)
    for w in ("interp", "gen"):
        assert_promo_batches(R.decode(PROMO_W, PROMO_R, data, off, len(recs), k, walker=w), vals, k, coracle)


@pytest.mark.parametrize("k", [1, 3])
def test_emu_default_strings_and_enum_text(coracle, k):
    recs, vals, data, off, odd = str_case(k)
    check_enum_staging_reach(vals, k, odd)
    assert_tiles_fit(off, k)
    for rj in (STR_RA, STR_RB, STR_RC):
        want = str_expected(coracle, rj, vals, k)
        for w in ("interp", "gen"):
            assert_str_batches(R.decode(STR_W, rj, data, off, len(recs), k, walker=w), want, rj)


def test_emu_enum_remap_without_default(coracle):
    recs, vals, data, off, odd = str_case(1, mapped_only=True)
    assert {v["e"] - 1 for v in vals} & UNMAPPED and 0 in {v["e"] for v in vals}   # mapped symbols next to unmapped ones
    for k in (1, 3):
        want = str_expected(coracle, STR_RD, vals, k)
        for w in ("interp", "gen"):
            assert_str_batches(R.decode(STR_W, STR_RD, data, off, len(recs), k, walker=w), want, STR_RD)
    for case in range(len(ENUM_ERRORS)):
        bad, first = enum_error_records(vals, case)
        d2, o2 = po.pack_records(bad)
        for k in (1, 3, 8):
            for w in ("interp", "gen"):
                with pytest.raises(emu.EmuError) as ei:
                    R.decode(STR_W, STR_RD, d2, o2, len(bad), k, walker=w)
                assert (ei.value.code, ei.value.record) == (6, first), (case, k, w, str(ei.value))


def test_out_of_range_number_defaults_are_refused():
    w = json.dumps(rec(fld("a", "int")))
    for t, text in (("double", "1e400"), ("double", "-1e400"), ("float", "1e400"), ("float", "2e308")):
        rj = with_raw_defaults(rec(fld("a", "int"), fld("b", t, default="@@0@@")), [text])
        with pytest.raises(ValueError, match="schema resolution") as ei:
            pr.Schema(w).read_as(rj)
        assert "field 'b'" in str(ei.value) and "does not match" in str(ei.value)
    for t, text in (("double", "1e-400"), ("float", "3.5e38"), ("double", "1.7976931348623157e308")):   # underflow and float overflow are values
        pr.Schema(w).read_as(with_raw_defaults(rec(fld("a", "int"), fld("b", t, default="@@0@@")), [text]))


# ==== GPU ===========================================================================================================
class _GpuError(Exception):
    def __init__(self, status, message):
        super().__init__(message)
        import re
        m = re.search(r"\(record (-?\d+)\)", message)
        self.status, self.record = status, int(m.group(1)) if m else -1


def gpu_decode(wj, rj, data, off, n, k):
    """rv_decode_host twice (the first call teaches the handle the tiles' sizes); (batches, slow tiles, tile rows)."""
    s = pr.Schema(wj).read_as(rj)
    data = np.ascontiguousarray(data, dtype=np.uint8)
    off = np.ascontiguousarray(off, dtype=np.int64)
    for _ in range(2):
        h = ctypes.c_void_p()
        rc = pr.lib.rv_decode_host(s.handle, data.ctypes.data, off.ctypes.data, n, k, ctypes.byref(h))
        if rc:
            raise _GpuError(rc, pr._last_error())
        got = pr._export_batches(h.value, s)
    return got, pr.lib.rv_last_slow_tiles(), pr.lib.rv_last_tile()


@pytest.fixture(params=["jit", "interp"])
def walker(request):
    pr.set_jit_enabled(1 if request.param == "jit" else 0)
    yield request.param
    pr.set_jit_enabled(-1)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3])
def test_gpu_promotions_and_defaults(coracle, walker, k):
    recs, vals, data, off, odd = promo_case(k)
    got, slow, _ = gpu_decode(PROMO_W, PROMO_R, data, off, len(recs), k)
    assert pr.last_walker() == walker
    assert slow == 0
    assert_promo_batches(got, vals, k, coracle)


@pytest.mark.gpu
@pytest.mark.parametrize("k", [1, 3])
def test_gpu_default_strings_and_enum_text(coracle, walker, k):
    recs, vals, data, off, odd = str_case(k)
    for rj, tile in ((STR_RA, 384 if walker == "jit" else 256), (STR_RB, 256), (STR_RC, 256)):
        got, slow, t = gpu_decode(STR_W, rj, data, off, len(recs), k)
        assert pr.last_walker() == walker and t == tile, (t, tile)
        assert (slow > 0) == (rj == STR_RC), slow
        assert_str_batches(got, str_expected(coracle, rj, vals, k), rj)


@pytest.mark.gpu
def test_gpu_enum_remap_without_default(coracle, walker):
    recs, vals, data, off, odd = str_case(1, mapped_only=True)
    for k in (1, 3):
        got, slow, _ = gpu_decode(STR_W, STR_RD, data, off, len(recs), k)
        assert slow == 0
        assert_str_batches(got, str_expected(coracle, STR_RD, vals, k), STR_RD)
    for case in range(len(ENUM_ERRORS)):
        bad, first = enum_error_records(vals, case)
        d2, o2 = po.pack_records(bad)
        for k in (1, 3, 8):
            with pytest.raises(_GpuError) as ei:
                gpu_decode(STR_W, STR_RD, d2, o2, len(bad), k)
            assert (ei.value.status, ei.value.record) == (6, first), (case, k, str(ei.value))
            assert "neither a reader symbol nor a reader default" in str(ei.value)
