"""Rebuild Arrow arrays of the direct-encode subset with a different physical layout and the same logical values.

Batches this library decodes always have one layout: offsets 0, list offsets from 0, nothing under null slots, union
type codes 0..N-1.  Batches built by pyarrow, Polars or a Rust producer need not.  `relayout(array, rng, ...)` rebuilds
an array with `pa.Array.from_buffers`, choosing per array (at every level) among the variations below, so that a test
can name which ones it exercises:

  offset         a non-zero offset on every array, so bitmaps start at bit offsets 1-7
  list_junk      list / map / string offsets that do not start at 0, with junk items before and after the rows' range
                 (map entries and struct children get offsets of their own as a consequence)
  validity       an all-valid bitmap where there are no nulls, or no bitmap at all
  null_junk      junk values under the null slots of nullable fields
  null_ranges    null slots of nullable lists and maps that cover a non-empty range of items
  union_codes    sparse unions whose children are permuted, with type codes permuted to match
  unaligned      buffers whose start address is 1-7 bytes past an 8-byte boundary (a sliced py_buffer)
  shared         top-level columns of equal type become two slices of one array (same buffers, different offsets)
  nonnull_junk   null slots with junk values in NON-nullable leaf fields

Every variation but `nonnull_junk` keeps the values of non-nullable fields' slots as they were, null or not: the
encoder writes those raw values (fast_encode.rs:401-409), so the encoded datums do not change.  `nonnull_junk` changes
them on purpose; its output is compared with the encode oracle only.
"""
import numpy as np
import pyarrow as pa

VARIATIONS = ("offset", "list_junk", "validity", "null_junk", "null_ranges", "union_codes", "unaligned", "shared",
              "nonnull_junk")
KEEPS_DATUMS = tuple(v for v in VARIATIONS if v != "nonnull_junk")


def _bits(buf, off, n):
    if buf is None:
        return np.ones(n, dtype=bool)
    return np.unpackbits(np.frombuffer(buf, dtype=np.uint8), bitorder="little")[off:off + n].astype(bool)


def _nulls(valid, o):  # an explicit null count: a map's entries must be KNOWN to have none
    return int((~valid[o:]).sum())


class _Relayout:
    def __init__(self, rng, variations):
        unknown = set(variations) - set(VARIATIONS)
        assert not unknown, unknown
        self.rng, self.v = rng, frozenset(variations)

    def _buf(self, data: bytes) -> pa.Buffer:
        if "unaligned" in self.v:
            sh = self.rng.randint(1, 7)
            return pa.py_buffer(bytes(8 + sh) + data)[8 + sh:]  # py_buffer data is at least 8-aligned
        return pa.py_buffer(data)

    def _text(self, n) -> bytes:  # junk that is still valid UTF-8: validate(full=True) checks every slot
        return bytes(self.rng.choice(b"#%&?@~qxz") for _ in range(n))

    def _bitmap(self, bits) -> pa.Buffer:
        return self._buf(np.packbits(np.asarray(bits, dtype=bool), bitorder="little").tobytes() + b"\0")

    def _own_offset(self):
        return self.rng.randint(1, 9) if "offset" in self.v else 0

    def _junk_run(self):
        return self.rng.randint(1, 5) if "list_junk" in self.v else 0

    def _validity(self, a, idx, nullable, o):
        """Bitmap buffer (or None) for slots idx (-1 = junk) behind o junk slots, and the per-slot validity."""
        had_nulls = a.null_count > 0
        old = _bits(a.buffers()[0] if had_nulls else None, a.offset, len(a))  # a bitmap with null_count 0 is not read
        valid = np.ones(o + len(idx), dtype=bool)
        for s, i in enumerate(idx):
            if i >= 0:
                valid[o + s] = old[i]
            elif nullable and had_nulls:
                valid[o + s] = self.rng.random() < 0.5
        if nullable and had_nulls:
            valid[:o] = [self.rng.random() < 0.5 for _ in range(o)]
        if valid.all():                              # no nulls: a bitmap as before, or (`validity`) either way
            drop = self.rng.random() < 0.5 if "validity" in self.v else a.buffers()[0] is None
            if drop:
                return None, valid
        return self._bitmap(valid), valid

    def _nonnull_junk(self, a, nullable, idx):
        """`nonnull_junk`: slots of a non-nullable leaf that become null (their values are then junk)."""
        if "nonnull_junk" not in self.v or nullable is not False:  # None: a map key, which may never be null
            return set()
        return {s for s, i in enumerate(idx) if i >= 0 and self.rng.random() < 0.25}

    # ------------------------------------------------------------------------------------------------
    def build(self, a: pa.Array, nullable: bool, idx):
        """A new array of len(idx) slots: slot s holds a's logical slot idx[s] (raw value, null or not), or junk for -1."""
        t = a.type
        o = self._own_offset()
        rng = self.rng
        if pa.types.is_null(t):
            return pa.nulls(len(idx))
        if pa.types.is_struct(t):
            vbuf, valid = self._validity(a, idx, nullable, o)
            cidx = [-1] * o + list(idx) + [-1] * rng.randint(0, 2)
            kids = [self.build(a.field(j), None if nullable is None and j == 0 else t.field(j).nullable, cidx)
                    for j in range(t.num_fields)]
            st = pa.struct([pa.field(f.name, k.type, f.nullable) for f, k in zip(t, kids)])  # unions below may be new
            return pa.Array.from_buffers(st, len(idx), [vbuf], _nulls(valid, o), o, kids)
        if pa.types.is_union(t):
            assert t.mode == "sparse", t
            n = len(a)
            tids = np.frombuffer(a.buffers()[1], dtype=np.int8)[a.offset:a.offset + n]
            codes = list(t.type_codes)
            new = np.array([tids[i] if i >= 0 else rng.choice(codes) for i in [-1] * o + list(idx)], dtype=np.int8)
            order = list(range(t.num_fields))
            if "union_codes" in self.v:
                rng.shuffle(order)
            cidx = [-1] * o + list(idx) + [-1] * rng.randint(0, 2)
            kids = [self.build(a.field(p), True, cidx) for p in order]
            ut = pa.sparse_union([pa.field(t.field(p).name, k.type, t.field(p).nullable) for p, k in zip(order, kids)],
                                 [codes[p] for p in order])
            return pa.Array.from_buffers(ut, len(idx), [None, self._buf(new.tobytes())], offset=o, children=kids)
        if pa.types.is_list(t) or pa.types.is_map(t):
            vbuf, valid = self._validity(a, idx, nullable, o)
            offs = np.frombuffer(a.buffers()[1], dtype=np.int32)[a.offset:a.offset + len(a) + 1]
            child = a.values                        # raw child: the offsets index it logically
            nchild = len(child)
            cidx = [-1] * self._junk_run()
            new_offs = [len(cidx)] * (o + 1)
            for s, i in enumerate(idx):
                if i >= 0 and valid[o + s]:
                    cidx += range(int(offs[i]), int(offs[i + 1]))
                elif i >= 0 and not nullable:       # a null slot of a non-nullable list keeps its items
                    cidx += range(int(offs[i]), int(offs[i + 1]))
                elif i >= 0 and "null_ranges" not in self.v:
                    cidx += range(int(offs[i]), int(offs[i + 1]))
                elif nchild:                         # junk slot, or a null slot covering junk items
                    cidx += [rng.randrange(nchild) for _ in range(rng.randint(0, 3) if i < 0 else rng.randint(1, 3))]
                new_offs.append(len(cidx))
            cidx += [-1] * self._junk_run()
            if pa.types.is_map(t):                  # the entries struct and its key field are never null
                kid = self.build(child, None, cidx)
                t = pa.map_(t.key_field, pa.field(t.item_field.name, kid.type.field(1).type, t.item_field.nullable))
            else:
                kid = self.build(child, t.value_field.nullable, cidx)
                t = pa.list_(pa.field(t.value_field.name, kid.type, t.value_field.nullable))
            ob = self._buf(np.array(new_offs, dtype=np.int32).tobytes())
            return pa.Array.from_buffers(t, len(idx), [vbuf, ob], _nulls(valid, o), o, [kid])
        # leaves
        vbuf, valid = self._validity(a, idx, nullable, o)
        junk_null = self._nonnull_junk(a, nullable, idx)
        if junk_null:
            valid[[o + s for s in junk_null]] = False
            vbuf = self._bitmap(valid)

        def is_junk(s, i):
            return i < 0 or s in junk_null or ("null_junk" in self.v and nullable and not valid[o + s])
        slots = [-1] * o + list(idx)
        sidx = [-1] * o + [(-1 if is_junk(s, i) else i) for s, i in enumerate(idx)]
        if pa.types.is_boolean(t):
            old = _bits(a.buffers()[1], a.offset, len(a))
            bits = [old[i] if i >= 0 else rng.random() < 0.5 for i in sidx]
            return pa.Array.from_buffers(t, len(idx), [vbuf, self._bitmap(bits)], _nulls(valid, o), o)
        if pa.types.is_string(t):
            offs = np.frombuffer(a.buffers()[1], dtype=np.int32)[a.offset:a.offset + len(a) + 1]
            data = a.buffers()[2]
            raw = bytes(memoryview(data)) if data is not None else b""
            real = [raw[offs[i]:offs[i + 1]] for i in range(len(a))]
            body = bytearray(self._text(self._junk_run()))
            new_offs = [len(body)]
            for s, i in enumerate(sidx):
                if i >= 0:
                    body += real[i]
                elif real and slots[s] >= 0:          # junk under a null slot: another slot's text (enum columns stay enums)
                    body += rng.choice(real)
                else:
                    body += self._text(rng.randint(0, 6))
                new_offs.append(len(body))
            body += self._text(self._junk_run())
            return pa.Array.from_buffers(t, len(idx), [vbuf, self._buf(np.array(new_offs, dtype=np.int32).tobytes()),
                                                      self._buf(bytes(body))], _nulls(valid, o), o)
        width = t.bit_width // 8
        old = np.frombuffer(a.buffers()[1], dtype=np.uint8)[width * a.offset:width * (a.offset + len(a))].reshape(-1, width)
        vals = np.frombuffer(rng.randbytes(width * len(sidx)), dtype=np.uint8).reshape(-1, width).copy()
        real = np.array([i >= 0 for i in sidx], dtype=bool)
        if real.any():
            vals[real] = old[np.array([i for i in sidx if i >= 0])]
        return pa.Array.from_buffers(t, len(idx), [vbuf, self._buf(vals.tobytes())], _nulls(valid, o), o)


def relayout(array: pa.Array, rng, variations=KEEPS_DATUMS, nullable: bool = True) -> pa.Array:
    """`array` with the same logical values (raw values under null slots of non-nullable fields kept) laid out anew."""
    r = _Relayout(rng, variations)
    pre = r._own_offset()
    out = r.build(array, nullable, [-1] * pre + list(range(len(array))) + [-1] * rng.randint(0, 3))
    return out.slice(pre, len(array))


def relayout_batch(batch: pa.RecordBatch, rng, variations=KEEPS_DATUMS) -> pa.RecordBatch:
    """Every column relaid; with `shared`, pairs of columns of equal type become two slices of one array."""
    cols = [relayout(c, rng, variations, f.nullable) for c, f in zip(batch.columns, batch.schema)]
    if "shared" in variations:
        r = _Relayout(rng, variations)
        seen = {}
        for j, f in enumerate(batch.schema):
            if f.type in seen:
                i = seen.pop(f.type)
                n = batch.num_rows
                pair = pa.concat_arrays([batch.column(i), batch.column(j)])
                both = r.build(pair, f.nullable, list(range(2 * n)))
                cols[i], cols[j] = both.slice(0, n), both.slice(n, n)
            else:
                seen[f.type] = j
    fields = [pa.field(f.name, c.type, f.nullable) for c, f in zip(cols, batch.schema)]  # unions may have new codes
    return pa.RecordBatch.from_arrays(cols, schema=pa.schema(fields))
