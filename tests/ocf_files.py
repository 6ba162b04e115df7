"""Avro object container files for the tests: a header, then blocks of datums between sync markers (the specification's
"Object Container Files" section).  The layouts, header forms and markers are the writer's choice, so the reader under
test sees what other writers produce: blocks of any size including empty ones, metadata maps in several blocks, extra
or repeated keys, no codec key, a marker whose bytes also occur in the datums."""
import random

from oracle import pyoracle as po
from tests import mutation as M
from tests.parity import gen_case


def zz(v: int) -> bytes:
    return po.zigzag_bytes(v)


def ocf_header(schema_json: str, sync: bytes, meta_extra=None, codec=b"null", meta_blocks: int = 1) -> bytes:
    """Magic, metadata and sync marker.  meta_extra: a dict updates avro.schema / avro.codec in place and adds keys after
    them; a list of (key, value) pairs is written before them (a repeated key: the later one, avro.schema's own, wins).
    codec=None leaves the key out.  meta_blocks > 1 splits the entries over that many map blocks, each written in the
    negative-count form (-count, byte size)."""
    pairs = [("avro.schema", schema_json.encode())] + ([("avro.codec", codec)] if codec is not None else [])
    if isinstance(meta_extra, dict):
        d = dict(pairs)
        d.update(meta_extra)
        pairs = list(d.items())
    elif meta_extra:
        pairs = list(meta_extra) + pairs
    out = bytearray(po.OCF_MAGIC)
    if meta_blocks <= 1:
        out += zz(len(pairs))
        for k, v in pairs:
            out += zz(len(k)) + k.encode() + zz(len(v)) + v
    else:
        step = -(-len(pairs) // meta_blocks)
        for i in range(0, len(pairs), step):
            body = b"".join(zz(len(k)) + k.encode() + zz(len(v)) + v for k, v in pairs[i:i + step])
            out += zz(-len(pairs[i:i + step])) + zz(len(body)) + body
    out += zz(0) + sync
    return bytes(out)


def ocf_block(count: int, body: bytes, sync: bytes) -> bytes:
    return zz(count) + zz(len(body)) + body + sync


def ocf_file(schema_json, recs, block_records=(1,), rng=None, meta_extra=None, *, counts=None, codec=b"null",
             meta_blocks: int = 1, sync=None) -> bytes:
    """A container of `recs`.  Block sizes: `counts` (records per block in order, 0 for an empty block; they add up to
    len(recs)), else rng.choice(block_records) records per block (the last one takes what is left).  sync: the 16-byte
    marker, else 16 random bytes from rng.  No records and no counts: a file that ends right after its header."""
    if sync is None:
        sync = bytes(rng.randrange(256) for _ in range(16))
    assert len(sync) == 16
    out = bytearray(ocf_header(schema_json, sync, meta_extra, codec, meta_blocks))
    if counts is None:
        counts, i = [], 0
        while i < len(recs):
            counts.append(min(len(recs) - i, rng.choice(block_records)))
            i += counts[-1]
    assert sum(counts) == len(recs), (sum(counts), len(recs))
    i = 0
    for n in counts:
        out += ocf_block(n, b"".join(recs[i:i + n]), sync)
        i += n
    return bytes(out)


def counts_with_edges(n: int, k: int, edges=(255, 256, 257, 383, 384, 385)):
    """Records per block such that blocks end right at `edges` records into every chunk of n records split k ways."""
    cuts = set()
    for j in range(k):
        c0 = j * (n // k)
        cuts.update(c0 + e for e in edges if c0 + e < n)
        cuts.add(c0)
    cuts = sorted(cuts | {n})      # (chunk 0 starts at record 0)
    return [b - a for a, b in zip(cuts, cuts[1:])]


def with_empty_blocks(counts, rng):
    """The same blocks with empty blocks in between."""
    out = []
    for c in counts:
        out += [0] * rng.choice([0, 0, 1, 2]) + [c]
    return out + [0]


def split(recs, counts):
    out, i = [], 0
    for n in counts:
        out.append(list(recs[i:i + n]))
        i += n
    return out


def from_blocks(schema_json, blocks, sync, bodies=None, counts=None) -> bytes:
    """A file of the given blocks of datums; `bodies` / `counts` override a block's bytes / claimed count by index."""
    out = bytearray(ocf_header(schema_json, sync))
    for i, b in enumerate(blocks):
        body = (bodies or {}).get(i, b"".join(b))
        out += ocf_block((counts or {}).get(i, len(b)), body, sync)
    return bytes(out)


def damaged_file(seed: int, schema_seed=None):
    """A container of a random schema's datums with damage inside its blocks: datums hit by tests/mutation.damage, one
    damaged datum in each of two blocks, or a block header that disagrees with its datums (count +-1, junk bytes before the
    sync marker that the size covers, a datum cut short).  Returns (file, k)."""
    rng = random.Random(seed * 613 + 7)
    sj, recs, _, _ = gen_case(seed % 300 if schema_seed is None else schema_seed, n=rng.choice([3, 40, 257, 300]))
    n = len(recs)
    counts, left = [], n
    while left:
        counts.append(min(left, rng.choice([1, 2, 7, 50, 256, 300])))
        left -= counts[-1]
    sync = bytes(rng.randrange(256) for _ in range(16))
    op = rng.choice(["datums", "datums", "datums", "two", "count+1", "count-1", "junk", "cut"])
    blocks = split(recs, counts)
    bodies, forged = {}, {}
    if op == "datums":
        blocks = split(M.damage(rng, recs), counts)
    elif op == "two" and len(blocks) > 1:
        for i in rng.sample(range(len(blocks)), 2):
            j = rng.randrange(len(blocks[i]))
            blocks[i][j] = M.damage(rng, [blocks[i][j]])[0]
    else:
        i = rng.randrange(len(blocks))
        if op == "count+1":
            forged[i] = len(blocks[i]) + 1
        elif op == "count-1":
            forged[i] = len(blocks[i]) - 1
        elif op == "junk":
            bodies[i] = b"".join(blocks[i]) + bytes(rng.randrange(256) for _ in range(rng.randrange(1, 9)))
        else:
            j = rng.randrange(len(blocks[i]))
            blocks[i][j] = blocks[i][j][:rng.randrange(len(blocks[i][j]) + 1)]
    return from_blocks(sj, blocks, sync, bodies, forged), rng.choice([1, 2, 3, 8])


def expected(coracle, f: bytes, k: int, wide: bool = False):
    """The reader's verdict on a container: "container", (error category, record), or the canonical batches at k chunks
    (the C oracle, or the Python decoder for the wider subset), with the datums the reader found."""
    try:
        sj, datums, _ = po.ocf_read(f, wide=wide)
    except po.ContainerError:
        return "container", None
    except po.DecodeError as e:
        return (e.code, e.record), None
    try:
        if wide:
            s = po.parse_schema(sj, wide=True)
            bounds = po.chunk_bounds(len(datums), po.clamp_chunks(k, len(datums)))
            return [po.py_decode(s, datums[a:b]) for a, b in bounds], datums
        data, off = po.pack_records(datums)
        return coracle.decode_threaded_packed(sj, data, off, len(datums), k, threads=4), datums
    except po.DecodeError as e:
        return (e.code, e.record), datums


def check(coracle, decode, error_of, f: bytes, k: int, wide: bool = False):
    """`decode(f, k)` -> batches or raises; `error_of(exc)` -> "container", (category, record), or None for an exception
    that is not a verdict of the decoder under test.  Returns the verdict kind: "decoded", "error" or "container"."""
    want, _ = expected(coracle, f, k, wide)
    try:
        got = decode(f, k)
    except Exception as e:  # noqa: BLE001 - classified right below
        g = error_of(e)
        if g is None:
            raise
        assert not isinstance(want, list), f"decoder reports {g}, the reader decodes this file"
        assert g == want, f"decoder reports {g}, the reader {want}"
        return "container" if g == "container" else "error"
    assert isinstance(want, list), f"decoder accepted a file the reader rejects with {want}"
    assert len(got) == len(want), (len(got), len(want))
    for i, (b, w) in enumerate(zip(got, want)):
        d = po.canon_diff(po.canon_from_batch(b), w, f"batch[{i}]")
        assert d is None, d
    return "decoded"


def block_spans(f: bytes):
    """(offset of the count varint, offset of the datums, byte size, count) of every block of a well-formed file."""
    c = po._Cur(f)
    c.p = 4
    while True:
        n = c.zigzag()
        if n == 0:
            break
        if n < 0:
            c.zigzag()
            n = -n
        for _ in range(n):
            c.take(c.zigzag())
            c.take(c.zigzag())
    c.p += 16
    out = []
    while c.p < len(f):
        head = c.p
        count, size = c.zigzag(), c.zigzag()
        out.append((head, c.p, size, count))
        c.p += size + 16
    return out
