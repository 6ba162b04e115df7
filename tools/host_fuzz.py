#!/usr/bin/env python
"""Host-side robustness fuzz (no GPU needed): damaged schema documents through the product's schema front-end and damaged
Avro Object Container Files through the container reader.  Every outcome must be a clean Python exception (ValueError) or a
success — never a crash, a hang or another exception type.  For schema documents that all three parsers accept the
product's Arrow schema must equal the pure-Python oracle's (tests use the same comparison on undamaged random schemas).

    python tools/host_fuzz.py FIRST_SEED N [schema | schema-tree | ocf | both]

Without a CUDA device a container that survives the reader ends in "no CUDA device" (RV_ERR_CUDA -> ValueError): the
container layer has then accepted the file, which is what this tool exercises."""
import os
import random
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

JSON_BITS = [b'"', b"{", b"}", b"[", b"]", b":", b",", b"null", b'"type"', b'"name"', b'"fields"', b'"items"', b'"values"', b'"symbols"',
             b'"size"', b'"logicalType"', b'"precision"', b'"scale"', b"0", b"-1", b"1e99", b"99999999999999999999", b'"\\u0000"',
             b'"record"', b'"array"', b'"map"', b'"fixed"', b'"enum"', b'"decimal"', b'"uuid"', b"\\", b"\xff", b"\x00", b" "]


def damage_text(rng, raw: bytes) -> bytes:
    b = bytearray(raw)
    for _ in range(rng.choice([1, 1, 2, 3, 6])):
        op = rng.randrange(6)
        j = rng.randrange(len(b) + 1)
        if op == 0 and b:
            b[min(j, len(b) - 1)] = rng.randrange(256)
        elif op == 1:
            b[j:j] = rng.choice(JSON_BITS)
        elif op == 2 and b:
            del b[j:j + rng.randrange(1, 12)]
        elif op == 3 and b:
            del b[j:]
        elif op == 4 and b:   # duplicate a slice somewhere else
            a = rng.randrange(len(b))
            piece = bytes(b[a:a + rng.randrange(1, 40)])
            b[j:j] = piece
        else:                 # swap two tokens' worth of bytes
            k = rng.randrange(len(b) + 1)
            b[j:j + 4], b[k:k + 4] = b[k:k + 4], b[j:j + 4]
    return bytes(b)


def fuzz_schema(first, count):
    import pyruhvro_b200 as pr
    from oracle import pyoracle as po
    ok = bad = same = 0
    for seed in range(first, first + count):
        rng = random.Random(seed * 31 + 7)
        sj = po.random_schema_json(random.Random(seed), wide=bool(seed & 1))
        doc = damage_text(rng, sj.encode())
        try:
            text = doc.decode("utf-8")
        except UnicodeDecodeError:
            text = doc.decode("latin-1")
        try:
            s = pr.Schema(text)
            supported = s.is_supported
            ok += 1
        except ValueError:
            bad += 1
            continue
        if supported:   # the product accepts and can decode it: the independent parser must translate it the same way
            try:
                from tests.parity import expected_schema_wide   # (through the C Data Interface, like the product's)
                want = expected_schema_wide(text)
            except Exception:  # noqa: BLE001 - the Python restatement is stricter / looser on damaged documents: not a product bug
                continue
            if s.arrow_schema.equals(want, check_metadata=True):
                same += 1
            else:
                print(f"DIFF seed={seed}: {text[:300]}", flush=True)
    return f"schema documents: {ok} parsed ({same} supported and equal to the Python oracle's translation), {bad} rejected cleanly"


TREE_VALUES = [None, True, False, 0, 1, -1, 16, 38, 39, 2**31, 1.5, "", "null", "int", "long", "string", "bytes", "record", "array", "map", "enum",
               "fixed", "decimal", "uuid", "date", "time-millis", "timestamp-micros", "Top", "R2", "a.b", "9x", "x y", [], {}, ["null"], ["null", "null"],
               ["int", "int"], {"type": "int"}, {"type": "array", "items": "int"}, ["null", ["int"]]]
TREE_KEYS = ["type", "name", "namespace", "fields", "items", "values", "symbols", "size", "logicalType", "precision", "scale", "doc", "aliases",
             "default", "order"]


def mutate_tree(rng, doc):
    """Mutations of the parsed document (always valid JSON): values replaced / dropped / added, list items removed,
    inserted or duplicated, names bent, subtrees copied over other subtrees."""
    import json

    def nodes(x, acc, path=()):
        acc.append((path, x))
        if isinstance(x, dict):
            for k, v in x.items():
                nodes(v, acc, path + (k,))
        elif isinstance(x, list):
            for i, v in enumerate(x):
                nodes(v, acc, path + (i,))

    def parent(path):
        x = doc
        for q in path[:-1]:
            x = x[q]
        return x

    def fresh(v):   # (never a shared object: later mutations write into what they find)
        return json.loads(json.dumps(v))
    for _ in range(rng.choice([1, 1, 2, 3])):
        acc = []
        nodes(doc, acc)
        path, x = rng.choice(acc)
        op = rng.randrange(7)
        if op == 0 and path:
            parent(path)[path[-1]] = fresh(rng.choice(TREE_VALUES))
        elif op == 1 and isinstance(x, dict) and x:
            del x[rng.choice(list(x))]
        elif op == 2 and isinstance(x, dict):
            x[rng.choice(TREE_KEYS)] = fresh(rng.choice(TREE_VALUES))
        elif op == 3 and isinstance(x, list) and x:
            if rng.random() < 0.5:
                del x[rng.randrange(len(x))]
            else:
                x.insert(rng.randrange(len(x) + 1), fresh(rng.choice(TREE_VALUES)))
        elif op == 4 and isinstance(x, list) and len(x) > 1:
            x.append(fresh(x[rng.randrange(len(x))]))
        elif op == 5 and isinstance(x, str) and path:
            parent(path)[path[-1]] = rng.choice([x + "x", x[:-1], x.upper(), "." + x, x + ".", "ns." + x])
        elif op == 6 and path:
            parent(path)[path[-1]] = fresh(rng.choice(acc)[1])
    return doc


def fuzz_schema_tree(first, count):
    """The product's front-end against the pure-Python restatement on mutated (still well-formed) documents.  The
    restatement is lenient where the library validates (names, symbols, duplicates, missing attributes), so only three
    outcomes are reported: the product accepts what the restatement cannot parse, the gates disagree, the translations differ."""
    import collections
    import json
    import pyruhvro_b200 as pr
    from oracle import pyoracle as po
    from tests.parity import expected_schema_wide
    stat = collections.Counter()
    for seed in range(first, first + count):
        rng = random.Random(seed * 17 + 1)
        doc = json.loads(po.random_schema_json(random.Random(seed), wide=bool(seed & 1)))
        try:
            text = json.dumps(mutate_tree(rng, doc))
        except (TypeError, ValueError, KeyError, IndexError):
            continue
        try:
            s = pr.Schema(text)
        except ValueError:
            stat["rejected by the product"] += 1
            continue
        try:
            o = po.parse_schema(text, wide=True)
        except Exception as e:  # noqa: BLE001
            stat["accepted by the product, not parsed by the restatement"] += 1
            print(f"ACCEPT seed={seed}: {e!r}"[:160], flush=True)
            continue
        if s.is_supported != po.is_supported(o):
            stat["gates differ (documented limits: nesting depth, 0-field records, ...)"] += 1
            continue
        if not s.is_supported:
            stat["outside the subset for both"] += 1
            continue
        try:
            want = expected_schema_wide(text)
        except Exception:  # noqa: BLE001 - pyarrow refuses what the restatement built (a non-nullable null field, a non-string doc)
            stat["restatement could not build the Arrow schema"] += 1
            continue
        if s.arrow_schema.equals(want, check_metadata=True):
            stat["equal translations"] += 1
        else:
            stat["DIFFERENT translations"] += 1
            print(f"DIFF seed={seed}: {text[:300]}", flush=True)
    return "mutated schema trees: " + ", ".join(f"{v} {k}" for k, v in sorted(stat.items()))


def fuzz_ocf(first, count):
    import pyruhvro_b200 as pr
    from oracle import pyoracle as po
    from tests.parity import gen_case
    from tests.ocf_files import ocf_file
    kinds = {}
    for seed in range(first, first + count):
        rng = random.Random(seed * 131 + 3)
        sj, recs, _, _ = gen_case(seed % 500, n=rng.choice([0, 1, 5, 40]))
        f = bytearray(ocf_file(sj, recs, [1, 3, 50], rng))
        for _ in range(rng.choice([1, 1, 2, 4])):
            op = rng.randrange(5)
            j = rng.randrange(len(f) + 1)
            if op == 0 and f:
                f[min(j, len(f) - 1)] = rng.randrange(256)
            elif op == 1:
                f[j:j] = rng.choice([b"\xff" * rng.randrange(1, 12), po.zigzag_bytes(rng.choice([-1, 2**31, 2**62, -2**63, 2**63 - 1])),
                                     bytes(rng.randrange(256) for _ in range(rng.randrange(1, 6)))])
            elif op == 2 and f:
                del f[j:]
            elif op == 3 and f:
                del f[j:j + rng.randrange(1, 20)]
            else:
                f.extend(bytes(rng.randrange(256) for _ in range(rng.randrange(1, 30))))
        try:
            pr.deserialize_ocf(bytes(f), rng.choice([1, 2, 8]))
            kind = "decoded"
        except ValueError as e:
            m = str(e)
            kind = "reached the decoder (no CUDA device here)" if ("CUDA" in m or "cuda" in m) else "rejected by the container reader / schema"
        kinds[kind] = kinds.get(kind, 0) + 1
    return "container files: " + ", ".join(f"{v} {k}" for k, v in sorted(kinds.items()))


if __name__ == "__main__":
    first, count = int(sys.argv[1]), int(sys.argv[2])
    what = sys.argv[3] if len(sys.argv) > 3 else "both"
    t0 = time.time()
    if what in ("schema", "both"):
        print(fuzz_schema(first, count), flush=True)
    if what == "schema-tree":
        print(fuzz_schema_tree(first, count), flush=True)
    if what in ("ocf", "both"):
        print(fuzz_ocf(first, count), flush=True)
    print(f"{int(time.time() - t0)} s, no crash")
