#!/usr/bin/env python
"""One-off GPU fuzz campaign: many random schemas x random data, both walkers, buffer-exact vs the C oracle,
plus encode round trips.  usage: fuzz_gpu.py [--warm] FIRST_SEED N_INTERP N_JIT
    fuzz_gpu.py --wide FIRST_SEED N   random schemas over the WIDER subset (bytes, fixed, uuid, decimal, time-*, named
                                      references) against the pure-Python oracle; every 16th case through a generated walker"""
import os
import random
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def schema_for(seed):
    from oracle import pyoracle as po
    return po.random_schema_json(random.Random(seed), max_depth=random.Random(seed * 7 + 1).choice([2, 3, 3, 4]))


def warm(seed):
    import pyruhvro_b200 as pr
    s = pr.Schema(schema_for(seed))
    if s.is_supported:
        s.precompile("sm_90a")
    return 1


def main_wide(first, n_cases):
    import pyruhvro_b200 as pr
    from tests.parity import assert_matches_pyoracle_wide, gen_case_wide
    bad = done = 0
    for seed in range(first, first + n_cases):
        rng = random.Random(seed * 31 + 7)
        sj, recs, data, off = gen_case_wide(seed, n=rng.choice([1, 7, 255, 256, 257, 600, 1500]))
        if not pr.Schema(sj).is_supported:
            continue
        k = rng.choice([1, 2, 8, 300])
        pr.set_jit_enabled(1 if seed % 16 == 0 else 0)
        try:
            assert_matches_pyoracle_wide(pr.deserialize_array_threaded(recs, sj, k), sj, recs, k)
            done += 1
        except Exception as e:
            bad += 1
            print(f"FAIL seed={seed} k={k} n={len(recs)}: {type(e).__name__}: {str(e)[:300]}\n  schema={sj[:400]}", flush=True)
    pr.set_jit_enabled(-1)
    print(f"wide fuzz done: first={first} cases={done} failures={bad}", flush=True)
    sys.exit(1 if bad else 0)


def main():
    if "--wide" in sys.argv:
        a = [x for x in sys.argv[1:] if x != "--wide"]
        return main_wide(int(a[0]), int(a[1]))
    args = [a for a in sys.argv[1:] if a != "--warm"]
    first, n_interp, n_jit = int(args[0]), int(args[1]), int(args[2])
    if "--warm" in sys.argv:
        from concurrent.futures import ProcessPoolExecutor
        with ProcessPoolExecutor(max_workers=os.cpu_count()) as ex:
            print("warmed", sum(ex.map(warm, range(first, first + n_jit))))
        return
    import pyruhvro_b200 as pr
    from oracle import pyoracle as po
    from tests.parity import assert_matches_oracle
    co = po.COracle()
    bad = 0
    for i in range(max(n_interp, n_jit)):
        seed = first + i
        sj = schema_for(seed)
        if not pr.Schema(sj).is_supported:   # beyond a documented limit (e.g. nesting depth 4)
            continue
        s = po.parse_schema(sj)
        rng = random.Random(seed + 99)
        n = rng.choice([1, 5, 64, 255, 256, 257, 1023, 3000])
        recs = [po.encode_datum(s, po.random_value(s, rng), neg_blocks=rng.random() < 0.3) for _ in range(n)]
        data, off = po.pack_records(recs)
        k = rng.choice([1, 2, 7, 5000])
        for walker, limit in (("interp", n_interp), ("jit", n_jit)):
            if i >= limit:
                continue
            pr.set_jit_enabled(1 if walker == "jit" else 0)
            try:
                got = pr.decode_packed(data, off, n, sj, k)
                assert pr.last_walker() == walker
                assert_matches_oracle(co, got, sj, data, off, n, k)
                if walker == "jit" and rng.random() < 0.5:   # encode round trip on canonical encodings
                    recs2 = [po.encode_datum(s, po.random_value(s, rng)) for _ in range(min(n, 300))]
                    b = pr.deserialize_array(recs2, sj)
                    out = [bytes(x.as_py()) for a in pr.serialize_record_batch(b, sj, 3) for x in a]
                    assert out == recs2
                    # the same rows in a layout the decoder never produces (offsets, junk, permuted union codes, ...)
                    from tests.arrow_layouts import relayout_batch
                    b2 = relayout_batch(b, rng)
                    out2 = [[bytes(x.as_py()) for x in a] for a in pr.serialize_record_batch(b2, sj, 3)]
                    assert out2 == po.py_encode(s, b2, 3) and [d for c in out2 for d in c] == recs2
            except Exception as e:
                bad += 1
                print(f"FAIL seed={seed} walker={walker} n={n} k={k}: {type(e).__name__}: {str(e)[:300]}\n  schema={sj[:400]}", flush=True)
    pr.set_jit_enabled(-1)
    print(f"fuzz done: first={first} interp={n_interp} jit={n_jit} failures={bad}", flush=True)
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
