#!/usr/bin/env python
"""Precompiles (NVRTC, no GPU needed) the schema-specialised kernels of every schema the GPU tests,
smoke() and bench.py decode with the "jit" walker, into pyruhvro_b200/_jitcache/ — the cache travels
with the repo snapshot, so GPU time is not spent compiling."""
import os
import sys
from concurrent.futures import ProcessPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def schemas():
    import workloads
    from tests import malformed
    from tests.golden import reference_datums as G
    from tests.parity import gen_case
    from tests.test_gpu_parity import JIT_SEEDS
    out = [G.G1_SCHEMA, G.G2_SCHEMA, G.G345_SCHEMA, malformed.FLAT]
    out += [cfg[1] for cfg in workloads.CONFIGS.values()]
    out += [gen_case(seed, n=1)[0] for seed in JIT_SEEDS]
    out += [gen_case(s, n=1)[0] for s in (5, 7)]
    out.append('{"type":"record","name":"L","fields":[{"name":"s","type":"string"},{"name":"a","type":{"type":"array","items":"long"}}]}')
    out.append('{"type":"record","name":"Z","fields":[{"name":"z","type":{"type":"array","items":"null"}},'
               '{"name":"m","type":{"type":"map","values":{"type":"array","items":{"type":"array","items":["null","string"]}}}}]}')
    out.append('{"type":"record","name":"C","fields":[{"name":"id","type":"long"},{"name":"s","type":["null","string"]},'
               '{"name":"xs","type":{"type":"array","items":"int"}}]}')
    out.append('{"type":"record","name":"H","fields":[{"name":"s","type":"string"},{"name":"xs","type":{"type":"array","items":"string"}}]}')
    from tests.parity import gen_case_wide
    from tests.test_wide_types import ALL_WIDE
    out.append(ALL_WIDE)
    out += [gen_case_wide(seed, n=1)[0] for seed in range(30) if seed % 3]
    out.append('{"type":"record","name":"R","fields":[{"name":"id","type":"long"},{"name":"u","type":{"type":"string","logicalType":"uuid"}}]}')
    from tests.test_gpu_fast_paths import JIT_PROJECTIONS, JIT_SCHEMAS
    out += JIT_SCHEMAS
    out += [(sj, tuple(cols)) for sj, cols in JIT_PROJECTIONS]  # a projected plan has its own walker
    from tests.test_gpu_tile384 import HB_SCHEMA, KAFKA_PROJECTIONS
    out.append(HB_SCHEMA)
    out += [(workloads.KAFKA_SCHEMA, tuple(cols)) for cols in KAFKA_PROJECTIONS]
    from tests.test_gpu_ocf import BIG_SCHEMA
    from tests.test_ocf import BOOL_STR_SCHEMA, ZW_SCHEMA
    out += [BIG_SCHEMA, BOOL_STR_SCHEMA, ZW_SCHEMA]
    from tests.test_resolve_edges import JIT_RESOLVED
    out += JIT_RESOLVED  # a resolved plan (writer, reader) has its own walker
    from tests.test_gpu_permissive import jit_permissive
    out += [("permissive",) + item for item in jit_permissive()]  # so has a permissive one (schema, columns, reader)
    return list(dict.fromkeys(out))


def one(item):
    """A schema, (schema, columns) for a projected plan, (writer, reader) for a resolved one or ("permissive", schema,
    columns, reader) for a permissive one."""
    import pyruhvro_b200 as pr
    if isinstance(item, tuple) and item[0] == "permissive":
        _, sj, cols, reader = item
        s = pr.Schema(sj)
        if reader is not None:
            s = s.read_as(reader)
        if cols is not None:
            s = s.project(list(cols))
        s.permissive().precompile("sm_90a")
        return 1
    sj, cols = item if isinstance(item, tuple) else (item, None)
    s = pr.Schema(sj)
    if isinstance(cols, str):
        s = s.read_as(cols)
    elif cols is not None:
        s = s.project(list(cols))
    s.precompile("sm_90a")
    return 1


if __name__ == "__main__":
    todo = schemas()
    with ProcessPoolExecutor(max_workers=os.cpu_count() or 4) as ex:
        done = sum(ex.map(one, todo))
    print(f"precompiled {done} schemas into pyruhvro_b200/_jitcache")
