"""Permissive decodes of several schema versions on one H100 (Versions.permissive, deserialize_confluent_versions(...,
errors="null")): 10 M Kafka messages, two schema ids alternating per message (workloads.KAFKA_SCHEMA and
workloads.kafka_v2_schema()), read as v2 with k = 8.

Four configurations alternated in rounds: the strict registry; its permissive form with no bad message; 0.01 % and 1 %
of the messages bad, half of them an empty datum (RV_ERR_EOF) and half an unregistered schema id (RV_ERR_FRAME).  Per
call: CUDA-event times of the partition, the groups' decodes and the take (rv_last_versions_timings), the device-resident
total (events around rv_decode_device_versions) and the end-to-end time through the host entry (rv_decode_host_versions
from pageable numpy input to pinned host batches).  Outside the timed loops each configuration's output is checked: the
clean permissive batches equal the strict ones column by column, and with bad messages the report lists exactly them and
the good rows equal the strict decode's.  The GPU's name and power limit are read in the same run (nvidia-smi
--query-gpu, read-only).  One JSON line per configuration and round.

    python tools/bench_versions_permissive.py [--n 10000000] [--k 8] [--steps 10] [--warmup 3] [--rounds 3]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def damaged(data, off, every, rng):
    """(data, offsets, bad indices) with one message in `every` bad: even ones cut to their header, odd ones id 99."""
    n = len(off) - 1
    bad = np.sort(rng.choice(n, size=max(1, n // every), replace=False))
    empty, unknown = bad[0::2], bad[1::2]
    lens = np.diff(off)
    is_empty = np.zeros(n, dtype=bool)
    is_empty[empty] = True
    pos = np.arange(int(off[-1])) - np.repeat(off[:-1], lens)
    keep = ~(np.repeat(is_empty, lens) & (pos >= 5))
    d = data.copy()
    d[off[unknown] + 4] = 99
    o = np.concatenate([[0], np.cumsum(np.where(is_empty, 5, lens))]).astype(np.int64)
    return np.ascontiguousarray(d[keep]), o, bad


def check(pa, batches, report, strict, bad):
    assert report.column(0).to_numpy().tolist() == bad.tolist(), "report"
    got = pa.Table.from_batches(batches)
    good = np.ones(strict.num_rows, dtype=bool)
    good[bad] = False
    mask = pa.array(good)
    for name in strict.column_names:
        g, w = got.column(name), strict.column(name)
        if pa.types.is_union(g.type):
            continue   # no validity: checked by tests/test_gpu_versions_permissive.py
        assert g.filter(mask).equals(w.filter(mask)), name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import pyarrow as pa
    import torch
    import pyruhvro_b200 as pr
    from tests import versions_cases as VC
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    L = pr.lib
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev)
    tbuf = (ctypes.c_float * 4)()
    data, off, _, _, v1, v2 = VC.kafka_versions_input(a.n, "alternate", k=a.k)
    strict_v = pr._get_or_create_versions({3: v1, 4: v2}, v2, None)
    perm_v = pr._get_or_create_versions({3: v1, 4: v2}, v2, None, permissive=True)
    rng = np.random.default_rng(7)
    inputs = {"strict": (strict_v, data, off, np.zeros(0, dtype=np.int64)), "clean": (perm_v, data, off, np.zeros(0, dtype=np.int64))}
    for name, every in (("bad_0.01pct", 10_000), ("bad_1pct", 100)):
        d, o, bad = damaged(data, off, every, rng)
        inputs[name] = (perm_v, d, o, bad)
    dev_in = {}
    for name, (v, d, o, bad) in inputs.items():
        dd = torch.zeros(len(d) + 64, dtype=torch.uint8, device=dev)
        dd[:len(d)].copy_(torch.from_numpy(d))
        dev_in[name] = (dd, torch.from_numpy(o).to(dev))

    def run_dev(name):
        v = inputs[name][0]
        dd, do = dev_in[name]
        h = ctypes.c_void_p()
        pr._check(L.rv_decode_device_versions(v.handle, dd.data_ptr(), do.data_ptr(), a.n, a.k, stream.cuda_stream, ctypes.byref(h)))
        return h.value

    def run_host(name):
        v, d, o, _ = inputs[name]
        h = ctypes.c_void_p()
        pr._check(L.rv_decode_host_versions(v.handle, d.ctypes.data, o.ctypes.data, a.n, a.k, ctypes.byref(h)))
        return h.value

    # outputs, outside the timed loops
    h = run_dev("strict")
    pr._check(L.rv_result_to_host(h))
    strict = pa.Table.from_batches(pr._export_batches(h, strict_v.reader))
    for name in ("clean", "bad_0.01pct", "bad_1pct"):
        h = run_dev(name)
        pr._check(L.rv_result_to_host(h))
        batches, report = pr._export_batches(h, perm_v.reader, True)
        check(pa, batches, report, strict, inputs[name][3])
        print(json.dumps({"config": name, "checked": "strict decode", "bad": len(inputs[name][3])}), flush=True)
    del strict

    for rnd in range(a.rounds):
        for name in inputs:
            for _ in range(a.warmup):
                L.rv_result_free(run_dev(name))
            torch.cuda.synchronize()
            parts = np.zeros(4)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(a.steps):
                h = run_dev(name)
                L.rv_last_versions_timings(tbuf, 4)
                parts += np.array(list(tbuf))
                L.rv_result_free(h)
            e1.record(stream)
            torch.cuda.synchronize()
            dev_ms = e0.elapsed_time(e1) / a.steps
            rec = {"config": name, "round": rnd, "n": a.n, "k": a.k, "bad": len(inputs[name][3]), "device_ms": round(dev_ms, 3),
                   "device_rec_per_s": round(a.n / (dev_ms / 1e3)), "gpu": gpu}
            rec.update({f"{p}_ms": round(x / a.steps, 3) for p, x in zip(("partition", "decodes", "take", "events_total"), parts)})
            L.rv_result_free(run_host(name))
            t0 = time.perf_counter()
            for _ in range(3):
                L.rv_result_free(run_host(name))
            rec["host_e2e_ms"] = round((time.perf_counter() - t0) / 3 * 1e3, 3)
            print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
