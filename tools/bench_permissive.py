"""What permissive decoding costs on one H100: the strict decode of 10 M Confluent-framed Kafka messages (workloads
.generate("kafka"), k = 8) against permissive decodes (errors="null") of the same messages with 0, 0.01 % and 1 % of them
damaged at known positions (every other damaged message emptied, the rest given a wrong magic byte).  The permissive
plan writes a validity bitmap for every top-level column, and each damaged message puts its warp on the precise walk.

For each configuration, alternated in rounds: the fused kernel's time (CUDA events, rv_last_timings[0]), the device-
resident call (rv_decode_device_framed, CUDA events around `steps` calls) and the end-to-end call from pageable numpy
input to pinned host batches (rv_decode_host_framed, host clock).  Every output is checked outside the timed loops: good
rows equal the strict decode's, bad rows are null, the report lists exactly the damaged messages.  The GPU's name and
power limit are read in the same run (nvidia-smi --query-gpu, read-only).  One JSON line per configuration and round.

    python tools/bench_permissive.py [--n 10000000] [--k 8] [--steps 10] [--warmup 3] [--rounds 3]
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

CONFIGS = (("strict", None), ("permissive_0", 0), ("permissive_0.01%", 10_000), ("permissive_1%", 100))   # (name, one damaged in)


def framed(data, off, damaged):
    """Confluent frames (schema id 7) around each datum; of the `damaged` messages, every other one is empty and the rest
    have a wrong magic byte."""
    lens = np.diff(off)
    empty = np.zeros(len(lens), dtype=bool)
    empty[damaged[::2]] = True
    mlens = np.where(empty, 0, lens + 5)
    moff = np.concatenate([[0], np.cumsum(mlens)]).astype(np.int64)
    out = np.zeros(int(moff[-1]), dtype=np.uint8)
    out[moff[:-1][~empty] + 4] = 7
    src = np.repeat(~empty, lens)   # per input byte: its message is kept
    dst = np.repeat(moff[:-1] + 5 - off[:-1], lens) + np.arange(int(off[0]), int(off[-1]))
    out[dst[src]] = data[int(off[0]):int(off[-1])][src]
    out[moff[:-1][damaged[1::2]]] = 1
    return out, moff


def check(strict, batches, bad, damaged):
    import pyarrow as pa
    assert bad.column(0).to_numpy().tolist() == damaged.tolist(), "report: damaged records"
    assert set(bad.column(1).to_pylist()) <= {12}, "report: statuses"
    assert [b.num_rows for b in batches] == [b.num_rows for b in strict], "batch row counts"
    got, want = pa.Table.from_batches(batches), pa.Table.from_batches(strict)
    good = np.ones(got.num_rows, dtype=bool)
    good[damaged] = False
    for name in want.column_names:
        g, w = got.column(name), want.column(name)
        if pa.types.is_union(g.type):
            gt = np.concatenate([np.frombuffer(c.buffers()[1], np.int8)[c.offset:c.offset + len(c)] for c in g.chunks])
            wt = np.concatenate([np.frombuffer(c.buffers()[1], np.int8)[c.offset:c.offset + len(c)] for c in w.chunks])
            assert np.array_equal(gt[good], wt[good]) and not gt[~good].any(), name
            continue
        if pa.types.is_map(g.type):     # an empty map at a bad row
            assert g.filter(pa.array(good)).equals(w.filter(pa.array(good))), name
            o = g.filter(pa.array(~good)).combine_chunks().offsets.to_numpy()
            assert o[0] == o[-1], name
            continue
        assert g.filter(pa.array(good)).equals(w.filter(pa.array(good))), name
        assert g.filter(pa.array(~good)).null_count == len(damaged), name


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import torch
    import pyruhvro_b200 as pr
    import workloads
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    L = pr.lib
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev)
    n, k = a.n, a.k
    sj, data, off = workloads.generate("kafka", n, seed=42)
    data, off = np.ascontiguousarray(data), np.ascontiguousarray(off, dtype=np.int64)
    framing = pr.Framing(5, 1, -1)
    tbuf = (ctypes.c_float * 6)()

    def timed(fn):
        for _ in range(a.warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(a.steps):
            fn()
        e1.record(stream)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.steps

    def host_ms(fn, reps=3):
        fn()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        return (time.perf_counter() - t0) / reps * 1e3

    def call(entry, *args):
        def run():
            h = ctypes.c_void_p()
            pr._check(entry(*args, ctypes.byref(h)))
            return h.value
        return run

    strict_out = None
    sides = {}
    for name, every in CONFIGS:
        damaged = np.arange(0, n, every, dtype=np.int64) if every else np.zeros(0, dtype=np.int64)
        mdata, moff = framed(data, off, damaged)
        s = pr._get_or_parse_schema(sj, permissive=every is not None)
        d_data = torch.zeros(len(mdata) + 64, dtype=torch.uint8, device=dev)
        d_data[:len(mdata)].copy_(torch.from_numpy(mdata))
        d_off = torch.from_numpy(moff).to(dev)
        dev_run = call(L.rv_decode_device_framed, s.handle, d_data.data_ptr(), d_off.data_ptr(), n, k, ctypes.byref(framing), stream.cuda_stream)
        host_run = call(L.rv_decode_host_framed, s.handle, mdata.ctypes.data, moff.ctypes.data, n, k, ctypes.byref(framing))
        h = dev_run()   # checked outside the timed loops
        pr._check(L.rv_result_to_host(h))
        if every is None:
            strict_out = pr._export_batches(h, s)
        else:
            batches, bad = pr._export_batches(h, s, True)
            check(strict_out, batches, bad, damaged)
            del batches
        print(json.dumps({"config": name, "damaged": int(len(damaged)), "checked": "strict decode", "n": n, "k": k, "gpu": gpu}), flush=True)
        sides[name] = (dev_run, host_run, (d_data, d_off, mdata, moff), int(moff[-1]))
    del strict_out
    for rnd in range(a.rounds):
        for name, (dev_run, host_run, _, nbytes) in sides.items():
            ms = timed(lambda: L.rv_result_free(dev_run()))
            L.rv_last_timings(tbuf, 6)
            kernel_ms = tbuf[0]
            e2e = host_ms(lambda: L.rv_result_free(host_run()))
            print(json.dumps({"config": name, "round": rnd, "kernel_ms": round(kernel_ms, 3), "device_ms": round(ms, 3),
                              "device_Mrec_s": round(n / ms / 1e3, 1), "host_e2e_ms": round(e2e, 3), "host_e2e_Mrec_s": round(n / e2e / 1e3, 1),
                              "input_GB": round(nbytes / 1e9, 3), "n": n, "k": k, "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
