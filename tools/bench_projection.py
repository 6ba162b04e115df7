"""Column projection on one H100: the full decode next to projected decodes of the same batch, measured in one run.

For each case (workload, columns) it reports the fused-kernel time (rv_last_timings[0]), device-resident records/s
(rv_decode_device, CUDA events around `--steps` calls), end-to-end records/s through rv_decode_host (pinned host buffers
in and out, wall clock around calls that end in a device synchronise) and rv_result_arrow_bytes.  Outside the timed
loops, every case's output is checked buffer for buffer against the C oracle's full decode, selected.  The GPU's name
and power limit are read in the same run (nvidia-smi --query-gpu, read-only).  Prints one JSON line per case.

    python tools/bench_projection.py [--n 10000000] [--k 8] [--steps 20] [--warmup 3]
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

CASES = [("kafka", None), ("kafka", ["created_at"]), ("kafka", ["name", "age", "created_at"]), ("kafka", ["emails", "phone_numbers"]),
         ("kafka", ["status", "class"]), ("flat", None), ("flat", ["i"])]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-check", action="store_true", help="skip the oracle comparison")
    a = ap.parse_args()
    import torch
    import pyruhvro_b200 as pr
    import workloads
    from oracle import pyoracle as po
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    L = pr.lib
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev)
    co = None if a.no_check else po.COracle()
    loaded = {}
    for wl, cols in CASES:
        if wl not in loaded:
            loaded.clear()
            sj, h_data, h_off = workloads.generate(wl, a.n, seed=42)
            total = int(h_off[a.n])
            p_data = np.frombuffer((ctypes.c_uint8 * total).from_address(L.rv_host_alloc(total)), dtype=np.uint8)
            p_data[:] = h_data
            p_off = np.frombuffer((ctypes.c_int64 * (a.n + 1)).from_address(L.rv_host_alloc((a.n + 1) * 8)), dtype=np.int64)
            p_off[:] = h_off
            d_data = torch.zeros(total + 64, dtype=torch.uint8, device=dev)
            d_data[:total].copy_(torch.from_numpy(p_data))
            d_off = torch.from_numpy(p_off).to(dev)
            want = co.decode_threaded_packed(sj, p_data, p_off, a.n, a.k, threads=os.cpu_count() or 4) if co else None
            loaded[wl] = (sj, p_data, p_off, d_data, d_off, want)
            torch.cuda.synchronize()
        sj, p_data, p_off, d_data, d_off, want = loaded[wl]
        s = pr._get_or_parse_schema(sj, cols)
        tbuf = (ctypes.c_float * 6)()

        def dev_step():
            h = ctypes.c_void_p()
            pr._check(L.rv_decode_device(s.handle, d_data.data_ptr(), d_off.data_ptr(), a.n, a.k, stream.cuda_stream, ctypes.byref(h)))
            return h.value

        def host_step():
            h = ctypes.c_void_p()
            pr._check(L.rv_decode_host(s.handle, p_data.ctypes.data, p_off.ctypes.data, a.n, a.k, ctypes.byref(h)))
            return h.value

        for _ in range(a.warmup):
            L.rv_result_free(dev_step())
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        kernel_ms = 0.0
        passes = 0
        e0.record(stream)
        for _ in range(a.steps):
            h = dev_step()
            L.rv_last_timings(tbuf, 6)
            kernel_ms += tbuf[0]
            passes = max(passes, L.rv_last_passes())
            arrow_bytes = L.rv_result_arrow_bytes(h)
            L.rv_result_free(h)
        e1.record(stream)
        torch.cuda.synchronize()
        dev_ms = e0.elapsed_time(e1) / a.steps
        for _ in range(a.warmup):
            L.rv_result_free(host_step())
        t0 = time.perf_counter()
        for _ in range(a.steps):
            L.rv_result_free(host_step())
        torch.cuda.synchronize()
        e2e_ms = 1e3 * (time.perf_counter() - t0) / a.steps
        checked = None
        if want is not None:  # outside the timed loops: one more call, checked buffer for buffer
            batches = pr._export_batches(host_step(), s)
            names = [f.name for f in pr.Schema(sj).arrow_schema]
            idx = list(range(len(names))) if cols is None else [names.index(c) for c in cols]
            for i, (b, w) in enumerate(zip(batches, want)):
                d = po.canon_diff(po.canon_from_batch(b), [w[j] for j in idx], f"batch[{i}]")
                if d:
                    raise SystemExit(f"{wl} {cols}: output differs from the oracle: {d}")
            checked = "oracle"
        print(json.dumps({"workload": wl, "columns": cols, "n": a.n, "k": a.k, "steps": a.steps, "walker": pr.last_walker(),
                          "kernel_ms": round(kernel_ms / a.steps, 4), "device_ms": round(dev_ms, 4),
                          "device_rec_per_s": round(a.n / (dev_ms / 1e3)), "e2e_ms": round(e2e_ms, 3),
                          "e2e_rec_per_s": round(a.n / (e2e_ms / 1e3)), "arrow_bytes": int(arrow_bytes), "passes": passes,
                          "checked": checked, "gpu": gpu}), flush=True)


if __name__ == "__main__":
    main()
