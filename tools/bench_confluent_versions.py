"""Confluent messages of several schema versions on one H100 (deserialize_confluent_versions / rv_decode_*_versions):
10 M Kafka messages whose rows come from workloads.generate("kafka"), each framed with the id of the schema it is
encoded with (workloads.KAFKA_SCHEMA or workloads.kafka_v2_schema()), read as v2 with k = 8.

Mixes: one id (alternated in the same run with deserialize_confluent(..., reader_schema=) on the same messages), two ids in
runs of 100 000, two ids alternating per message, four ids (two ids per schema) alternating.  Per call: CUDA-event times
of the partition, the groups' decodes and the take (rv_last_versions_timings), the device-resident total (events
around rv_decode_device_versions) and the end-to-end time through the host entry (rv_decode_host_versions from pageable
numpy input to pinned host batches).  Outside the timed loops every buffer is checked against the C oracle.  The GPU's
name and power limit are read in the same run (nvidia-smi --query-gpu, read-only).  One JSON line per mix and round.

    python tools/bench_confluent_versions.py [--n 10000000] [--k 8] [--steps 10] [--warmup 3] [--rounds 3]
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-check", action="store_true")
    a = ap.parse_args()
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
    mixes = [("one", "one", (3, 4)), ("runs", ("runs", 100_000), (3, 4)), ("alternate", "alternate", (3, 4)), ("four_ids", "alternate", (3, 4, 5, 6))]
    for name, mix, ids in mixes:
        data, off, h_data, h_off, v1, v2 = VC.kafka_versions_input(a.n, mix, ids=ids, k=a.k)
        d_data = torch.zeros(len(data) + 64, dtype=torch.uint8, device=dev)
        d_data[:len(data)].copy_(torch.from_numpy(data))
        d_off = torch.from_numpy(off).to(dev)
        writers = {i: (v1 if q % 2 == 0 else v2) for q, i in enumerate(ids)}
        v = pr._get_or_create_versions(writers, v2, None)
        resolved = pr._get_or_parse_schema(v1, None, v2)
        framing = pr.Framing(5, 1, 3)

        def versions_dev():
            h = ctypes.c_void_p()
            pr._check(L.rv_decode_device_versions(v.handle, d_data.data_ptr(), d_off.data_ptr(), a.n, a.k, stream.cuda_stream, ctypes.byref(h)))
            return h.value

        def single_dev():
            h = ctypes.c_void_p()
            pr._check(L.rv_decode_device_framed(resolved.handle, d_data.data_ptr(), d_off.data_ptr(), a.n, a.k, ctypes.byref(framing),
                                                stream.cuda_stream, ctypes.byref(h)))
            return h.value

        def versions_host():
            h = ctypes.c_void_p()
            pr._check(L.rv_decode_host_versions(v.handle, data.ctypes.data, off.ctypes.data, a.n, a.k, ctypes.byref(h)))
            return h.value

        calls = [("versions", versions_dev)] + ([("reader_schema", single_dev)] if name == "one" else [])
        for rnd in range(a.rounds):
            for cname, fn in calls:
                for _ in range(a.warmup):
                    L.rv_result_free(fn())
                torch.cuda.synchronize()
                parts = np.zeros(4)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(a.steps):
                    h = fn()
                    if cname == "versions":
                        L.rv_last_versions_timings(tbuf, 4)
                        parts += np.array(list(tbuf))
                    L.rv_result_free(h)
                e1.record(stream)
                torch.cuda.synchronize()
                dev_ms = e0.elapsed_time(e1) / a.steps
                rec = {"mix": name, "round": rnd, "call": cname, "n": a.n, "k": a.k, "device_ms": round(dev_ms, 3),
                       "device_rec_per_s": round(a.n / (dev_ms / 1e3)), "gpu": gpu}
                if cname == "versions":
                    rec.update({f"{p}_ms": round(x / a.steps, 3) for p, x in zip(("partition", "decodes", "take", "events_total"), parts)})
                    L.rv_result_free(versions_host())
                    t0 = time.perf_counter()
                    for _ in range(3):
                        L.rv_result_free(versions_host())
                    rec["host_e2e_ms"] = round((time.perf_counter() - t0) / 3 * 1e3, 3)
                print(json.dumps(rec), flush=True)
        if not a.no_check:
            h = versions_dev()
            pr._check(L.rv_result_to_host(h))
            VC.check_kafka_v2(pr._export_batches(h, v.reader), v1, v2, h_data, h_off, a.n, a.k)
            print(json.dumps({"mix": name, "checked": "oracle"}), flush=True)
        del d_data, d_off


if __name__ == "__main__":
    main()
