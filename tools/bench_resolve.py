"""Schema resolution on one H100: Kafka records written with the bench's schema (workloads.KAFKA_SCHEMA), decoded plain and
read as "Kafka v2" (workloads.kafka_v2_schema: a dropped map, a widened int, three default fields, a new enum symbol,
a reshaped nested record, a moved column), measured in one process.

Each round times the plain decode and then the resolved one (`--rounds` alternations): the fused-kernel time
(rv_last_timings[0]) and device-resident records/s (rv_decode_device, CUDA events around `--steps` calls).  Outside the
timed loops, the resolved batches are checked against the C oracle's decode of the same records, converted column by
column the way Kafka v2 reads them.  The GPU's name and power limit are read in the same run (nvidia-smi --query-gpu,
read-only).  Prints one JSON line per round and decode.

    python tools/bench_resolve.py [--n 10000000] [--k 8] [--steps 20] [--warmup 3] [--rounds 3]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def expected_v2(plain, v2_schema):
    """A plain Kafka batch as Kafka v2 reads it (Arrow compute on the oracle's columns)."""
    import pyarrow as pa
    import pyarrow.compute as pc
    n = plain.num_rows
    addr = plain.column("address")
    country = pc.if_else(addr.is_valid(), pa.scalar("US"), pa.scalar(None, pa.string()))
    address = pa.StructArray.from_arrays([addr.field("city"), addr.field("street"), country], fields=list(v2_schema.field("address").type),
                                         mask=addr.is_null())
    cols = {"created_at": plain.column("created_at"), "name": plain.column("name"), "age": plain.column("age").cast(pa.int64()),
            "emails": plain.column("emails"), "address": address, "preferences": plain.column("preferences"),
            "status": plain.column("status"), "class": plain.column("class"), "country": pa.nulls(n, pa.string()),
            "score": pa.array(np.zeros(n)), "source": pa.array(["kafka"] * n)}
    return [cols[f.name] for f in v2_schema]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=10_000_000)
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
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
    sj, h_data, h_off = workloads.generate("kafka", a.n, seed=42)
    total = int(h_off[a.n])
    d_data = torch.zeros(total + 64, dtype=torch.uint8, device=dev)
    d_data[:total].copy_(torch.from_numpy(np.ascontiguousarray(h_data)))
    d_off = torch.from_numpy(np.ascontiguousarray(h_off, dtype=np.int64)).to(dev)
    v2 = workloads.kafka_v2_schema()
    handles = {"plain": pr._get_or_parse_schema(sj), "resolved": pr._get_or_parse_schema(sj, None, v2)}
    tbuf = (ctypes.c_float * 6)()

    def dev_step(s):
        h = ctypes.c_void_p()
        pr._check(L.rv_decode_device(s.handle, d_data.data_ptr(), d_off.data_ptr(), a.n, a.k, stream.cuda_stream, ctypes.byref(h)))
        return h.value

    for rnd in range(a.rounds):
        for name in ("plain", "resolved"):
            s = handles[name]
            for _ in range(a.warmup):
                L.rv_result_free(dev_step(s))
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            kernel_ms, passes = 0.0, 0
            e0.record(stream)
            for _ in range(a.steps):
                h = dev_step(s)
                L.rv_last_timings(tbuf, 6)
                kernel_ms += tbuf[0]
                passes = max(passes, L.rv_last_passes())
                L.rv_result_free(h)
            e1.record(stream)
            torch.cuda.synchronize()
            dev_ms = e0.elapsed_time(e1) / a.steps
            print(json.dumps({"round": rnd, "decode": name, "n": a.n, "k": a.k, "steps": a.steps, "walker": pr.last_walker(),
                              "tile": L.rv_last_tile(), "kernel_ms": round(kernel_ms / a.steps, 4), "device_ms": round(dev_ms, 4),
                              "device_rec_per_s": round(a.n / (dev_ms / 1e3)), "passes": passes, "gpu": gpu}), flush=True)
    if not a.no_check:   # outside the timed loops: the resolved batches against the oracle's decode, converted
        co = po.COracle()
        want = co.decode_threaded_packed(sj, np.ascontiguousarray(h_data), np.ascontiguousarray(h_off, dtype=np.int64), a.n, a.k,
                                         threads=os.cpu_count() or 4)
        s = handles["resolved"]
        h = dev_step(s)
        pr._check(L.rv_result_to_host(h))
        got = pr._export_batches(h, s)
        plain_schema = handles["plain"].arrow_schema
        for i, (b, w) in enumerate(zip(got, want)):
            exp = expected_v2(po.canon_to_batch(w, plain_schema), s.arrow_schema)
            for j, col in enumerate(exp):
                if not b.column(j).equals(col):
                    raise SystemExit(f"batch {i} column {s.arrow_schema.names[j]}: differs from the oracle")
        print(json.dumps({"checked": "oracle", "batches": len(got)}), flush=True)


if __name__ == "__main__":
    main()
