"""The framed encodes on one H100: 10 M Kafka records decoded into a pinned batch, then encoded as bare datums
(serialize_record_batch, k = 8), as Confluent-framed messages (serialize_confluent, k = 8) and as one Object Container
File (serialize_ocf, 1024 records per block), measured in one process.

Each round times the three encodes one after the other (`--rounds` alternations, `--steps` calls each after `--warmup`):
median call time, records/s, the summed encode kernel time (rv_last_encode_timings [0] + [1] + [2]: size, scan, write
with the framing) and output bytes.  Outside the timed loops, the Confluent arrays are checked byte for byte against
serialize_record_batch's datums with the 5-byte header, and the file against a numpy assembly of header + blocks from
serialize_record_batch's datums.  The GPU's name and power limit are read in the same run (nvidia-smi --query-gpu,
read-only).  Prints one JSON line per round and encode.

    python tools/bench_encode_framed.py [--n 10000000] [--k 8] [--block 1024] [--steps 10] [--warmup 2] [--rounds 3]
"""
import argparse
import ctypes
import json
import os
import statistics
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
    ap.add_argument("--block", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    import pyruhvro_b200 as pr
    import workloads
    from tests import ocf_files as O
    if subprocess.run(["nvidia-smi", "-L"], capture_output=True).returncode != 0:
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    sj, h_data, h_off = workloads.generate("kafka", a.n, seed=42)
    batch = pr.decode_packed(h_data, h_off, a.n, sj, 1)[0]     # pinned buffers: the upload goes direct
    sid, sync = 0x2A, bytes(range(16))
    calls = {
        "serialize_record_batch": lambda: pr.serialize_record_batch(batch, sj, a.k),
        "serialize_confluent": lambda: pr.serialize_confluent(batch, sj, sid, a.k),
        "serialize_ocf": lambda: pr.serialize_ocf(batch, sj, a.block, sync_marker=sync),
    }

    def out_bytes(r):
        if isinstance(r, list):
            return sum(int(np.frombuffer(x.buffers()[1], dtype=np.int32)[len(x)]) for x in r)
        return r.size

    tb = (ctypes.c_float * 5)()
    for rnd in range(a.rounds):
        for name, call in calls.items():
            for _ in range(a.warmup):
                call()
            times, kern = [], []
            for _ in range(a.steps):
                t0 = time.perf_counter()
                r = call()                      # returns after the last download was synchronised
                times.append(time.perf_counter() - t0)
                pr.lib.rv_last_encode_timings(tb, 5)
                kern.append(tb[0] + tb[1] + tb[2])
                size = out_bytes(r)
                del r
            med = statistics.median(times)
            print(json.dumps({"round": rnd, "encode": name, "n": a.n, "k": a.k if name != "serialize_ocf" else None,
                              "block_records": a.block if name == "serialize_ocf" else None, "steps": a.steps,
                              "median_ms": round(med * 1e3, 3), "rec_per_s": round(a.n / med),
                              "kernel_ms": round(statistics.median(kern), 3), "out_bytes": size, "gpu": gpu}), flush=True)

    # outside the timed loops: byte-for-byte checks against serialize_record_batch's datums
    plain = pr.serialize_record_batch(batch, sj, a.k)
    conf = pr.serialize_confluent(batch, sj, sid, a.k)
    head = np.frombuffer(b"\x00" + sid.to_bytes(4, "big"), dtype=np.uint8)
    for p, c in zip(plain, conf):
        m = len(p)
        po_ = np.frombuffer(p.buffers()[1], dtype=np.int32)[:m + 1]
        co = np.frombuffer(c.buffers()[1], dtype=np.int32)[:m + 1]
        if len(c) != m or not np.array_equal(co, po_ + 5 * np.arange(m + 1, dtype=np.int32)):
            raise SystemExit("Confluent offsets differ from the datums' with 5-byte headers")
        got = np.frombuffer(c.buffers()[2], dtype=np.uint8)[:co[-1]]
        heads = (co[:-1, None] + np.arange(5)).ravel()
        mask = np.ones(len(got), dtype=bool)
        mask[heads] = False
        if not (np.array_equal(got[heads], np.tile(head, m)) and np.array_equal(got[mask], np.frombuffer(p.buffers()[2], dtype=np.uint8)[:po_[-1]])):
            raise SystemExit("Confluent bytes differ from the header + datum")
    (one,) = pr.serialize_record_batch(batch, sj, 1)
    off = np.frombuffer(one.buffers()[1], dtype=np.int32)[:a.n + 1]
    data = np.frombuffer(one.buffers()[2], dtype=np.uint8)
    parts = [np.frombuffer(O.ocf_header(sj, sync), dtype=np.uint8)]
    s = np.frombuffer(sync, dtype=np.uint8)
    for i in range(0, a.n, a.block):
        j = min(a.n, i + a.block)
        parts += [np.frombuffer(O.zz(j - i) + O.zz(int(off[j] - off[i])), dtype=np.uint8), data[off[i]:off[j]], s]
    f = pr.serialize_ocf(batch, sj, a.block, sync_marker=sync)
    if not np.array_equal(np.frombuffer(f, dtype=np.uint8), np.concatenate(parts)):
        raise SystemExit("the container file differs from the assembly of serialize_record_batch's datums")
    print(json.dumps({"checked": "bytes", "confluent_chunks": len(conf), "file_bytes": f.size}), flush=True)


if __name__ == "__main__":
    main()
