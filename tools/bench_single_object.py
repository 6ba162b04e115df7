"""Avro single-object messages against Confluent-framed ones on one H100: the same 10 M Kafka rows
(workloads.generate("kafka")) framed both ways, k = 8.  Three pairs, the two sides of each alternated in the same run:

  decode     deserialize_confluent / deserialize_single_object: rv_decode_device_framed against
             rv_decode_device_single_object (device-resident), rv_decode_host_framed against rv_decode_host_single_object
             (end to end, pageable numpy input to pinned host batches)
  versions   deserialize_confluent_versions / deserialize_single_object_versions: two writers (workloads.KAFKA_SCHEMA and
             workloads.kafka_v2_schema()) alternating per message, read as v2; rv_decode_device_versions on each registry
             (device-resident) and rv_decode_host_versions (end to end)
  encode     serialize_confluent / serialize_single_object of a pinned batch (end to end) and the encode kernels' CUDA-event
             times (rv_last_encode_timings: size, scan, write)

Warm-up first; every output is checked outside the timed loops (decodes against the C oracle, encodes byte for byte
against serialize_record_batch's datums behind the header).  The GPU's name and power limit are read in the same run
(nvidia-smi --query-gpu, read-only).  One JSON line per pair, side and round.

    python tools/bench_single_object.py [--n 10000000] [--k 8] [--steps 10] [--warmup 3] [--rounds 3]
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


def kafka_single_object_input(n, k, v1, v2, h_data, h_off):
    """n single-object messages of the Kafka rows, alternating between v1 (the generated datum) and v2 (the row read as
    v2 and re-encoded by the GPU encoder): the messages of versions_cases.kafka_versions_input(n, "alternate"), framed
    with the writers' fingerprints."""
    import pyarrow as pa
    import pyarrow.compute as pc
    import pyruhvro_b200 as pr
    plain = pr.decode_packed(h_data, h_off, n, v1, k)
    as_v2 = pr.decode_packed(h_data, h_off, n, v1, k, reader_schema=v2)
    out, row = [], 0
    for p1, b2 in zip(plain, as_v2):
        m = b2.num_rows
        a1 = pr.serialize_single_object(p1, v1, 1)[0].cast(pa.large_binary())
        a2 = pr.serialize_single_object(b2, v2, 1)[0].cast(pa.large_binary())
        out.append(pc.if_else(pa.array((np.arange(row, row + m) % 2) == 1), a2, a1))
        row += m
    data, off, _ = pr._packed_view(pa.concat_arrays(out))
    return np.ascontiguousarray(data), np.ascontiguousarray(off, dtype=np.int64)


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
    import workloads
    from oracle import pyoracle as po
    from tests import single_object as SO
    from tests import versions_cases as VC
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()
    L = pr.lib
    L.rv_last_encode_timings.argtypes = [ctypes.POINTER(ctypes.c_float), ctypes.c_int]
    dev = torch.device("cuda", 0)
    stream = torch.cuda.current_stream(dev)
    n, k = a.n, a.k

    def on_device(data, off):
        d_data = torch.zeros(len(data) + 64, dtype=torch.uint8, device=dev)
        d_data[:len(data)].copy_(torch.from_numpy(data))
        return d_data, torch.from_numpy(off).to(dev)

    def timed(fn):
        """device ms per call: CUDA events around `steps` calls, after the warm-up"""
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

    def decode_call(entry, *args):
        def run():
            h = ctypes.c_void_p()
            pr._check(entry(*args, ctypes.byref(h)))
            return h.value
        return run

    def freed(run):
        return lambda: L.rv_result_free(run())

    def emit(rec):
        rec.update({"n": n, "k": k, "gpu": gpu})
        print(json.dumps(rec), flush=True)

    # ---- decode: one writer ---------------------------------------------------------------------------------------
    v1, h_data, h_off = workloads.generate("kafka", n, seed=42)
    v2 = workloads.kafka_v2_schema()
    h_data, h_off = np.ascontiguousarray(h_data), np.ascontiguousarray(h_off, dtype=np.int64)
    src = pr.decode_packed(h_data, h_off, n, v1, k)
    conf = pa.concat_arrays([pr.serialize_confluent(b, v1, 77, 1)[0].cast(pa.large_binary()) for b in src])
    sobj = pa.concat_arrays([pr.serialize_single_object(b, v1, 1)[0].cast(pa.large_binary()) for b in src])
    s1 = pr._get_or_parse_schema(v1)
    framing = pr.Framing(5, 1, 77)
    sides = {}
    for name, arr in (("confluent", conf), ("single_object", sobj)):
        data, off, _ = pr._packed_view(arr)
        data, off = np.ascontiguousarray(data), np.ascontiguousarray(off, dtype=np.int64)
        d_data, d_off = on_device(data, off)
        if name == "confluent":
            dev_run = decode_call(L.rv_decode_device_framed, s1.handle, d_data.data_ptr(), d_off.data_ptr(), n, k, ctypes.byref(framing), stream.cuda_stream)
            host_run = decode_call(L.rv_decode_host_framed, s1.handle, data.ctypes.data, off.ctypes.data, n, k, ctypes.byref(framing))
        else:
            dev_run = decode_call(L.rv_decode_device_single_object, s1.handle, d_data.data_ptr(), d_off.data_ptr(), n, k, stream.cuda_stream)
            host_run = decode_call(L.rv_decode_host_single_object, s1.handle, data.ctypes.data, off.ctypes.data, n, k)
        sides[name] = (dev_run, host_run, (d_data, d_off, data, off))
    want = po.COracle().decode_threaded_packed(v1, h_data, h_off, n, k, threads=os.cpu_count() or 4)
    for name, (dev_run, host_run, _) in sides.items():   # checked outside the timed loops
        h = dev_run()
        pr._check(L.rv_result_to_host(h))
        got = pr._export_batches(h, s1)
        assert len(got) == len(want)
        for i, (b, w) in enumerate(zip(got, want)):
            d = po.canon_diff(po.canon_from_batch(b), w, f"{name} batch[{i}]")
            assert d is None, d
        emit({"pair": "decode", "side": name, "checked": "oracle"})
    for rnd in range(a.rounds):
        for name, (dev_run, host_run, _) in sides.items():
            emit({"pair": "decode", "side": name, "round": rnd, "device_ms": round(timed(freed(dev_run)), 3),
                  "host_e2e_ms": round(host_ms(freed(host_run)), 3)})
    del sides

    # ---- decode: two writers alternating per message, read as v2 ----------------------------------------------------
    cdata, coff, _, _, _, _ = VC.kafka_versions_input(n, "alternate", ids=(3, 4), k=k)
    sdata, soff = kafka_single_object_input(n, k, v1, v2, h_data, h_off)
    v_conf = pr._get_or_create_versions({3: v1, 4: v2}, v2, None)
    v_so = pr.Versions([v1, v2], v2, single_object=True)
    sides = {}
    for name, v, data, off in (("confluent_versions", v_conf, cdata, coff), ("single_object_versions", v_so, sdata, soff)):
        d_data, d_off = on_device(data, off)
        sides[name] = (decode_call(L.rv_decode_device_versions, v.handle, d_data.data_ptr(), d_off.data_ptr(), n, k, stream.cuda_stream),
                       decode_call(L.rv_decode_host_versions, v.handle, data.ctypes.data, off.ctypes.data, n, k), v, (d_data, d_off))
    for name, (dev_run, _, v, _) in sides.items():
        h = dev_run()
        pr._check(L.rv_result_to_host(h))
        VC.check_kafka_v2(pr._export_batches(h, v.reader), v1, v2, h_data, h_off, n, k)
        emit({"pair": "versions", "side": name, "checked": "oracle"})
    tbuf = (ctypes.c_float * 4)()
    for rnd in range(a.rounds):
        for name, (dev_run, host_run, _, _) in sides.items():
            ms = timed(freed(dev_run))
            L.rv_last_versions_timings(tbuf, 4)
            emit({"pair": "versions", "side": name, "round": rnd, "device_ms": round(ms, 3),
                  "last_call_ms": dict(zip(("partition", "decodes", "take", "device"), (round(x, 3) for x in tbuf))),
                  "host_e2e_ms": round(host_ms(freed(host_run)), 3)})
    del sides

    # ---- encode ------------------------------------------------------------------------------------------------------
    batch = pr.decode_packed(h_data, h_off, n, v1, 1)[0]   # pinned, as decoded
    bare = pr.serialize_record_batch(batch, v1, k)
    for name, fn, hdr in (("confluent", lambda: pr.serialize_confluent(batch, v1, 77, k), b"\x00" + (77).to_bytes(4, "big")),
                          ("single_object", lambda: pr.serialize_single_object(batch, v1, k), SO.header(SO.fingerprint(v1)))):
        out = fn()
        assert len(out) == len(bare)
        H = len(hdr)
        for g, w in zip(out, bare):
            gd, go, m = pr._packed_view(g)
            wd, wo, _ = pr._packed_view(w)
            assert m == len(w) and np.array_equal(np.diff(go), np.diff(wo) + H), f"{name}: message sizes"
            at = (go[:-1, None] + np.arange(H)).ravel()
            assert np.array_equal(gd[at].reshape(m, H), np.broadcast_to(np.frombuffer(hdr, np.uint8), (m, H))), f"{name}: headers"
            keep = np.ones(int(go[-1] - go[0]), dtype=bool)
            keep[at - go[0]] = False
            assert np.array_equal(gd[go[0]:go[-1]][keep], wd[wo[0]:wo[-1]]), f"{name}: datums differ from serialize_record_batch"
        emit({"pair": "encode", "side": name, "checked": "serialize_record_batch"})
    ebuf = (ctypes.c_float * 5)()
    for rnd in range(a.rounds):
        for name, fn in (("confluent", lambda: pr.serialize_confluent(batch, v1, 77, k)), ("single_object", lambda: pr.serialize_single_object(batch, v1, k))):
            for _ in range(a.warmup):
                fn()
            t = []
            kern = np.zeros(3)
            for _ in range(a.steps):
                t0 = time.perf_counter()
                fn()
                t.append((time.perf_counter() - t0) * 1e3)
                L.rv_last_encode_timings(ebuf, 5)
                kern += np.array(list(ebuf)[:3])
            emit({"pair": "encode", "side": name, "round": rnd, "host_e2e_median_ms": round(float(np.median(t)), 3),
                  "kernels_ms": round(float(kern.sum()) / a.steps, 3)})


if __name__ == "__main__":
    main()
