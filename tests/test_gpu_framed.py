"""Framed inputs (SURVEY.md 8(f) rank 4): Confluent wire format (5-byte header per message) and Avro Object Container
Files.  Not in the reference (bare datums only, README.md:93-94); results must equal decoding the bare datums."""
import json
import random
import struct

import numpy as np
import pytest

import pyruhvro_b200 as pr
from oracle import pyoracle as po
from tests.golden import reference_datums as G
from tests.ocf_files import ocf_file
from tests.parity import assert_matches_oracle, gen_case

pytestmark = pytest.mark.gpu


def _confluent(recs, schema_id):
    return [b"\x00" + struct.pack(">I", schema_id) + r for r in recs]


@pytest.mark.parametrize("jit", [1, 0])
def test_confluent_header_is_skipped_inside_the_kernel(coracle, jit):
    import workloads
    pr.set_jit_enabled(jit)
    try:
        sj, data, off = workloads.generate("kafka", 40_000, seed=9)
        recs = [data[off[i]:off[i + 1]].tobytes() for i in range(40_000)]
        framed = _confluent(recs, 77)
        for k in (1, 8):
            assert_matches_oracle(coracle, pr.deserialize_confluent(framed, sj, k, schema_id=77), sj, data, off, len(recs), k, full_validate=False)
        assert_matches_oracle(coracle, pr.deserialize_confluent(framed, sj, 3), sj, data, off, len(recs), 3, full_validate=False)   # any id
        # packed C-ABI form
        fd, fo = po.pack_records(framed)
        got = pr.decode_packed(fd, fo, len(framed), sj, 2, framing=pr.Framing(5, 1, 77))
        assert_matches_oracle(coracle, got, sj, data, off, len(recs), 2, full_validate=False)
        for seed in (3, 11):                                    # random schemas, ragged messages
            sj2, recs2, data2, off2 = gen_case(seed, n=700)
            assert_matches_oracle(coracle, pr.deserialize_confluent(_confluent(recs2, 5), sj2, 2, schema_id=5), sj2, data2, off2, 700, 2)
        # errors carry the record index
        bad = list(framed)
        bad[1234] = b"\x01" + bad[1234][1:]
        with pytest.raises(ValueError, match=r"framed message.*record 1234"):
            pr.deserialize_confluent(bad, sj, 4)
        with pytest.raises(ValueError, match=r"framed message.*record 0"):
            pr.deserialize_confluent(framed, sj, 4, schema_id=78)
        with pytest.raises(ValueError, match=r"framed message.*record 39999"):
            pr.deserialize_confluent(framed[:-1] + [b"\x00\x00"], sj, 1)
    finally:
        pr.set_jit_enabled(-1)


def test_object_container_file(coracle):
    import workloads
    rng = random.Random(12)
    sj, data, off = workloads.generate("kafka", 30_000, seed=4)
    recs = [data[off[i]:off[i + 1]].tobytes() for i in range(30_000)]
    f = ocf_file(sj, recs, [1, 7, 300, 1000], rng)
    for k in (1, 4):
        got = pr.deserialize_ocf(f, k)
        assert_matches_oracle(coracle, got, sj, data, off, len(recs), k, full_validate=False)
    recs3 = [bytes.fromhex(h) for h in (G.G3_HEX, G.G4_HEX, G.G5_HEX)]      # G3 has trailing bytes inside the block: sizes disagree
    with pytest.raises(ValueError):
        pr.deserialize_ocf(ocf_file(G.G345_SCHEMA, recs3, [3], rng), 1)
    ok3 = [recs3[1], recs3[2]]
    d3, o3 = po.pack_records(ok3)
    assert_matches_oracle(coracle, pr.deserialize_ocf(ocf_file(G.G345_SCHEMA, ok3, [1], rng), 1), G.G345_SCHEMA, d3, o3, 2, 1)
    assert pr.deserialize_ocf(ocf_file(sj, [], [1], rng), 1)[0].num_rows == 0
    with pytest.raises(ValueError, match="magic"):
        pr.deserialize_ocf(b"nope" + f[4:], 1)
    with pytest.raises(ValueError, match="sync"):
        pr.deserialize_ocf(f[:-1] + bytes([f[-1] ^ 1]), 1)
    with pytest.raises(ValueError, match="codec"):
        pr.deserialize_ocf(ocf_file(sj, recs[:10], [10], rng, {"avro.codec": b"deflate"}), 1)
    cut = bytearray(ocf_file(sj, recs[:100], [100], rng))
    with pytest.raises(ValueError):
        pr.deserialize_ocf(bytes(cut[:len(cut) // 2]), 1)
