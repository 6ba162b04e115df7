#!/usr/bin/env python
"""Damaged-input fuzz at any size (tests/mutation.py): valid datums of random schemas get byte-level damage; the C oracle
says whether the batch still decodes (then every buffer must match) or which record fails first with which category (then
the implementation under test must say the same).

    python tools/mutation_fuzz.py FIRST_SEED N [emu-interp | emu-gen | emu-warp | gpu-interp | gpu-jit] [--forge]

--forge: structured damage instead (tests/mutation.forge_varints: edge-value / padded / over-long varints spliced in).

emu-*: the host emulation of the product's readers (no GPU; emu-warp: the generated walkers with each fast emit warp in
lock step, so the item-parallel list emit runs); gpu-*: the CUDA path through rv_decode_host.  emu-gen, emu-warp and
gpu-jit draw their schemas from 80 seeds (one compilation each)."""
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    forge = "--forge" in sys.argv
    argv = [a for a in sys.argv if a != "--forge"]
    first, count = int(argv[1]), int(argv[2])
    mode = argv[3] if len(argv) > 3 else "emu-interp"
    from oracle import pyoracle as po
    from tests import mutation as M
    co = po.COracle()
    if mode.startswith("emu"):
        from tests import emu
        walker = "gen" if mode.endswith("gen") else "interp"
        decode = lambda sj, data, off, n, k: emu.decode(sj, data, off, n, k, walker=walker)  # noqa: E731
        if mode == "emu-warp":
            from tests.emu import warp
            decode = warp.decode
        error_of = lambda e: (po.ERR_NAMES.get(e.code, str(e.code)), e.record) if isinstance(e, emu.EmuError) else None  # noqa: E731
        supported = lambda sj: True  # noqa: E731
    else:
        import pyruhvro_b200 as pr
        from tests.test_zz_gpu_damaged_inputs import _gpu as decode, _gpu_error as error_of
        pr.set_jit_enabled(1 if mode.endswith("jit") else 0)
        supported = lambda sj: pr.Schema(sj).is_supported  # noqa: E731
    few = mode in ("emu-gen", "emu-warp", "gpu-jit")
    seen = {"decoded": 0, "error": 0}
    bad = 0
    t0 = time.time()
    for seed in range(first, first + count):
        sj, recs, k = (M.forged_case if forge else M.damaged_case)(seed, schema_seed=7000 + seed % 80 if few else None)
        if not supported(sj):
            continue
        try:
            seen[M.check(co, decode, error_of, sj, recs, k)] += 1
        except AssertionError as e:
            bad += 1
            print(f"FAIL seed={seed} k={k}: {str(e)[:300]}", flush=True)
    print(f"mutation fuzz ({mode}{', forged varints' if forge else ''}): decoded-equal {seen['decoded']}, same-error {seen['error']}, failures {bad}, {int(time.time() - t0)} s")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
