"""Every one of the 2^32 float32 bit patterns through the mjai writer's Q-value formatter (csrc/mjx_mjai_write.cuh mw_format_f32, host
build) against CPython's PyOS_double_to_string(x, 'r', 0, Py_DTSF_ADD_DOT_0) — what json.dumps(float(np.float32(x))) prints — and
json's NaN / Infinity / -Infinity. One process per slice (each holds its own GIL for the callbacks). Prints the mismatch count.

    python tests/check_float_repr_exhaustive.py [--procs N] [--slices M]
"""
from __future__ import annotations

import argparse
import multiprocessing as mp
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _slice(bounds):
    import mjai_write_lib as W

    return (bounds[0],) + W.sweep(bounds[0], bounds[1])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--procs", type=int, default=os.cpu_count())
    ap.add_argument("--slices", type=int, default=4096)
    a = ap.parse_args()
    import emul_lib

    emul_lib.build()
    step = (1 << 32) // a.slices
    parts = [(i * step, (i + 1) * step if i + 1 < a.slices else 1 << 32) for i in range(a.slices)]
    t0, bad, first = time.time(), 0, None
    with mp.Pool(a.procs) as pool:
        for k, (lo, n, f) in enumerate(pool.imap_unordered(_slice, parts)):
            bad += n
            if n and (first is None or f < first):
                first = f
            if (k + 1) % 256 == 0:
                print(f"{k + 1}/{a.slices} slices, {bad} mismatches, {time.time() - t0:.0f} s", flush=True)
    print(f"2^32 float32 patterns: {bad} mismatches" + (f" (first {first:#010x})" if first is not None else "")
          + f", {time.time() - t0:.0f} s with {a.procs} processes")
    return 1 if bad else 0


if __name__ == "__main__":
    sys.exit(main())
