#!/usr/bin/env python
"""Runs the mjai log renderer (csrc/mjx_mjai_write.cuh, host build) under AddressSanitizer + UBSan over hand-built games (every event
type, every meta variant) and hostile inputs: random words, lengths past the capacity or negative, random bounds, records with
random keys, actions, flags and masks. Every rendered game must stay inside its buffer; valid games must equal the host writer.
Usage (not part of the pytest suite):

    LD_PRELOAD=$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so) ASAN_OPTIONS=detect_leaks=0 \\
        python tests/sanitized_mjai_write_run.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import emul_lib as E  # noqa: E402
import mjai_write_lib as W  # noqa: E402
import test_emul_mjai_write as T  # noqa: E402

E.lib(sanitize=True)
rng = np.random.default_rng(41)
for version in (4, 0):
    words, lens, rec = T.synthetic_batch(6, version, rng)
    T.compare(words, lens, rec, 6)
print("hand-built games equal the host writer")
W.format_f32(rng.integers(0, 1 << 32, size=1 << 20, dtype=np.uint64).astype(np.uint32))
hostile = 0
for trial in range(400):
    n, cap = int(rng.integers(1, 6)), int(rng.integers(1, 64))
    words = rng.integers(0, 1 << 63, size=(n, cap), dtype=np.int64).astype(np.uint64)
    if trial % 2:  # mostly valid types and tiles, so the walk goes deep
        words &= np.uint64(0x00FF_FFFF_FF1F_FF0F)
        words |= rng.integers(1, 15, size=(n, cap)).astype(np.uint64)
    lens = rng.integers(-2, cap + 3, size=n).astype(np.int32)
    n_steps = int(rng.integers(1, 8))
    bounds = rng.integers(-5, cap + 5, size=(n_steps, n)).astype(np.int32)
    nr = int(rng.integers(0, 40))
    recs = None
    if nr:
        recs = dict(table=rng.integers(0, n, nr), cycle=rng.integers(0, n_steps, nr), seat=rng.integers(0, 4, nr), kan=rng.integers(0, 2, nr),
                    action=rng.integers(-3, 50, nr), mask=rng.integers(0, 1 << 63, nr, dtype=np.int64).astype(np.uint64),
                    q=rng.standard_normal((nr, 46)).astype(np.float32), i64=rng.integers(-(1 << 62), 1 << 62, (nr, 2)),
                    flags=rng.integers(0, 16, nr), shanten=rng.integers(-9, 9, nr), row=rng.integers(0, 100, nr))
    status, texts = W.render(words, lens, bounds, recs)
    hostile += int((status != 0).sum())
print(f"sanitised renderer run finished: 400 hostile batches, {hostile} games with a non-zero status")
# the recorder: hostile row indices (negative, past row_cap) and more rows than the capacity left
bad_rows = 0
for trial in range(200):
    row_cap, n, cap = int(rng.integers(1, 40)), int(rng.integers(1, 60)), int(rng.integers(1, 80))
    recs = W.EmulRecords(cap)
    recs.count = int(rng.integers(0, cap))
    idx = rng.integers(-5, row_cap + 5, size=n)
    masks = rng.integers(0, 2, size=(row_cap, 46))
    obs = rng.standard_normal((row_cap, 1012, 34)).astype(np.float32) if trial % 2 else None
    recs.record(int(trial), rng.standard_normal((n, 46)), rng.integers(0, 8, row_cap), rng.integers(0, 8, row_cap),
                rng.integers(0, 46, row_cap), masks, idx=idx, greedy=rng.integers(0, 2, n), obs=obs, row_cap=row_cap)
    bad_rows += int(((idx < 0) | (idx >= row_cap)).sum())
print(f"sanitised recorder run finished: 200 calls, {bad_rows} hostile row indices")
