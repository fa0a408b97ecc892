#!/usr/bin/env python
"""Runs the arena-words converter (csrc/mjx_selfplay.cuh, host build) under AddressSanitizer + UBSan over emulated self-play games,
hand-built games and hostile inputs: random words, lengths past the capacity or negative, a pitch wider than the capacity, and
every capacity argument cut short. Valid games must equal the written files' arrays; no read or write may leave its buffer.
Usage (not part of the pytest suite):

    LD_PRELOAD=$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so) ASAN_OPTIONS=detect_leaks=0 \\
        python tests/sanitized_selfplay_run.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import emul_lib as E  # noqa: E402

E.lib(sanitize=True)
import test_emul_mjai_write as MW  # noqa: E402
import test_emul_selfplay as T  # noqa: E402

words, lens = T.emul_games(4, 0, 1)
for augment in (False, True):
    _, got = T.convert(words, lens, augment)
    for g in range(4):
        T.check_game(got[g], T.reference(words[g], int(lens[g]), augment))
words, lens, _ = MW.synthetic_batch(3, 4, np.random.default_rng(9))
_, got = T.convert(words, lens, True)
for g in range(3):
    T.check_game(got[g], T.reference(words[g], int(lens[g]), True))
for short in (1, 2, 5):
    T.convert(words, lens, short=short)
print("self-play and hand-built games equal the written files' arrays")
rng = np.random.default_rng(43)
statuses = np.zeros(3, dtype=np.int64)
for trial in range(500):
    n, cap = int(rng.integers(1, 6)), int(rng.integers(1, 64))
    pitch = cap + int(rng.integers(0, 3))
    w = rng.integers(0, 1 << 63, size=(n, pitch), dtype=np.int64).astype(np.uint64)
    if trial % 2:  # mostly valid types and tiles, so the walk goes deep
        w &= np.uint64(0x00FF_FFFF_FF1F_FF0F)
        w |= rng.integers(1, 15, size=(n, pitch)).astype(np.uint64)
    ln = rng.integers(-2, cap + 3, size=n).astype(np.int32)
    counts, _ = T.convert(w, ln, bool(trial % 3 == 0), log_cap=cap, short=int(rng.integers(0, 3)))
    statuses += np.bincount(counts[:, 0], minlength=3)[:3]
print(f"sanitised converter run finished: 500 hostile batches, statuses OK / CORRUPT / CAPACITY = {statuses.tolist()}")
