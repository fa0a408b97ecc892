#!/usr/bin/env python
"""Runs the review (csrc/mjx_review.cuh and the review mode of csrc/mjx_replay.cuh, single-lane emulation build) under
AddressSanitizer + UBSan: whole reviews of self-play logs, their single-viewpoint versions and guard variants with the stub engine
(guard on and off), reviews whose reactions cannot be decoded, and renders into buffers cut short, so an out-of-range read or
write shows on the host. Usage (not part of the pytest suite):

    LD_PRELOAD=$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so) ASAN_OPTIONS=detect_leaks=0 \\
        python tests/sanitized_review_run.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import emul_lib as E
import review_lib
import validate_lib as VL
from viewpoint_lib import viewpoint

E.lib(sanitize=True)
games = VL.emul_games(3, 1, seed0=8300) + VL.emul_games(3, 0, seed0=8400)
logs = [(g, [0, 1, 2, 3]) for g in games] + [(viewpoint(games[0], p), [p]) for p in range(4)] + [(viewpoint(games[1], 0), [2])]
logs += review_lib.guard_logs(games)
for engine in (review_lib.StubEngine(True), review_lib.StubEngine(False), review_lib.IllegalStubEngine(True)):
    got = review_lib.emul_review(engine, [ev for ev, _ in logs], [s for _, s in logs])
    jobs = [(ev, p) for ev, ps in logs for p in ps]
    for (ev, _), (text, _, err, stop) in zip(jobs, got):
        assert (text is None) == (err != 0)
        assert text is None or text.count("\n") == len(ev)
        assert 0 <= stop <= len(ev)

# renders into short buffers: nothing is written at or past the capacity
L = E.lib()
rng = np.random.default_rng(7)
n = 3
ev_cnt = np.array([5, 0, 7], np.int32)
rec_off = np.array([0, 2, 2, 4], np.int64)
event = np.array([1, 1, 0, 6], np.int32)
kan = np.array([0, 1, 0, 0], np.uint8)
word = np.array([3 | (1 << 8) | (5 << 12), 0, 0, 8 | (2 << 8) | (0x05050505 << 24)], np.uint64)
info = np.array([[42, 7, 1, -1], [5, 7, 1, 5], [45, 1, 0, 45], [0, 15, 6, 0]], np.int32)
mask = rng.integers(0, 1 << 46, 4).astype(np.uint64)
q = rng.normal(size=(4, 46)).astype(np.float32)
i64s = np.array([[2, 10], [2, 10], [1, 3], [1, 4]], np.int64)
skip = np.zeros(n, np.uint8)
args = (n, ev_cnt.ctypes.data, rec_off.ctypes.data, 4, event.ctypes.data, kan.ctypes.data, word.ctypes.data, info.ctypes.data,
        mask.ctypes.data, q.ctypes.data, i64s.ctypes.data, skip.ctypes.data)
nb = np.zeros(n, np.int64)
L.emulr_render(*args, nb.ctypes.data, None, None, 0)
off = np.zeros(n + 1, np.int64)
off[1:] = np.cumsum(nb)
for cap in (0, 1, int(off[-1]) // 2, int(off[-1])):
    buf = np.zeros(max(cap, 1), np.uint8)
    L.emulr_render(*args, None, off.ctypes.data, buf.ctypes.data, cap)
print("sanitized review run ok")
