#!/usr/bin/env python
"""Runs the mjai decoder's logic (csrc/mjx_mjai.cuh, host build) under AddressSanitizer + UBSan over self-play logs in varied
formats (all accepted, arrays equal to the host path's) and over byte-level hostile mutations of them (declined or decoded
identically), so an out-of-range read on hostile text shows on the host. Usage (not part of the pytest suite):

    LD_PRELOAD=$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so) ASAN_OPTIONS=detect_leaks=0 \\
        python tests/sanitized_mjai_run.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import emul_lib as E
import mjai_lib as M
import validate_lib as VL

E.lib(sanitize=True)
rng = np.random.default_rng(31)
games = VL.emul_games(8, 1) + VL.emul_games(8, 0, seed0=5000)
texts = [M.game_text(g) for g in games] + [M.vary(g, rng) for g in games]
got = M.emul_decode([t.encode() for t in texts])
assert all(g is not None and M.same(g, M.host_decode(t.encode())) for t, g in zip(texts, got))
corpus = M.hostile_corpus(texts, 60, rng)
got = M.emul_decode([b for _, b in corpus])
declined = 0
for (cls, b), g in zip(corpus, got):
    if g is None:
        declined += 1
    else:
        want = M.host_decode(b)
        assert want is not None and M.same(g, want), cls
print(f"sanitised decoder run finished: {len(texts)} logs accepted, {len(corpus)} hostile logs, {declined} declined")
