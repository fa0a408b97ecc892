#!/usr/bin/env python
"""Runs k_grp_logs's logic (csrc/mjx_grp.cuh, host build) under AddressSanitizer + UBSan: on self-play logs and their mutations
(the Grp equals Grp.load_events, or a non-zero status where Python raises) and on hostile arrays (offsets, counts and capacities
out of range or inconsistent with each other, random presence bytes and deltas), so an out-of-range read or write shows on the
host. Usage (not part of the pytest suite):

    LD_PRELOAD=$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so) ASAN_OPTIONS=detect_leaks=0 \\
        python tests/sanitized_grp_run.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import emul_lib as E
import grp_lib as G
import log_mutations as LM
import validate_lib as VL

E.lib(sanitize=True)
rng = np.random.default_rng(41)
games = VL.emul_games(8, 1) + VL.emul_games(8, 0, seed0=6100)
logs = list(games)
for _, text in LM.mutated_corpus(games, 4, rng):
    try:
        logs.append([json.loads(ln) for ln in text.splitlines() if ln.strip()])
    except ValueError:
        pass
a = G.encode(logs)
out = G.run_emul(a)
for i, ev in enumerate(logs):
    want = G.host_grp(ev)
    assert (out[3][i] != 0) if isinstance(want, type) else (out[3][i] == 0 and G.same(G.grp_of(a, out, i), want)), i

# hostile arrays: every log's offsets and counts drawn around and past the arrays, capacities shrunk below what the logs need
n, n_hdr, n_ky = len(logs), len(a["hdr"]), len(a["kyoku"])
hostile = 0
for rep in range(400):
    h = dict(a)
    pick = lambda lo, hi: rng.integers(lo, hi, size=n).astype(np.int32)
    if rep % 5 == 0:
        h["ev_off"] = pick(-5, n_hdr + 5)
    if rep % 5 == 1:
        h["ev_cnt"] = pick(-5, n_hdr // 2)
    if rep % 5 == 2:
        h["ky_off"] = pick(-5, n_ky // 19 + 5)
    if rep % 5 == 3:  # presence bytes and deltas at random: any value is read, none is trusted for an index
        h["has"] = rng.integers(0, 256, size=n_hdr).astype(np.uint8)
        h["deltas"] = rng.integers(-2**31, 2**31, size=(n_hdr, 4)).astype(np.int32)
    cap_h = int(rng.integers(0, n_hdr + 1)) if rep % 5 == 4 else n_hdr
    cap_k = (int(rng.integers(0, n_ky // 19 + 1)) * 19) if rep % 5 == 4 else n_ky
    # the arrays the kernel may read are cut to the capacities, so ASan sees any read past them
    h["hdr"] = np.ascontiguousarray(h["hdr"][:cap_h]); h["deltas"] = np.ascontiguousarray(h["deltas"][:cap_h])
    h["has"] = np.ascontiguousarray(h["has"][:cap_h]); h["kyoku"] = np.ascontiguousarray(h["kyoku"][:cap_k])
    _, rank, final, status = G.run_emul(h)
    assert set(np.unique(status)) <= {0, 1, 2, 3} and not rank[status != 0].any() and not final[status != 0].any()
    hostile += int((status == 3).sum())
print(f"sanitised grp run finished: {n} logs, 400 hostile array sets ({hostile} CAPACITY statuses)")
