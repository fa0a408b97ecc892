#!/usr/bin/env python
"""Runs k_stat_logs's logic (csrc/mjx_stat.cuh, host build) under AddressSanitizer + UBSan: on self-play logs and their mutations
(counters equal Stat.from_game, or a non-zero status where Python raises) and on hostile arrays (offsets, counts and capacities
out of range or inconsistent with each other, random seat masks), so an out-of-range read shows on the host. Also runs the
decoder's deltas reader over byte-mutated hora and ryukyoku lines. Usage (not part of the pytest suite):

    LD_PRELOAD=$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so) ASAN_OPTIONS=detect_leaks=0 \\
        python tests/sanitized_stat_run.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import emul_lib as E
import log_mutations as LM
import stat_lib as S
import validate_lib as VL

E.lib(sanitize=True)
rng = np.random.default_rng(37)
games = VL.emul_games(8, 1) + VL.emul_games(8, 0, seed0=6000)
logs = list(games)
for _, text in LM.mutated_corpus(games, 4, rng):
    try:
        logs.append([json.loads(ln) for ln in text.splitlines() if ln.strip()])
    except ValueError:
        pass
a = S.encode(logs)
for m in range(16):
    out, status = S.run_emul(a, np.full(len(logs), m))
    for i, ev in enumerate(logs):
        want = S.host_row(ev, m)
        assert (status[i] == 0 and np.array_equal(out[i], want)) if want is not None else status[i] != 0, (i, m)

# hostile arrays: every log's offsets and counts drawn around and past the arrays, capacities shrunk below what the logs need
n, n_hdr, n_ky = len(logs), len(a["hdr"]), len(a["kyoku"])
hostile = 0
for rep in range(400):
    h = dict(a)
    pick = lambda lo, hi: rng.integers(lo, hi, size=n).astype(np.int32)
    if rep % 4 == 0:
        h["ev_off"] = pick(-5, n_hdr + 5)
    if rep % 4 == 1:
        h["ev_cnt"] = pick(-5, n_hdr // 2)
    if rep % 4 == 2:
        h["ky_off"] = pick(-5, n_ky // 19 + 5)
    cap_h = int(rng.integers(0, n_hdr + 1)) if rep % 4 == 3 else n_hdr
    cap_k = (int(rng.integers(0, n_ky // 19 + 1)) * 19) if rep % 4 == 3 else n_ky
    # the arrays the kernel may read are cut to the capacities, so ASan sees any read past them
    h["hdr"] = np.ascontiguousarray(a["hdr"][:cap_h]); h["deltas"] = np.ascontiguousarray(a["deltas"][:cap_h])
    h["has"] = np.ascontiguousarray(a["has"][:cap_h]); h["kyoku"] = np.ascontiguousarray(a["kyoku"][:cap_k])
    out, status = S.run_emul(h, rng.integers(0, 256, size=n))
    assert set(np.unique(status)) <= {0, 1, 2, 3} and not out[status != 0].any()
    hostile += int((status == 3).sum())

# the deltas reader over byte-mutated lines of the decoder's accepted hora / ryukyoku events
lines = [ln for ev in games for e in ev if e["type"] in ("hora", "ryukyoku") for ln in [json.dumps(e).encode()]]
for _ in range(4000):
    b = bytearray(lines[int(rng.integers(len(lines)))])
    for _ in range(int(rng.integers(1, 4))):
        k = int(rng.integers(len(b)))
        if rng.integers(2):
            b[k] = int(rng.integers(0, 256))
        else:
            del b[k:]
            if not b:
                break
    S.line_deltas(bytes(b))
print(f"sanitised stat run finished: {n} logs x 16 masks, 400 hostile array sets ({hostile} CAPACITY statuses), 4000 mutated lines")
