#!/usr/bin/env python
"""Runs k_replay_viewpoints's scan (csrc/mjx_replay.cuh replay_hidden_seats, single-lane emulation build) under AddressSanitizer +
UBSan: on hostile arrays (jobs of 0-3 events, offsets and counts past the words, start_kyoku words with no payload left, all-`?`
logs, `?` in dora markers and consumed tiles, random words), where every result must equal the restatement over the events or be
-1 (not marked), and on whole single-viewpoint replays with observations, so an out-of-range read shows on the host. Usage (not part
of the pytest suite):

    LD_PRELOAD=$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so) ASAN_OPTIONS=detect_leaks=0 \\
        python tests/sanitized_viewpoint_run.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import emul_lib as E
import validate_lib as VL
from mortal_b200 import dataset_codec as DC
from viewpoint_lib import hidden_seats, viewpoint

E.lib(sanitize=True)
rng = np.random.default_rng(43)
games = VL.emul_games(6, 1, seed0=8100) + VL.emul_games(6, 0, seed0=8200)


def scan(jobs):
    rep = E.EmulReplay(jobs)
    m = rep.viewpoints()
    rep.close()
    return m


# 1. whole single-viewpoint replays with observations, and the all-`?` / odd-`?` logs
for L in games[:4]:
    vs = [viewpoint(L, p) for p in range(4)]
    rep = E.EmulReplay(DC.build_jobs(vs, [[p] for p in range(4)]))
    assert rep.viewpoints().tolist() == [hidden_seats(v) for v in vs]
    for it in range(5000):
        rep.replay_step()
        if rep.num_rows() and it % 3 == 0:
            rep.encode_obs(sp=it % 9 == 0, version=4)
        if rep.live == 0:
            break
    assert rep.live == 0 and not rep.errs().any()
    rep.close()
odd = []
for L in games:
    all_q = [{**ev, "tehais": [["?"] * 13] * 4} if ev["type"] == "start_kyoku" else
             ({**ev, "pai": "?"} if ev["type"] == "tsumo" else ev) for ev in L]
    dq = [{**ev, "dora_marker": "?"} if ev["type"] in ("start_kyoku", "dora") else
          ({**ev, "consumed": ["?"] * len(ev["consumed"])} if "consumed" in ev else ev) for ev in L]
    odd += [all_q, dq]
jobs = DC.build_jobs(odd, [[0, 1, 2, 3]] * len(odd))
assert scan(jobs).tolist() == [hidden_seats(g) for g in odd for _ in range(4)]

# 2. hostile arrays: short jobs, offsets and counts past the words, payloads cut short, random words; every array is cut to the
# capacity the scan is given, so ASan sees any read past it
views = [viewpoint(L, int(rng.integers(4))) for L in games]
base = DC.build_jobs(views, [[0, 1, 2, 3]] * len(games))
n, n_hdr, n_ky = len(base["players"]), len(base["hdr"]), len(base["kyoku"]) // 19
want = np.array([hidden_seats(v) for v in views for _ in range(4)])
unmarked = 0
for rep_i in range(300):
    h = {k: v.copy() for k, v in base.items()}
    pick = lambda lo, hi: rng.integers(lo, hi, size=n).astype(np.int32)
    kind = rep_i % 6
    if kind == 0:
        h["ev_cnt"] = pick(0, 4)  # jobs of 0-3 events
    elif kind == 1:
        h["ev_off"] = pick(-5, n_hdr + 5)
    elif kind == 2:
        h["ev_cnt"] = pick(-5, n_hdr // 2)
    elif kind == 3:
        h["ky_off"] = pick(-5, n_ky + 5)
    elif kind == 4:  # start_kyoku words with no payload left
        h["kyoku"] = np.ascontiguousarray(h["kyoku"][: 19 * int(rng.integers(0, n_ky + 1))])
    else:  # random words and payload bytes: any value is read, none is trusted for an index
        h["hdr"] = rng.integers(0, 2**63, size=n_hdr, dtype=np.uint64)
        h["hdr"][rng.random(n_hdr) < 0.3] &= ~np.uint64(0xFF)
        h["hdr"][rng.random(n_hdr) < 0.2] |= np.uint64(1)  # start_kyoku
        h["kyoku"] = rng.integers(0, 2**63, size=len(h["kyoku"]), dtype=np.uint64)
    got = scan(h)
    assert ((got >= -1) & (got <= 15)).all()
    if kind in (1, 2, 3, 4):
        ok = got != -1
        if kind == 4:
            assert (got[ok] == want[ok]).all()
        unmarked += int((~ok).sum())
print(f"sanitised viewpoint run finished: {len(games)} logs, 300 hostile array sets ({unmarked} unmarked jobs)")
