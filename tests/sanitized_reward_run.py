#!/usr/bin/env python
"""Runs k_grp_matrix's and k_train_targets's logic (csrc/mjx_reward.cuh, host build) under AddressSanitizer + UBSan: on random
nets and games (equal to the torch restatement of the reference) and on hostile arrays (game offsets, move ranges, game and seat
indices, at_kyoku and rank_by_player values out of range or inconsistent with each other; counts and shapes the argument checks
must refuse), so an out-of-range read or write shows on the host. Usage (not part of the pytest suite):

    LD_PRELOAD=$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so) ASAN_OPTIONS=detect_leaks=0 \\
        python tests/sanitized_reward_run.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import emul_lib as E
import reward_lib as R

E.lib(sanitize=True)
rng = np.random.default_rng(43)

# valid runs: every shape class, compared with the reference
for hidden, layers in ((64, 2), (5, 1), (33, 4)):
    grp = R.random_grp(hidden, layers, hidden)
    w, h, nl = R.pack(grp)
    feats = [R.random_feature(n, rng) for n in (1, 3, 9)]
    ranks, finals = [rng.permutation(4) for _ in feats], [rng.integers(0, 500, size=4) * 100 for _ in feats]
    gps = [R.random_gameplay(len(f), rng, int(rng.integers(0, 4)), g) for g, f in enumerate(feats) for _ in range(2)]
    jobs = R.jobs_of(gps, feats, ranks, finals)
    rc, m, steps, reward, rank, status = R.run_emul(w, h, nl, feats, jobs)
    assert rc == 0 and not status.any()
    off = np.cumsum([0] + [len(f) for f in feats])
    for g, f in enumerate(feats):
        assert np.abs(m[off[g]:off[g + 1]] - R.ref_calc_grp(grp, f).numpy()).max() <= 1e-12
    for j, (pid, ak, dn, ag, g) in enumerate(gps):
        sl = slice(jobs["move_off"][j], jobs["move_off"][j + 1])
        ws, wr, wk = R.ref_targets(R.ref_delta_pt(R.ref_calc_grp(grp, feats[g]), None, False, pid, ranks[g]), pid, feats[g], finals[g],
                                   ak, dn, ag)
        assert np.array_equal(steps[sl], ws) and np.array_equal(rank[sl], wk) and np.abs(reward[sl] - wr).max() <= 1e-10

# hostile arrays: every array the kernels index drawn around and past its bounds; the arrays are exactly as long as the counts
grp = R.random_grp(12, 2, 9)
w, h, nl = R.pack(grp)
n_games, n_rows = 6, 30
statuses = np.zeros(3, dtype=np.int64)
for rep in range(300):
    feat = rng.normal(size=(n_rows, 7)) * 3
    off = np.sort(rng.integers(0, n_rows + 1, size=n_games + 1)).astype(np.int32)
    if rep % 3 == 0:
        off = rng.integers(-4, n_rows + 6, size=n_games + 1).astype(np.int32)
    n_jobs = int(rng.integers(1, 12))
    move_off = np.sort(rng.integers(0, 80, size=n_jobs + 1)).astype(np.int32)
    if rep % 3 == 1:
        move_off = rng.integers(-5, 90, size=n_jobs + 1).astype(np.int32)
    n_moves = int(rng.integers(0, 81))
    jobs = dict(move_off=move_off, job_game=rng.integers(-2, n_games + 2, size=n_jobs), job_player=rng.integers(0, 6, size=n_jobs),
                at_kyoku=rng.integers(-3, 12, size=n_moves), apply_gamma=rng.integers(0, 256, size=n_moves),
                dones=rng.integers(0, 256, size=n_moves), rank=rng.integers(0, 6, size=(n_games, 4)),
                final=rng.integers(-2**40, 2**40, size=(n_games, 4)), n_moves=n_moves)
    rc, m, steps, reward, rank, status = R.run_emul(w, h, nl, dict(feat=feat, game_off=off), jobs, uniform_init=rep % 2)
    assert rc == 0 and set(np.unique(status)) <= {0, 1, 2}
    statuses += np.bincount(status, minlength=3)

# argument checks: shapes and counts the kernels must refuse
f = [R.random_feature(4, rng)]
for kw in (dict(n_rows=-1), dict(n_weights=w.size + 1)):
    assert R.run_emul(w, h, nl, f, **kw)[0] == -2, kw
for hid, lay in ((0, 2), (300, 2), (12, 0), (12, 9)):
    assert R.run_emul(w, hid, lay, f)[0] == -2
print(f"sanitised reward run finished: 3 nets compared, 300 hostile array sets (job statuses OK/CAPACITY/KYOKU = "
      f"{statuses.tolist()})")
