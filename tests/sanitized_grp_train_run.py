#!/usr/bin/env python
"""Runs the GRP training step's logic (csrc/mjx_grp_train.cuh, host build) under AddressSanitizer + UBSan: on random nets and
batches (equal to the torch restatement of the reference) and on hostile arrays (game indices, lengths, job groupings and game
offsets out of range or inconsistent with each other, rank rows that are no permutation; counts, shapes and weight counts the
argument checks must refuse), so an out-of-range read or write shows on the host. Usage (not part of the pytest suite):

    LD_PRELOAD=$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so) ASAN_OPTIONS=detect_leaks=0 \\
        python tests/sanitized_grp_train_run.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import emul_lib as E
import grp_train_lib as T

E.lib(sanitize=True)
rng = np.random.default_rng(47)

# valid runs: several shape classes, compared with the reference
for hidden, layers in ((64, 2), (5, 1), (33, 4)):
    grp = T.random_grp(hidden, layers, hidden)
    w, h, nl = T.pack(grp)
    feats = [T.random_feature(n, rng) for n in (1, 3, 9)]
    game = rng.integers(0, 3, size=40)
    length = np.array([rng.integers(1, len(feats[g]) + 1) for g in game])
    rank = np.array([rng.permutation(4) for _ in game])
    rank[0] = [1, 1, 2, 3]
    rc, loss, acc, g, status = T.run_emul(w, h, nl, feats, game, length, rank)
    assert rc == 0 and not status.any()
    want, want_acc = T.ref_step(grp, [torch.as_tensor(feats[a][:b]) for a, b in zip(game, length)], rank)
    assert abs(loss - want) <= 1e-12 * abs(want) and acc == want_acc and T.grad_err(g, grp) <= 1e-12

# hostile arrays: every array the kernels index drawn around and past its bounds; the arrays are exactly as long as the counts
grp = T.random_grp(12, 2, 9)
w, h, nl = T.pack(grp)
n_games, n_rows = 5, 30
counts = np.zeros(3, dtype=np.int64)
for rep in range(300):
    feat = rng.normal(size=(n_rows, 7)) * 3
    off = np.sort(rng.integers(0, n_rows + 1, size=n_games + 1)).astype(np.int32)
    if rep % 3 == 0:
        off = rng.integers(-4, n_rows + 6, size=n_games + 1).astype(np.int32)
    B = int(rng.integers(1, 20))
    J = int(rng.integers(1, B + 1))
    game = rng.integers(-2, n_games + 2, size=B)
    length = rng.integers(-1, 14, size=B)
    rank = rng.integers(-1, 5, size=(B, 4))
    max_steps = int(rng.integers(1, 14))
    jobs = dict(job_game=rng.integers(-2, n_games + 2, size=J).astype(np.int32),
                job_steps=rng.integers(-1, 16, size=J).astype(np.int32), sample_job=rng.integers(-2, J + 2, size=B).astype(np.int32),
                job_sample_off=rng.integers(-3, B + 4, size=J + 1).astype(np.int32),
                job_sample=rng.integers(-2, B + 2, size=B).astype(np.int32), max_steps=max_steps)
    if rep % 4 == 0:
        jobs["job_sample_off"].sort()
    rc, loss, acc, g, status = T.run_emul(w, h, nl, dict(feat=feat, game_off=off), game, length, rank, grad=rep % 5 != 0,
                                          jobs=jobs)
    assert rc == 0 and set(np.unique(status)) <= {0, 1, 2}
    counts += np.bincount(status, minlength=3)

# argument checks: shapes and counts the kernels must refuse
f = [T.random_feature(4, rng)]
for kw in (dict(n_rows=0), dict(n_weights=w.size + 1), dict(n_samples=0), dict(scratch_bytes=16)):
    assert T.run_emul(w, h, nl, f, [0], [2], [[0, 1, 2, 3]], **kw)[0] == -2, kw
for hid, lay in ((0, 2), (300, 2), (12, 0), (12, 9)):
    assert T.run_emul(w, hid, lay, f, [0], [2], [[0, 1, 2, 3]])[0] == -2
print(f"sanitised GRP training run finished: 3 nets compared, 300 hostile array sets (sample statuses OK/GAME/LEN = "
      f"{counts.tolist()})")
