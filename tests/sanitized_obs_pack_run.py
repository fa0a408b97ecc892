#!/usr/bin/env python
"""Runs k_obs_pack's and k_obs_unpack's logic (csrc/mjx_obs_pack.cuh, host build) under AddressSanitizer + UBSan: round trips of
oracle observations of every version, hostile cells in mask rows (0.5, -0.0, NaN, 2.0, denormals, infinities), random bits in
value rows, sample pitches larger than an observation, gathers with repeats and with indices outside the records, and the
arguments the checks must refuse, so an out-of-range read or write shows on the host. Usage (not part of the pytest suite):

    LD_PRELOAD=$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so) ASAN_OPTIONS=detect_leaks=0 \\
        python tests/sanitized_obs_pack_run.py
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, ROOT)
import emul_lib as E
import obs_pack_lib as P

E.lib(sanitize=True)
rng = np.random.default_rng(47)
bits = lambda a: np.ascontiguousarray(a).view(np.int32)
hostile = np.array([0.5, -0.0, np.nan, 2.0, 1e-45, -1e-40, np.inf, -1.0], dtype=np.float32)
n_refused = 0
for version in (1, 2, 3, 4):
    obs, inv = P.sample_obs(version, seed=version)
    for invisible, x in ((False, obs), (True, inv)):
        vals = P.value_rows(version, invisible)
        mask_rows = np.setdiff1d(np.arange(x.shape[1]), vals)
        # round trip with a pitch of 1.5 observations (read in place from a larger buffer)
        rows = x.shape[1]
        pitch = rows * 34 + rows * 17
        buf = np.full((len(x), pitch), np.nan, dtype=np.float32)
        buf[:, :rows * 34] = x.reshape(len(x), -1)
        rc, rec, status = P.pack(buf, version, invisible, pitch=pitch, n=len(x))
        assert rc == 0 and not status.any()
        idx = rng.integers(-3, len(x) + 3, size=2 * len(x))
        rc, y = P.unpack(rec, idx, version, invisible)
        ok = (idx >= 0) & (idx < len(x))
        assert rc == 0 and np.array_equal(bits(y[ok]), bits(x[idx[ok]])) and not y[~ok].any()
        # hostile mask cells and random value-row bits
        for rep in range(20):
            z = x.copy()
            zb = z.view(np.uint32)
            zb[:, vals] = rng.integers(0, 2**32, size=(len(z), len(vals), 34), dtype=np.uint32)
            want = np.zeros(len(z), dtype=np.int32)
            for i in rng.choice(len(z), size=len(z) // 3, replace=False):
                r = sorted(rng.choice(mask_rows, size=int(rng.integers(1, 5)), replace=False))
                for row in r:
                    z[i, row, int(rng.integers(0, 34))] = hostile[int(rng.integers(0, len(hostile)))]
                want[i] = r[0] + 1
            rc, rec, status = P.pack(z, version, invisible)
            assert rc == 0 and np.array_equal(status, want)
            n_refused += int((status != 0).sum())
            clean = np.nonzero(want == 0)[0]
            rc, y = P.unpack(rec, clean, version, invisible)
            assert rc == 0 and np.array_equal(bits(y), bits(z[clean]))
# arguments the checks must refuse
x = P.sample_obs(1, seed=9)[0][:3]
for version, invisible, kw in ((0, 0, {}), (5, 0, {}), (1, 2, {}), (1, 0, dict(pitch=100)), (1, 0, dict(n=-1))):
    assert P.pack(x, version, invisible, **kw)[0] == -2
rc, rec, _ = P.pack(x, 1, 0)
assert P.unpack(rec, [0], 0, 0)[0] == -2 and P.unpack(rec, [0], 1, 0, n_records=-1)[0] == -2
print(f"sanitised obs pack run finished: 4 versions x (plain, invisible), {n_refused} hostile samples refused")
