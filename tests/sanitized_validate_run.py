#!/usr/bin/env python
"""Runs the log validator's logic (csrc/mjx_validate.cuh, single-lane emulation build) under AddressSanitizer + UBSan over mutated
self-play logs (verdicts must equal the oracle's) and over hostile event-word sequences (every log must get a verdict). Shows on
the host that hostile input is rejected before the device sees it. Usage (not part of the pytest suite; takes ~1 minute):

    LD_PRELOAD=$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so) ASAN_OPTIONS=detect_leaks=0 \\
        python tests/sanitized_validate_run.py
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
import validate_lib as VL
from mortal_b200.validate_logs import encode_log

E.lib(sanitize=True)
games = VL.emul_games(16, 1) + VL.emul_games(16, 0, seed0=5000)
corpus = LM.mutated_corpus(games, 10, np.random.default_rng(11))
assert VL.emul_validate([t for _, t in corpus]) == [VL.oracle_validate(t) for _, t in corpus]
enc = [encode_log("\n".join(json.dumps(e) for e in g)) for g in games]
rows = VL.emul_run_packed(LM.malformed_batch(enc, 2000, np.random.default_rng(12)))
assert ((rows[:, 0] >= 0) & (rows[:, 0] <= 4)).all()
print("sanitised validation run finished: mutated", len(corpus), "malformed", len(rows), "verdicts by status",
      np.bincount(rows[:, 0], minlength=5).tolist())
