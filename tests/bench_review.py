#!/usr/bin/env python
"""Reviewing arena logs: mortal_b200.review.review_logs (batched, one device pass) against the per-line libriichi.mjai.Bot (what
mortal.py's review mode runs), both with a version-4 checkpoint on the fp32 DeviceEngine (TF32 off). N arena logs x 4 seats are
reviewed batched; the Bot reviews a subset of them (it is the slow leg). Prints one JSON line with logs/s and decisions/s of each,
the card and its power limit, read in the same run. Usage: python tests/bench_review.py [--logs 256] [--bot-logs 4]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logs", type=int, default=256)
    ap.add_argument("--bot-logs", type=int, default=4)
    a = ap.parse_args()
    import torch

    import mortal_ckpt
    from mortal_b200 import _lib
    from mortal_b200.engine import DeviceEngine
    from mortal_b200.libriichi.arena import OneVsThree
    from mortal_b200.model import load_mortal
    from mortal_b200.review import review_logs
    from review_lib import bot_review
    from test_gpu_arena_logs import DevEngine

    _lib.init(0)
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    tmp = tempfile.mkdtemp()
    torch.manual_seed(0)
    OneVsThree(disable_progress_bar=True, log_dir=tmp).py_vs_py(DevEngine(torch, "a", salt=0.1), DevEngine(torch, "b"), (31000, 7),
                                                                max(1, a.logs // 4))
    paths = sorted(os.path.join(tmp, f) for f in os.listdir(tmp))[: a.logs]
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    fx = mortal_ckpt.load_fixture()
    brain, dqn = load_mortal(mortal_ckpt.checkpoint("v4", fx["v4"]))
    engine = DeviceEngine(brain, dqn, version=4, enable_amp=False, enable_quick_eval=False, enable_rule_based_agari_guard=True)
    seats = [[0, 1, 2, 3]] * len(paths)
    review_logs(engine, paths[:8], seats[:8])  # warm-up: module load, cuDNN heuristics
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    got = review_logs(engine, paths, seats)
    torch.cuda.synchronize()
    t_batch = time.perf_counter() - t0
    assert all(r.error is None for rs in got for r in rs)
    dec = sum(int(r.action.numel()) for rs in got for r in rs)
    import gzip

    texts = [gzip.open(p, "rt").read() for p in paths[: a.bot_logs]]
    t0 = time.perf_counter()
    for t in texts:
        for s in range(4):
            bot_review(engine, t, s)
    t_bot = time.perf_counter() - t0
    dec_bot = sum(int(r.action.numel()) for rs in got[: a.bot_logs] for r in rs)
    print(json.dumps({"gpu": gpu, "logs": len(paths), "jobs": 4 * len(paths), "decisions": dec,
                      "batched_s": round(t_batch, 3), "batched_logs_per_s": round(len(paths) / t_batch, 2),
                      "batched_decisions_per_s": round(dec / t_batch, 1), "bot_logs": len(texts), "bot_s": round(t_bot, 3),
                      "bot_logs_per_s": round(len(texts) / t_bot, 3), "bot_decisions_per_s": round(dec_bot / t_bot, 1)}))


if __name__ == "__main__":
    main()
