"""Hanchans per hour of the 1v3 evaluation (`mortal_b200.one_vs_three`) on the GPU — BENCHMARK, not a test.

Two version-4 192 x 40 checkpoints with random weights (seeded) play `--iters` iterations of `--games-per-iter` games for every
`iters_per_call` in `--iters-per-call`, each without and with `log_dir`, in one process. Every arm runs `one_vs_three` end to end
(engine loading, the games, the per-call Stat.from_games of both sides, the log files when asked) and is timed on the host clock;
every call ends in a copy back to the host. `Stat.from_games` is timed per call as well. The arms print their iteration lines to
a buffer, which is compared between arms: the games of arms with the same iters_per_call must be the same with and without logs.

    python tests/bench_one_vs_three.py [--games-per-iter 2000] [--iters 4] [--iters-per-call 1,2,4] [--out PATH]

One JSON object goes to stdout (and to --out): the card, its power limit and max SM clock, and per arm the games, seconds,
hanchans per hour and the time of Stat.from_games per 2,000 games.
"""
from __future__ import annotations

import argparse
import io
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def _checkpoints(d):
    import torch

    from mortal_b200.model import DQN, Brain, mortal_state_dict

    paths = {}
    for name, seed in (("challenger", 1), ("champion", 2)):
        torch.manual_seed(seed)
        brain, dqn = Brain(conv_channels=192, num_blocks=40, version=4), DQN(version=4)
        paths[name] = os.path.join(d, f"{name}.pth")
        torch.save({"mortal": mortal_state_dict(brain), "current_dqn": dqn.state_dict(),
                    "config": {"control": {"version": 4}, "resnet": {"conv_channels": 192, "num_blocks": 40}}}, paths[name])
    return paths


def _config(paths, games_per_iter, iters, iters_per_call, log_dir):
    side = lambda name: {"device": "cuda:0", "name": name, "state_file": paths[name], "stochastic_latent": False,
                         "enable_compile": False, "enable_amp": True, "enable_rule_based_agari_guard": True}
    return {"1v3": {"seed_key": 0x2000, "games_per_iter": games_per_iter, "iters": iters, "iters_per_call": iters_per_call,
                    "log_dir": log_dir, "challenger": side("challenger"), "champion": side("champion"),
                    "akochan": {"enabled": False}}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--games-per-iter", type=int, default=2000)
    ap.add_argument("--iters", type=int, default=4)
    ap.add_argument("--iters-per-call", default="1,2,4")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    from mortal_b200 import one_vs_three as ovt
    from mortal_b200 import stat

    if not torch.cuda.is_available():
        raise SystemExit("bench_one_vs_three needs a CUDA device")
    tmp = tempfile.mkdtemp(prefix="bench_1v3_")
    stat_times = []
    real = stat.Stat.from_games

    def timed(games, name, idx=None):
        t = time.perf_counter()
        r = real(games, name, idx)
        stat_times.append((len(games) if idx is None else len(idx), time.perf_counter() - t))
        return r

    stat.Stat.from_games = staticmethod(timed)
    try:
        paths = _checkpoints(tmp)
        ovt.one_vs_three(_config(paths, 64, 1, 1, ""), out=io.StringIO())  # warm-up: module loads, cuDNN algorithm choice
        arms = []
        lines = {}
        for ipc in (int(x) for x in args.iters_per_call.split(",")):
            for logs in (False, True):
                log_dir = os.path.join(tmp, "logs") if logs else ""
                stat_times.clear()
                out = io.StringIO()
                torch.cuda.synchronize()
                t = time.perf_counter()
                res = ovt.one_vs_three(_config(paths, args.games_per_iter, args.iters, ipc, log_dir), out=out)
                torch.cuda.synchronize()
                dt = time.perf_counter() - t
                n_games = args.iters * (args.games_per_iter // 4) * 4
                text = out.getvalue().split("=" * 50)[0]
                lines[(ipc, logs)] = text
                arms.append(dict(iters_per_call=ipc, log_dir=logs, games=n_games, seconds=round(dt, 2),
                                 hanchans_per_hour=round(n_games / dt * 3600),
                                 # both sides' Stat.from_games (two calls per arena call), per 2,000 games played
                                 from_games_ms_per_2000_games=round(1000 * sum(s for _, s in stat_times) * 2000 / n_games, 1),
                                 avg_pt=res.avg_pt, avg_pt_stderr=res.avg_pt_stderr,
                                 files=len(os.listdir(log_dir)) if logs else 0))
                print(json.dumps(arms[-1]), file=sys.stderr, flush=True)
                if logs:
                    shutil.rmtree(log_dir)
        ipcs = sorted({a["iters_per_call"] for a in arms})
        result = dict(card=_card(), games_per_iter=args.games_per_iter, iters=args.iters, arms=arms,
                      same_games_with_and_without_logs={str(i): lines[(i, False)] == lines[(i, True)] for i in ipcs},
                      same_lines_as_iters_per_call_1={str(i): lines[(i, False)] == lines[(ipcs[0], False)] for i in ipcs})
    finally:
        stat.Stat.from_games = real
        shutil.rmtree(tmp, ignore_errors=True)
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
