#!/usr/bin/env python
"""Online training throughput: the sequential loop against self-play actors beside the trainer (not part of the pytest suite).

    python tests/bench_online.py [--rounds 4] [--games 400] [--capacity 400] [--batch-size 512] [--channels 192] [--blocks 40]

Builds random-init checkpoints (the baseline Brain / DQN of `--channels` x `--blocks`, a GRP) in a temporary directory and runs
`train_online` from a fresh trainer of the same size for `--rounds` rounds in each arm, one after another in this process:
  seq       the sequential loop (no `actor_devices`);
  same:1    one actor on the trainer's GPU (cuda:0), force_sequential = false;
  same:2    two actors on the trainer's GPU;
  other:N   one actor on each other GPU, when there are any.
Nothing is saved or test-played during the timed rounds (save_every = test_every = 10**6, submit_every = `--submit-every`).

Per arm it reports the trainer's steps/s and the games/s trained on, both over the rounds after the first (from the end of the
first training pass to the end of the last, so the actors' start-up and the first round's wait are not counted), the mean
param-version lag of the drained sessions (the version at drain minus the version the session played; 0 for the sequential
loop, which always plays the current parameters), and the whole call's wall time. It prints one JSON line with every arm, the
GPU's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import mortal_b200.train as train_mod  # noqa: E402
from mortal_b200.model import DQN, GRP, Brain, mortal_state_dict  # noqa: E402


def _config(d, args):
    resnet = {"conv_channels": args.channels, "num_blocks": args.blocks}
    return {
        "control": {"version": 4, "online": True, "batch_size": args.batch_size, "opt_step_every": 1, "save_every": 10**6,
                    "test_every": 10**6, "submit_every": args.submit_every, "device": "cuda:0", "enable_cudnn_benchmark": False,
                    "enable_amp": True, "enable_compile": False, "state_file": os.path.join(d, "mortal.pth"),
                    "best_state_file": os.path.join(d, "best.pth"), "tensorboard_dir": os.path.join(d, "tb")},
        "dataset": {"globs": [], "file_index": os.path.join(d, "index.pth"), "file_batch_size": 20, "reserve_ratio": 0.0,
                    "num_workers": 1, "player_names_files": [], "num_epochs": 1, "enable_augmentation": False,
                    "augmented_first": False},
        "env": {"gamma": 1.0, "pts": [6.0, 4.0, 2.0, 0.0]},
        "resnet": resnet,
        "cql": {"min_q_weight": 5.0},
        "aux": {"next_rank_weight": 0.2},
        "freeze_bn": {"mortal": False},
        "optim": {"eps": 1e-8, "betas": [0.9, 0.999], "weight_decay": 0.1, "max_grad_norm": 1.0,
                  "scheduler": {"peak": 1e-4, "final": 1e-5, "warm_up_steps": 100, "max_steps": 10**6}},
        "test_play": {"games": 8, "log_dir": os.path.join(d, "test_play")},
        "baseline": {"test": {"device": "cuda:0", "enable_compile": False, "state_file": os.path.join(d, "baseline.pth")},
                     "train": {"device": "cuda:0", "enable_compile": False, "state_file": os.path.join(d, "baseline.pth")}},
        "grp": {"network": {"hidden_size": 64, "num_layers": 2}, "state_file": os.path.join(d, "grp.pth")},
        "train_play": {"default": {"games": args.games, "log_dir": os.path.join(d, "train_play"), "boltzmann_epsilon": 0.005,
                                   "boltzmann_temp": 0.05, "top_p": 1.0, "repeats": 1}},
        "online": {"history_window": 50, "enable_compile": False, "remote": {"host": "127.0.0.1", "port": 5000},
                   "server": {"buffer_dir": os.path.join(d, "buffer"), "drain_dir": os.path.join(d, "drain"),
                              "capacity": args.capacity, "force_sequential": False}},
    }


def run_arm(root, name, actor_devices, args):
    d = os.path.join(root, name.replace(":", "_"))
    os.makedirs(d)
    for f in ("baseline.pth", "grp.pth"):
        os.link(os.path.join(root, f), os.path.join(d, f))
    cfg = _config(d, args)
    if actor_devices:
        cfg["online"]["actor_devices"] = actor_devices
    passes, lags = [], []
    inner = train_mod._train_pass

    def timed_pass(T, config, grp, games, steps, done):
        t0 = time.perf_counter()
        out = inner(T, config, grp, games, steps, done)
        torch.cuda.synchronize(T.device)
        passes.append((t0, time.perf_counter(), out - done, len(games)))
        return out

    def monitor(kind, **info):
        if kind == "drain":
            lags.extend(info["param_version"] - s.param_version for s in info["submissions"])

    train_mod._train_pass = timed_pass
    try:
        t0 = time.perf_counter()
        total = train_mod.train_online(cfg, rounds=args.rounds, monitor=monitor)[4]
        wall = time.perf_counter() - t0
    finally:
        train_mod._train_pass = inner
    window = passes[-1][1] - passes[0][1]
    steps = sum(p[2] for p in passes[1:])
    games = sum(p[3] for p in passes[1:])
    return {"actors": actor_devices or [], "total_steps": total, "games": sum(p[3] for p in passes), "wall_s": round(wall, 2),
            "steady_s": round(window, 2), "steps_per_s": round(steps / window, 3), "games_per_s": round(games / window, 3),
            "mean_param_lag": round(sum(lags) / len(lags), 3) if lags else 0.0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--games", type=int, default=400)
    ap.add_argument("--capacity", type=int, default=400)
    ap.add_argument("--batch-size", type=int, default=512)
    ap.add_argument("--submit-every", type=int, default=50)
    ap.add_argument("--channels", type=int, default=192)
    ap.add_argument("--blocks", type=int, default=40)
    args = ap.parse_args()
    if args.rounds < 2:
        raise SystemExit("--rounds must be at least 2: the rates are taken over the rounds after the first")
    if not torch.cuda.is_available():
        raise SystemExit("bench_online needs a CUDA device")
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    n_gpus = torch.cuda.device_count()
    arms = [("seq", None), ("same:1", ["cuda:0"]), ("same:2", ["cuda:0", "cuda:0"])]
    if n_gpus > 1:
        arms.append((f"other:{n_gpus - 1}", [f"cuda:{i}" for i in range(1, n_gpus)]))
    out = {"rounds": args.rounds, "games_per_session": args.games, "capacity": args.capacity, "batch_size": args.batch_size,
           "submit_every": args.submit_every, "net": f"{args.channels}x{args.blocks}", "gpus": gpu, "arms": {}}
    with tempfile.TemporaryDirectory() as root:
        torch.manual_seed(0)
        b = Brain(conv_channels=args.channels, num_blocks=args.blocks, version=4)
        torch.save({"mortal": mortal_state_dict(b), "current_dqn": DQN(version=4).state_dict(),
                    "config": {"control": {"version": 4}, "resnet": {"conv_channels": args.channels, "num_blocks": args.blocks}}},
                   os.path.join(root, "baseline.pth"))
        torch.save({"model": GRP(hidden_size=64, num_layers=2).state_dict()}, os.path.join(root, "grp.pth"))
        for name, devices in arms:
            torch.manual_seed(1)
            out["arms"][name] = run_arm(root, name, devices, args)
            print(f"{name}: {out['arms'][name]}", file=sys.stderr, flush=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
